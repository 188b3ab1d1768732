"""filtlong_b200 -- H100-native (sm_90a) implementation of Filtlong's per-read scoring and
filtering hot path behind a C ABI (include/filtlong_b200.h). See DESIGN.md."""
from .capi import FLError, make_params  # noqa: F401

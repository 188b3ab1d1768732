"""The work-item Phred kernels' schedule (tests/phred_items_model.py) against the oracle's sequential loops, bit for
bit: the plan's items per read, the segment prediction and the merge's check, the mean chain's tiles. Window sizes
from 1 to 2^31 - 1: 1..15 and 16384 cover every residue of ws mod 16 on segmented reads, the three near 2^31 are where
ws + PH_SEG does not fit in an int. The designed reads must between them take every path of the model."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import phred_items_model as m


def check(reads, ws):
    """the model's mean and window quality of (kind, qual) reads equal the oracle's; the path counts per kind"""
    got, ks = m.score_designed(reads, m.Tables(ws))
    sc = orc.score([(b"A" * len(qs), qs) for _, qs in reads], orc.make_params(window_size=ws), None)
    for (kind, qs), g, row in zip(reads, got, sc.parents):
        assert g == (row.mean_q, row.window_q), (ws, kind, len(qs))
    return ks


@pytest.mark.parametrize("ws", m.WINDOWS)
def test_model_equals_the_oracle(ws):
    rng = np.random.default_rng(ws % 100003)
    ks = check(m.designed_reads(ws, rng), ws)
    for p in m.reachable_paths(ws):
        assert sum(st[p] for st in ks.values()) > 0, (p, ks)
    m.check_designed_paths(ws, ks)
    seams = [L for L in m.seam_lengths(ws) if L <= m.MAX_DESIGNED]
    randoms = [int(rng.integers(1, 60000)) for _ in range(4)]
    other = [("random", (np.clip(np.rint(rng.normal(rng.uniform(5, 30), 4, size=L)), 1, 50).astype(np.uint8) + 33).tobytes())
             for L in seams + randoms]
    check(other, ws)


def test_plan():
    # A read longer than PH_LONG but not longer than the window is one fused item. (Tested as L <= ws + PH_SEG in int,
    # ws > 2^31 - 16385 wrapped the sum negative: L = 30000, ws = 2^31 - 1 then had (L - ws + PH_SEG - 1) / PH_SEG =
    # -131068 segments, about 2^64 items.)
    for ws in (2 ** 31 - 16385, 2 ** 31 - 16384, 2 ** 31 - 1):
        assert m.items_of(30000, ws) == 1
    assert m.items_of(m.PH_LONG, 1) == 1 and m.items_of(m.PH_LONG + 1, 1) == 3
    assert m.items_of(10000 + m.PH_SEG, 10000) == 1 and m.items_of(10001 + m.PH_SEG, 10000) == 3
    assert m.items_of(10000 + 2 * m.PH_SEG, 10000) == 3
    assert m.items_of(10000 + 2 * m.PH_SEG + 1, 10000) == 4        # a one-base last segment
    assert m.items_of(2 ** 31 - 1, 1) == 1 + (2 ** 31 - 3) // m.PH_SEG + 1

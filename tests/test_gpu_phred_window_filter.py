"""k_phred_win's filter pass on the device: the adversarial reads of test_phred_window_filter_model (a minimum
that recurs in every step, a near-tie inside the filter band, the minimum in the last partial step or in the
first window, invalid bytes at the edges of the first window, the read and the last step, a grid-tie byte
only in the first window, L = ws + 1) next to ordinary reads, across the window kernel's sizes. Every read
must match the oracle bit for bit."""
import random

import numpy as np
import pytest

from tests import util
from tests.test_gpu_parity import full_check, run_both
from tests.test_phred_window_filter_model import adversarial_reads

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ws", [250, 16, 33, 64, 65, 128, 129, 200, 256])
def test_phred_window_filter_edges(ws):
    rng = np.random.default_rng(2000 + ws)
    reads = [(b"A" * len(qs), bytes(qs)) for qs in adversarial_reads(ws, random.Random(ws))]
    for L in [ws + 1, 2 * ws + 1, 9 * ws - 1, 4100, 40000]:
        reads.append((b"A" * L, util.rand_qual(rng, L, mean_q=rng.uniform(5, 30))))
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    paths, _ = ctx.phred_paths()
    assert paths["candidates"][0] > 0 and paths["reject_byte"][0] > 0
    ctx.close()

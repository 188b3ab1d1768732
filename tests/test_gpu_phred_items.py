"""The work-item Phred kernels on the device (k_phred_plan / k_phred_fill / k_phred_items / k_phred_mean_long /
k_phred_merge / k_phred_fallback): every window size outside 16..256, and all of them under FL_PHRED_MODE=0. The
cases aim at that path's own seams -- read lengths around the window, at PH_LONG and around segment edges (a one-base
last segment included), windows near 2^31 where ws + PH_SEG does not fit in an int -- at the reads of
tests/phred_items_model.py that the model shows take each path (prediction failure and fallback, serial, retried and
tie-rejected tiles of the mean chain, bytes outside the Phred range), at the lattice kernels' seam corpora scored by
the work-item kernels instead, and at batching and the end of a device arena. Every read must match the oracle bit
for bit."""
import random

import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import phred_items_model as m
from tests import util
from tests.test_gpu_parity import full_check, run_both
from tests.test_gpu_phred_lengths import step_lengths
from tests.test_phred_window_filter_model import adversarial_reads

pytestmark = pytest.mark.gpu


def _read(rng, L, mean_q=None):
    return (b"A" * L, util.rand_qual(rng, L, mean_q=rng.uniform(5, 30) if mean_q is None else mean_q))


@pytest.mark.parametrize("ws", m.WINDOWS)
def test_plan_seams(ws):
    """lengths at the plan's seams between short reads, and one 1 Mbase read; for the windows near 2^31 every read is
    shorter than the window (one fused item each)"""
    rng = np.random.default_rng(7000 + ws % 100003)
    short = [_read(rng, 300) for _ in range(20)]
    reads = short[:10] + [_read(rng, L) for L in m.seam_lengths(ws)] + [_read(rng, 1_000_000, 15)] + short[10:]
    assert all(m.items_of(len(q), ws) == 1 for _, q in reads) == (ws > 1_000_000)
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", m.WINDOWS)
def test_designed_reads(ws):
    """the model's designed reads: each kind takes its path in the model (check_designed_paths), and the device
    computes the oracle's bits for all of them"""
    reads = m.designed_reads(ws, np.random.default_rng(ws % 100003))
    _, ks = m.score_designed(reads, m.Tables(ws))
    m.check_designed_paths(ws, ks)
    ctx, summ, sc, _ = run_both([(b"A" * len(q), q) for _, q in reads], dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", [16, 33, 64, 129, 250, 256])
def test_lattice_corpora_under_work_items(ws, monkeypatch):
    """the lattice kernels' seam corpora scored by the work-item kernels (FL_PHRED_MODE=0, read when the context is
    created): the oracle's bits, and the default mode's read and row arrays byte for byte"""
    rng = np.random.default_rng(3000 + ws)
    reads = [_read(rng, L) for L in step_lengths(ws)]
    reads += [(b"A" * len(qs), bytes(qs)) for qs in adversarial_reads(ws, random.Random(ws))]
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("FL_PHRED_MODE", mode)
        ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
        full_check(ctx, summ, sc)
        out[mode] = (ctx.read_results(), ctx.row_results())
        ctx.close()
    for x, y in zip(out["1"], out["0"]):
        for k in x:
            assert np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)), k


def _batch_reads(ws, rng):
    reads = [(b"A" * len(q), q) for _, q in m.designed_reads(ws, rng)[:6]]
    return reads + [_read(rng, L) for L in (ws + 1, 300, 30000, 5, ws + 2 * m.PH_SEG + 1)]


@pytest.mark.parametrize("ws", [7, 1000])
def test_results_do_not_depend_on_batching(ws):
    rng = np.random.default_rng(8000 + ws)
    reads = _batch_reads(ws, rng)
    outs = []
    for pushes in (1, 3):
        ctx = api.Context(api.make_params(keep_percent=70.0, window_size=ws))
        cuts = np.linspace(0, len(reads), pushes + 1).astype(int)
        for a, b in zip(cuts[:-1], cuts[1:]):
            ctx.push(api.HostBatch([s for s, _ in reads[a:b]], [q for _, q in reads[a:b]], want_seq=False))
        ctx.finalize(sum(len(s) for s, _ in reads))
        outs.append((ctx.read_results(), ctx.row_results()))
        ctx.close()
    for x, y in zip(*outs):
        for k in x:
            assert np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)), k


@pytest.mark.parametrize("ws", [7, 1000])
def test_arena_ends_with_a_segmented_read(ws):
    """device-resident batch whose quality arena is exactly padded_bases bytes, a segmented read last: no load of the
    segments, the mean chain's tiles or the fallback may reach beyond it"""
    import torch
    rng = np.random.default_rng(9000 + ws)
    reads = _batch_reads(ws, rng)
    assert m.items_of(len(reads[-1][1]), ws) == 4
    opts = dict(keep_percent=70.0, window_size=ws)
    sc = orc.finalize(orc.score(reads, orc.make_params(**opts), None), orc.make_params(**opts))
    hb = api.HostBatch([r[0] for r in reads], [r[1] for r in reads], want_seq=False)
    dev = torch.device("cuda", 0)
    qual = torch.from_numpy(hb.qual[:hb.padded_bases].copy()).to(dev)
    assert qual.numel() == hb.padded_bases
    off, length = torch.from_numpy(hb.off.view(np.int64)).to(dev), torch.from_numpy(hb.len).to(dev)
    ctx = api.Context(api.make_params(**opts), device=0)
    ctx.push_device(api.device_batch(hb.n, hb.padded_bases, off, length, qual=qual))
    torch.cuda.synchronize(dev)
    summ = ctx.finalize(hb.total_bases)
    full_check(ctx, summ, sc)
    ctx.close()

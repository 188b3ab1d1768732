"""k_phred_sum walks a read in 512-byte steps from the head k_phred_first summed, k_phred_win in steps of one window, one
warp per read taken longest first from a shared counter. The cases here aim at the seams of that: read lengths one base
around whole numbers of 512-byte steps (counted from 0 and from the head), one base over the head and over the window, a
1 Mbase read next to runs of short reads in both orders, reads the two kernels skip between reads they score, a single
read, invalid bytes in a read's first and last 512 bytes and at its last base, and a device arena that ends at the last
read's last padded byte. Every read must match the oracle bit for bit."""
import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import util
from tests.test_gpu_parity import full_check, run_both

pytestmark = pytest.mark.gpu

TILE, DEPTH = 512, 4          # k_phred_sum's step; how many steps the length cases go past
WINDOWS = [250, 16, 33, 64, 65, 128, 129, 200, 256]


def _read(rng, L, mean_q=None):
    return (b"A" * L, util.rand_qual(rng, L, mean_q=rng.uniform(5, 30) if mean_q is None else mean_q))


def step_lengths(ws):
    head = (ws + 15) & ~15
    out = [ws + 1, head + 1, head + 2]
    for k in list(range(1, 2 * DEPTH + 2)) + [3 * DEPTH, 3 * DEPTH + 1]:
        for d in (-1, 0, 1):
            out += [k * TILE + d, head + k * TILE + d]          # the window kernel starts at 0, the sum kernel at head
    return [L for L in out if L > 0]


@pytest.mark.parametrize("ws", WINDOWS)
def test_lengths_around_steps(ws):
    rng = np.random.default_rng(3000 + ws)
    reads = [_read(rng, L) for L in step_lengths(ws)]
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", WINDOWS)
def test_long_read_among_short_runs(ws):
    """1 Mbase reads before, between and after runs of 200-base reads (skipped by both kernels when ws >= 200, scored
    otherwise), with reads of a few steps and reads not longer than the window in between"""
    rng = np.random.default_rng(4000 + ws)
    short = [_read(rng, 200) for _ in range(40)]
    mixed = []
    for i in range(60):
        mixed.append(_read(rng, [ws, ws + 1, 3 * ws + 7, 700, 1500, 2049, 5000][i % 7]))
    reads = [_read(rng, 1_000_000, 12)] + short + mixed + [_read(rng, 1_000_000, 20)] + short[:17] + [_read(rng, ws - 1)]
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=80.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", [250, 16, 129])
@pytest.mark.parametrize("L", [300, 512 * 4, 40000])
def test_one_read(ws, L):
    rng = np.random.default_rng(L + ws)
    ctx, summ, sc, _ = run_both([_read(rng, L)], dict(keep_percent=100.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", WINDOWS)
def test_invalid_bytes_first_and_last_step(ws):
    """a byte outside the Phred range in a read's first 512 bytes, in its last ones, and at its last base: those reads go
    to k_phred_fallback, the reads around them do not"""
    rng = np.random.default_rng(5000 + ws)
    L = 6 * TILE + 37
    reads = []
    for pos in (ws + 3, TILE - 1, L - 40, L - 1):
        q = bytearray(_read(rng, L)[1])
        q[pos] = 0x20                                            # below '!'
        reads += [_read(rng, L), (b"A" * L, bytes(q))]
    reads.append(_read(rng, L))
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    paths, _ = ctx.phred_paths()
    # (a small window also rejects clean reads: their first window lies below the lattice's lower bound)
    assert paths["reject_byte"][0] >= 4 and sum(v[0] for v in paths.values()) == 9, paths
    ctx.close()


@pytest.mark.parametrize("ws", [250, 64])
def test_arena_ends_with_the_last_read(ws):
    """device-resident batch whose quality arena is exactly padded_bases bytes: no load may reach beyond it"""
    import torch
    rng = np.random.default_rng(6000 + ws)
    reads = [_read(rng, L) for L in (5000, 777, 2 * TILE, DEPTH * TILE + 1, 3 * TILE - 1)]
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

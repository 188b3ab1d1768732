"""--trim_q through the C ABI: per-read first / last / bad ranges / children and the rows equal the model
(tests/qtrim_model.py); every row's mean and window quality is bit-identical to the oracle's score of its substring;
normalisation and selection are exact over those rows. A context with trim_q = 0 is plain Phred mode, and trim_q with
a k-mer set is refused."""
import ctypes as C

import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import parity, util
from tests import qtrim_model as qm

pytestmark = pytest.mark.gpu


def reads_with_bad_blocks(seed, n, max_len=12000):
    """util.long_reads with low-quality blocks spliced into the qualities (start, middle, end), plus the crafted reads"""
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, 100000)
    out = []
    for name, seq, qual in util.long_reads(rng, genome, n, max_len=max_len):
        q = bytearray(qual)
        L = len(q)
        for _ in range(int(rng.integers(0, 4))):
            where = rng.random()
            ln = int(rng.integers(1, 900))
            s = 0 if where < 0.25 else (max(0, L - ln) if where < 0.5 else int(rng.integers(0, max(L, 1))))
            q[s:s + ln] = bytes(rng.integers(33, 33 + 6, size=len(q[s:s + ln])).astype(np.uint8))
        out.append((seq, bytes(q)))
    for _, qual, _ in qm.crafted():
        out.append((b"ACGT" * (len(qual) // 4) + b"A" * (len(qual) % 4), qual))
    return out


def run_ctx(reads, kw, pushes):
    ctx = api.Context(api.make_params(**kw))
    total = sum(len(s) for s, _ in reads)
    cuts = np.linspace(0, len(reads), pushes + 1).astype(int)
    for a, b in zip(cuts[:-1], cuts[1:]):
        ctx.push(api.HostBatch([s for s, _ in reads[a:b]], [q for _, q in reads[a:b]], want_seq=False))
    summary = ctx.finalize(total)
    return ctx, summary


CASES = [
    # Q, trim, split, window size, pushes, thresholds
    (10, True, None, 250, 1, dict(keep_percent=80.0)),
    (10, True, 500, 250, 3, dict(keep_percent=70.0, min_length=300)),
    (7, False, 1, 250, 1, dict(min_mean_q=9.0)),
    (20, True, 16, 16, 2, dict(target_bases=400000)),
    (20, False, 32, 250, 1, dict(keep_percent=90.0)),
    (10, False, 32, 300, 2, dict(keep_percent=60.0, min_window_q=5.0)),
    (7, True, 500, 300, 1, dict(keep_percent=50.0)),
    (20, True, 1, 100, 1, dict(min_length=100)),
    # window sizes the work-item kernels score; max_len (not a threshold) makes parents long enough that children of more
    # than PH_LONG = 24576 bases are cut into window segments
    (20, True, 16, 7, 1, dict(keep_percent=80.0)),
    (10, True, 500, 1000, 2, dict(keep_percent=70.0, max_len=100000)),
]


@pytest.mark.parametrize("Q,trim,split,ws,pushes,thr", CASES, ids=lambda x: str(x))
def test_rows_and_scores_equal_the_model(Q, trim, split, ws, pushes, thr):
    thr = dict(thr)
    max_len = thr.pop("max_len", None)
    reads = reads_with_bad_blocks(100 + Q + ws, 150, **({"max_len": max_len} if max_len else {}))
    kw = dict(window_size=ws, trim=trim, split=split, **thr)
    ctx, summary = run_ctx(reads, dict(kw, trim_q=Q), pushes)
    sc = qm.score_rows(reads, Q, kw)
    rr, rw = ctx.read_results(), ctx.row_results()
    parity.check_reads_vs_oracle(rr, sc)
    parity.check_rows_vs_oracle(rw, rr, sc, summary)
    p = api.make_params(**dict(kw, trim_q=Q))
    parity.check_rescale_exact(rw, summary, p)
    parity.check_selection_exact(rw, summary, p)
    assert sum(len(k) for k in sc.children) > len(reads) // 4          # the case does split reads
    if max_len:
        assert max(c.end - c.start for k in sc.children for c in k) > 24576
    ctx.close()


def test_trim_q_zero_is_plain_phred_mode():
    reads = reads_with_bad_blocks(3, 120)
    kw = dict(trim=True, split=500, keep_percent=80.0)
    ctx, summary = run_ctx(reads, dict(kw, trim_q=0), 2)
    op = orc.make_params(**kw)
    sc = orc.finalize(orc.score(reads, op), op)
    rr, rw = ctx.read_results(), ctx.row_results()
    parity.check_reads_vs_oracle(rr, sc)
    parity.check_rows_vs_oracle(rw, rr, sc, summary)
    assert len(rw["parent"]) == len(reads)
    ctx.close()


def test_device_push_equals_host_push():
    import torch
    reads = reads_with_bad_blocks(9, 100)
    kw = dict(trim=True, split=32, keep_percent=75.0, trim_q=12)
    a, _ = run_ctx(reads, kw, 1)
    hb = api.HostBatch([s for s, _ in reads], [q for _, q in reads], want_seq=False)
    b = api.Context(api.make_params(**kw))
    d = {k: torch.from_numpy(getattr(hb, k).view(np.int64 if k == "off" else getattr(hb, k).dtype)).cuda()
         for k in ("off", "len", "qual")}
    b.push_device(api.device_batch(hb.n, hb.padded_bases, d["off"], d["len"], qual=d["qual"]))
    b.finalize(hb.total_bases)
    for x, y in ((a.read_results(), b.read_results()), (a.row_results(), b.row_results())):
        for k in x:
            assert np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)), k
    a.close(); b.close()


def test_trim_q_with_a_kmer_set_is_refused():
    rng = np.random.default_rng(1)
    genome = util.rand_seq(rng, 5000)
    ctx = api.Context(api.make_params(trim=True, trim_q=10))
    ctx.kmers_add([genome], False)
    hb = api.HostBatch([genome[:1000]], [b"5" * 1000])
    rc = ctx.L.fl_reads_push(ctx.h, C.byref(hb.c_batch()))
    assert rc == -1
    assert b"trim_q" in ctx.L.fl_last_error(ctx.h)
    ctx.close()


def test_trim_q_out_of_range_is_refused():
    for q in (-1, 94):
        with pytest.raises(api.FLError):
            api.Context(api.make_params(trim=True, trim_q=q))

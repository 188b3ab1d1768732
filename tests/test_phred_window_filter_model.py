"""CPU model of k_phred_win's schedule (fl_phred.cu), against the oracle.

While the window chain stays in [0.5, 1) every window value is W0 plus a whole number of grid steps
(2^-53): bits(w_j) = bits(W0) + S_A(window j) - S_A(first window), A_c = a[c] on that grid as an integer.
The kernel first finds the minimum of the 32-bit filter sums S~ (A_c >> 30 per base), in the same lanes and
window-length steps as the exact walk, tracks per lane the step of its lowest filter value and the lowest
value of its other steps, and then walks exactly only the steps that can hold the true minimum (its S~ is
below the filter minimum + ws), or every step when such a lane has another step within ws of its lowest. Bytes the lattice
cannot take read as a sentinel filter value that lifts any window holding them above every valid sum.
This file restates that schedule in plain Python integers and floats and checks it bit for bit against
the oracle's sequential loop, on ordinary, adversarial and benchmark-like reads."""
import math
import random

import numpy as np
import pytest

from oracle import oracle as orc
from tests.test_phred_lattice_model import tables

SHIFT, BAD, NONE = 30, 1 << 23, (1 << 32) - 1


def grid_tables(ws, a):
    ra, fa = [], []
    for v in a:
        ok = v >= 0 and v * ws <= 1 - 1e-10
        if ok and v > 0:
            sc = math.ldexp(v, 53)
            ok = sc - math.floor(sc) != 0.5
        g = (0.5 + v) - 0.5
        ra.append(g if ok else float("nan"))
        fa.append(int(math.ldexp(g, 53)) >> SHIFT if ok else BAD)
    return ra, fa


def model_window(qs, ws, q, a, stats):
    """k_phred_win: returns the window minimum, or None when the read goes to k_phred_fallback."""
    L = len(qs)
    K = 2 if ws <= 64 else (4 if ws <= 128 else 8)
    ra, fa = grid_tables(ws, a)
    thr = 0.5 + 2 * max(x for x in ra if x == x)
    nb = [max(0, min(K, ws - K * l)) for l in range(32)]
    s0 = 0.0
    for c in qs[:ws]:
        s0 += q[c]
    W0 = s0 / ws
    if not (thr <= W0 < 1.0):
        stats["reject_byte"] += 1
        return None
    # filter pass
    S0f = sum(fa[c] for c in qs[:ws])
    if S0f >= BAD:
        stats["reject_byte"] += 1
        return None
    nsteps = (L - 1) // ws
    best, bstep, other = [NONE] * 32, [0] * 32, [NONE] * 32
    Wf = S0f
    for t in range(nsteps):
        j = ws + t * ws
        n = min(ws, L - j)
        inc = 0
        for l in range(32):
            x = m = 0
            for k in range(nb[l]):
                p = K * l + k
                if p < n:
                    x += fa[qs[j + p]] - fa[qs[j + p - ws]]
                    m = min(m, x)
            cand = Wf + inc + m
            other[l] = min(other[l], max(cand, best[l]))         # the lowest candidate of the lane's other steps
            if cand < best[l]:
                best[l], bstep[l] = cand, t
            inc += x
        Wf += inc
        assert 0 <= Wf < 1 << 32
        if Wf >= BAD:
            stats["reject_byte"] += 1
            return None
    mt = min(min(best), S0f)
    rel = [b <= mt + ws for b in best]
    ambiguous = any(rel[l] and other[l] <= best[l] + ws for l in range(32))
    walks = [(0, nsteps)] if ambiguous else [(t, t + 1) for t in sorted({bstep[l] for l in range(32) if rel[l]})]
    # exact pass: entry of step t from the identity, then the exact per-step walk
    S = lambda t: sum(int(math.ldexp(ra[c], 53)) for c in qs[t * ws:t * ws + ws])
    mn = W0
    for t0, t1 in walks:
        W = W0 + math.ldexp(S(t0) - S(0), -53)
        for t in range(t0, t1):
            j = ws + t * ws
            n = min(ws, L - j)
            off = 0.0
            for l in range(32):
                x = m = 0.75
                for k in range(nb[l]):
                    p = K * l + k
                    if p < n:
                        x = x + (ra[qs[j + p]] - ra[qs[j + p - ws]])
                        m = min(m, x)
                mn = min(mn, (W + off) + (m - 0.75))
                off += x - 0.75
            W += off
            stats["exact_steps"] += 1
    if not mn >= thr:
        stats["reject_low"] += 1
        return None
    stats["full_walk" if ambiguous else "candidates"] += 1
    return mn


def check_reads(reads, ws, stats):
    q, a = tables(ws)
    sc = orc.score([(b"A" * len(qs), bytes(qs)) for qs in reads], orc.make_params(window_size=ws), None)
    for qs, row in zip(reads, sc.parents):
        mn = model_window(qs, ws, q, a, stats)
        if mn is None:
            continue                                  # k_phred_fallback: the reference's own loop
        assert mn == mn
        assert 100.0 * (0.0 if mn < 0.5 / ws else mn) == row.window_q


def adversarial_reads(ws, rng):
    def noisy(L, mq=14.0):
        return [min(126, max(34, int(round(rng.gauss(mq, 4))) + 33)) for _ in range(L)]

    reads = []
    base = noisy(ws)
    reads.append(base * 9 + base[:ws // 3])                      # period ws: the minimum recurs in every step
    # two windows in different steps that differ by one Q40 <-> Q41 swap: a near-tie inside the band
    w1 = [33 + 40] * (ws // 2) + [33 + 41] * (ws - ws // 2)
    w2 = list(w1)
    w2[0], w2[-1] = 33 + 41, 33 + 40
    r = noisy(3 * ws, 42)
    r[ws:2 * ws] = w1
    r += noisy(2 * ws, 42) + w2 + noisy(ws // 2, 42)
    reads.append(r)
    r = noisy(6 * ws + ws // 2, 20)                               # minimum in the last, partial step
    r[-ws // 3:] = [33 + 6] * (ws // 3)
    reads.append(r)
    r = [33 + 8] * ws + noisy(5 * ws, 25)                         # minimum = the first window
    reads.append(r)
    for pos in (0, ws - 1, "last", "tail"):                       # an invalid byte
        r = noisy(4 * ws + ws // 2)
        p = {"last": len(r) - 1, "tail": 4 * ws + ws // 4}.get(pos, pos)
        r[p] = 200
        reads.append(r)
    reads.append([33 + 9] + noisy(6 * ws - 1))                    # Q9 (a grid tie at ws 200) only in the first window
    reads.append(noisy(ws + 1))
    reads.append([33 + 20] * (2 * ws) + [33 + 3] * ws + [33 + 20] * ws)   # the window dips below 0.5 after the first
    return reads


@pytest.mark.parametrize("ws", [250, 16, 33, 64, 100, 128, 200, 256])
def test_filter_schedule_reproduces_the_sequential_window(ws):
    rnd = random.Random(ws)
    stats = {k: 0 for k in ("candidates", "full_walk", "reject_byte", "reject_low", "exact_steps")}
    reads = adversarial_reads(ws, rnd)
    for t in range(18):                                           # the read kinds of test_phred_lattice_model
        L = rnd.randint(ws + 1, rnd.choice([1500, 6000]))
        kind = t % 6
        if kind == 0:
            qs = [rnd.randint(33 + 40, 33 + 50) for _ in range(L)]
        elif kind == 1:
            qs = [rnd.choice([33, 34, 126, 112, 122]) for _ in range(L)]
        elif kind == 2:
            qs = [min(126, max(33, int(round(rnd.gauss(3, 1.5))) + 33)) for _ in range(L)]
        else:
            mq = rnd.uniform(5, 40)
            qs = [min(126, max(34, int(round(rnd.gauss(mq, 4))) + 33)) for _ in range(L)]
        reads.append(qs)
    check_reads(reads, ws, stats)
    assert stats["full_walk"] > 0 and stats["candidates"] > 0 and stats["reject_byte"] > 0 and stats["reject_low"] > 0


def test_filter_paths_on_benchmark_reads():
    """A seeded sample of bench.py's config 2 reads (fl_synth_qual_host, default window): the filter alone
    decides almost every read, and few need the whole chain walked exactly."""
    from filtlong_b200 import capi
    S = capi.synth_host_lib()
    rng = np.random.default_rng(5)
    n = 40
    lens = np.clip(rng.lognormal(8.8, 0.9, size=n), 300, 60000).astype(np.int32)
    off = np.zeros(n, dtype=np.uint64)
    off[1:] = np.cumsum((lens.astype(np.uint64) + 63) & ~np.uint64(63))[:-1]
    qbar = np.clip(np.rint(rng.normal(14, 4, size=n)), 5, 30).astype(np.uint8)
    qual = np.zeros(int(off[-1]) + int(lens[-1]) + 64, dtype=np.uint8)
    S.fl_synth_qual_host(1, n, capi.ptr(off), capi.ptr(lens), capi.ptr(qbar), 0, capi.ptr(qual))
    reads = [list(qual[int(o):int(o) + int(L)]) for o, L in zip(off, lens)]
    stats = {k: 0 for k in ("candidates", "full_walk", "reject_byte", "reject_low", "exact_steps")}
    check_reads(reads, 250, stats)
    total_steps = sum((len(r) - 1) // 250 for r in reads)
    print("paths over %d reads: %r, exact steps %d of %d" % (n, stats, stats["exact_steps"], total_steps))
    assert stats["reject_byte"] == stats["reject_low"] == 0
    assert stats["full_walk"] <= n // 8
    assert stats["exact_steps"] <= total_steps // 4

"""CPU model of the work-item Phred kernels of fl_phred.cu: k_phred_plan / k_phred_fill (items per read),
k_phred_items (fused reads and window segments), k_phred_mean_long (the mean chain of a long read), k_phred_merge
and k_phred_fallback. These kernels score every window size outside 16..256, and all of them under FL_PHRED_MODE=0.

A read of at most PH_LONG bases, or not longer than ws + PH_SEG, is one fused item: the reference's loop. A longer
read is one mean item plus ceil((L - ws) / PH_SEG) window segments; segment k covers [ws + k PH_SEG, ...). Every
segment after the first starts from a PREDICTED entry value (grid steps in the binade of the first window), runs the
true chain, and the merge accepts the read only if each exit equals the next segment's predicted entry bit for bit;
otherwise the whole read is scored again by the reference's loop. The mean chain adds 2048-base tiles, or 128-base
pieces, on the grid of the sum's binade and walks a tile serially when it carries into the next binade, holds a
rounding tie or a byte outside the Phred range, or starts below 2^6.

Everything here is IEEE double arithmetic in plain Python floats and numpy float64, both round-to-nearest like the
library built with --fmad=false. Sequential chains use np.cumsum, which adds left to right (no pairwise summation):
a window chain is the cumulative sum of w0, -a[out_1], +a[in_1], -a[out_2], ... . score_read returns the mean, the
window quality and counts of the paths the read took, so tests can show that a designed read takes its path."""
import math

import numpy as np

from tests.test_phred_lattice_model import tables, tie_info

PH_SEG = 16384
PH_LONG = PH_SEG + PH_SEG // 2
TILE, PIECE = 2048, 128
PATHS = ("items", "segments", "fallback", "big", "retry", "small", "serial", "tie", "invalid")
LL_MIN, LL_MAX = -(1 << 63), (1 << 63) - 1
MAX_DESIGNED = 200_000                      # designed reads stay at or below this length
WINDOWS = [1, 2, 3, 7, 15, 257, 300, 470, 1000, 4097, 16383, 16384, 16385, 24576, 100000,
           2 ** 31 - 16385, 2 ** 31 - 16384, 2 ** 31 - 1]


def n_segments(L, ws):
    return (L - ws - 1) // PH_SEG + 1


def items_of(L, ws):
    """k_phred_plan: 1 for a fused read, 1 + segments for a long one"""
    return 1 if L <= PH_LONG or L - ws <= PH_SEG else 1 + n_segments(L, ws)


class Tables:
    def __init__(self, ws):
        q, a = tables(ws)
        self.ws = ws
        self.q = np.array(q)
        self.a = np.array(a)
        # k_phred_mean_long's shared table: a quality outside [0, 1) is NaN
        self.q_grid = np.where((self.q >= 0.0) & (self.q < 1.0), self.q, np.nan)
        self.tie_any, _ = tie_info(q)


def seq_sum(s, x):
    """s + x[0] + x[1] + ..., left to right"""
    if len(x) == 0:
        return s
    return float(np.cumsum(np.concatenate(([s], x)))[-1])


def window_chain(w, a_in, a_out):
    """w -= a_out[i]; w += a_in[i]; the exit value and the least value after an addition (+inf if none)"""
    n = len(a_in)
    if n == 0:
        return w, math.inf
    v = np.empty(2 * n + 1)
    v[0] = w
    v[1::2] = -a_out
    v[2::2] = a_in
    c = np.cumsum(v)
    return float(c[-1]), float(c[2::2].min())


def pow2(e):
    return math.ldexp(1.0, e) if e <= 1023 else math.inf


def double2ll_rn(x):
    """__double2ll_rn on an array: round half to even, saturate to the long long range"""
    assert not np.isnan(x).any()
    r = np.rint(x)
    out = np.zeros(len(r), dtype=np.int64)
    hi, lo = r >= 2.0 ** 63, r < -(2.0 ** 63)
    mid = ~(hi | lo)
    out[mid] = r[mid].astype(np.int64)
    out[hi], out[lo] = LL_MAX, LL_MIN
    return out


def wrap_ll(v):
    return (v - LL_MIN) % (1 << 64) + LL_MIN


def predicted_entry(w0, a_codes, P, ws):
    """score_segment's entry for the segment starting at P: w0 plus the grid steps S(P) - S(ws) in w0's binade"""
    e = math.frexp(w0)[1]
    scale = pow2(53 - e)
    s0 = int(double2ll_rn(a_codes[:ws] * scale).sum())            # long long adds: wrap mod 2^64
    sp = int(double2ll_rn(a_codes[P - ws:P] * scale).sum())
    return w0 + float(wrap_ll(sp - s0)) / scale


def finish(s, best, L, ws):
    if best < 0.5 / ws:
        best = 0.0
    return 100.0 * s / L, 100.0 * best


def fused(qv, av, ws):
    """score_fused / k_phred_fallback: the reference's loop"""
    L = len(qv)
    s = seq_sum(0.0, qv)
    if L <= ws:
        m = 100.0 * s / L
        return m, m
    w0 = seq_sum(0.0, qv[:ws]) / ws
    _, b = window_chain(w0, av[ws:], av[:L - ws])
    return finish(s, min(w0, b), L, ws)


def mean_long(qv, gv, tie_any, st):
    """k_phred_mean_long: qv the true table values of the read, gv the grid table's (NaN outside [0, 1))"""
    L = len(qv)
    s, j, small_left = 0.0, 0, 0
    while j < L:
        e = math.frexp(s)[1] - 1 if s > 0.0 else -2000
        big = 10 <= e <= 1000 and small_left == 0
        lattice_ok = big or 6 <= e <= 1000
        hi = min(j + (TILE if big else PIECE), L)
        done = False
        if lattice_ok:
            C, half_ulp = math.ldexp(1.0, e), math.ldexp(1.0, e - 53)
            x = gv[j:hi]
            rq = (C + x) - C                                       # x on the grid of [C, 2C)
            tie = e < 64 and (tie_any >> e) & 1 and bool((np.abs(x - rq) == half_ulp).any())
            d = float(rq.sum())                                    # exact in any order (grid multiples, below 2C), or NaN
            st["tie"] += tie
            st["invalid"] += d != d
            if not tie and s + d < C + C:
                s, done = s + d, True
                st["big" if big else "small"] += 1
        if not done:
            if big:
                st["retry"] += 1
                small_left = TILE // PIECE
                continue
            st["serial"] += 1
            s = seq_sum(s, qv[j:hi])
        if small_left > 0:
            small_left -= 1
        j = hi
    return s


def new_stats():
    return {k: 0 for k in PATHS}


def score_read(qs, T, st):
    """(mean, window quality) of one read as the work-item kernels compute them; adds to the path counts in st"""
    codes = np.frombuffer(bytes(qs), dtype=np.uint8)
    qv, av, ws = T.q[codes], T.a[codes], T.ws
    L = len(codes)
    n_it = items_of(L, ws)
    st["items"] += n_it
    if n_it == 1:
        return fused(qv, av, ws)
    st["segments"] += n_it - 1
    s = mean_long(qv, T.q_grid[codes], T.tie_any, st)
    w0 = seq_sum(0.0, qv[:ws]) / ws
    best, prev_exit = w0, None
    for k in range(n_it - 1):
        P = ws + k * PH_SEG
        entry = w0 if k == 0 else predicted_entry(w0, av, P, ws)
        if k > 0 and np.float64(entry).view(np.int64) != np.float64(prev_exit).view(np.int64):
            st["fallback"] += 1                                    # k_phred_merge: not the chain's value
            return fused(qv, av, ws)
        end = min(P + PH_SEG, L)
        prev_exit, b = window_chain(entry, av[P:end], av[P - ws:end - ws])
        best = min(best, b)
    return finish(s, best, L, ws)


def designed_reads(ws, rng):
    """quality strings aimed at each path of the work-item kernels (the plan, prediction and fallback, the mean chain's
    tiles). rng: numpy Generator. Reads stay at or below 2 * PH_SEG + ws + a few thousand bases (about 200 kbases)."""
    def rq(n, mq=14.0, sd=4.0, lo=1, hi=50):
        return bytearray((np.clip(np.rint(rng.normal(mq, sd, size=n)), lo, hi).astype(np.uint8) + 33).tobytes())

    Ls = max(PH_LONG, ws + PH_SEG) + 1                              # the shortest segmented read
    Lm = ws + 2 * PH_SEG + 3000                                     # three segments
    segmented = Lm <= MAX_DESIGNED
    if not segmented:                                               # longer than PH_LONG, but one fused item
        Ls, Lm = PH_LONG + 1, 30000
    reads = []
    # window quality stays in [0.5, 1) (for ws >= 16): the predictions hold unless a value ties on the grid
    reads.append(("steady", rq(Lm, 25, 2, 15, 45)))
    reads.append(("steady", rq(Ls)))
    # window quality crosses 0.5 and 0.25 before a segment start: the prediction fails, the read falls back
    for k, q in ((1, b"#"), (2, b'"')):
        r = rq(Lm, 20, 2, 12, 40)
        P = ws + k * PH_SEG if segmented else Lm // 2
        lo = max(P - ws - 64, ws + 1) if segmented else P - 300
        r[lo:P - 8] = q * (P - 8 - lo)
        reads.append(("crossing", r))
    # Q3..Q6 (about 0.6) then Q1 (0.21) from the first window on: w falls through 0.5 after about 0.3 ws bases, in a segment
    # that is not the last for every window size up to 100000
    h, n = (ws, ws + 3 * PH_SEG + 3000) if segmented else (300, Lm)
    reads.append(("crossing", rq(h, 4, 1, 3, 6) + b'"' * (n - h)))
    # Q1 / Q2 throughout: w near 0.21 / 0.37, in one binade
    reads.append(("constant", bytearray(b'"' * Lm)))
    reads.append(("constant", bytearray(b"#" * Ls)))
    # a run of '!' first: the sum stays 0, the mean chain walks serially
    r = rq(Lm)
    r[:5000] = b"!" * 5000
    reads.append(("serial", r))
    # high qualities: the sum crosses 2^10 .. 2^17 inside big tiles
    reads.append(("retry", rq(Lm, 40, 3, 30, 60)))
    # the tie bytes: Q44 while the sum is in [512, 1024), Q79 and Q89 in [128, 512)
    reads.append(("tie", bytearray(rng.integers(33 + 40, 33 + 50, size=Ls).astype(np.uint8).tobytes())))
    reads.append(("tie", bytearray(rng.integers(33 + 75, 33 + 93, size=Ls).astype(np.uint8).tobytes())))
    # bytes outside the Phred range: first window, segment edges, inside a big tile, last base
    for bad in (0x20, 200):
        for where in ("first", "edge", "tile", "last"):
            r = rq(Lm)
            if where == "first":
                r[min(ws - 1, 3)] = bad
            elif where == "edge":
                P = ws + PH_SEG if segmented else Lm // 2
                r[P] = r[P - 1] = bad
                if segmented:
                    r[P - ws] = bad                                 # leaves the window as segment 1 starts
            elif where == "tile":
                r[10 * TILE + 777] = bad
            else:
                r[-1] = bad
            reads.append(("invalid", r))
    return [(kind, bytes(r)) for kind, r in reads]


def seam_lengths(ws, max_len=2_000_000):
    """read lengths at the plan's seams: around the window, at PH_LONG, at ws + PH_SEG and around segment edges
    (ws + k PH_SEG + 1 leaves a one-base last segment)"""
    out = [ws - 1, ws, ws + 1, PH_LONG, PH_LONG + 1, ws + PH_SEG, ws + PH_SEG + 1]
    out += [ws + k * PH_SEG + d for k in (1, 2, 3) for d in (-1, 0, 1)]
    return sorted({L for L in out if 0 < L <= max_len})


def reachable_paths(ws):
    """paths the designed reads take at this window size: all of them where a segmented read fits, else the fused one"""
    return PATHS if ws + 2 * PH_SEG + 3000 <= MAX_DESIGNED else ("items",)


def check_designed_paths(ws, kind_stats):
    """each kind of designed read took the path it was designed for (where a segmented read fits)"""
    ks = kind_stats
    if "segments" not in reachable_paths(ws):
        assert all(st["segments"] == 0 for st in ks.values()), ks
        return
    assert ks["constant"]["fallback"] == 0, ks
    # (a one-base window holds the last base's value exactly: its prediction fails only for a value off w0's grid)
    assert ws == 1 or ks["crossing"]["fallback"] > 0, ks
    assert ks["serial"]["serial"] > 5000 // PIECE, ks
    assert ks["retry"]["retry"] > 0, ks
    assert ks["tie"]["tie"] > 0, ks
    assert ks["invalid"]["invalid"] > 0 and ks["invalid"]["fallback"] > 0, ks


def score_designed(reads, T):
    """score_read over (kind, qual) pairs: the results and the path counts per kind"""
    out, ks = [], {}
    for kind, qs in reads:
        out.append(score_read(qs, T, ks.setdefault(kind, new_stats())))
    return out, ks

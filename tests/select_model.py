"""A plain restatement of the last stage, normalisation and the cut (fl_select.cu), exact enough to judge
the device by its own statistics.

Given the global statistics fl_select_summary reports (mean_q, stdev_q, min_z, max_z: the very bits
k_norm_apply used), each row's rescaling is a fixed sequence of IEEE double operations (main.cpp:202-208,
read.cpp:241-264), so `rescale` reproduces it bit for bit wherever the reference's pow() is exact. Given the
final scores, the cut is a stable descending sort plus the prefix walk of main.cpp:247-257, restated by
`expected_cut`. numpy only: no GPU needed."""
import hashlib
import math
from fractions import Fraction

import numpy as np

from tests.numpy_phases import score_keys, target_and_status  # noqa: F401  (re-exported for the tests)

U = 2.0 ** -53                 # unit roundoff of IEEE double
POW_REL = 4 * U                # CUDA's double pow(): <= 2 ulp (CUDA C Programming Guide), and 1 ulp <= 2u relative
SQRT_REL = U                   # sqrt is correctly rounded: <= 0.5 ulp <= u relative


def _pow_rel_err(y):
    """Relative error bound of the device's ref_pow(x, y) for a weight-derived exponent y (fl_select.cu)."""
    if y == 1.0 or y == 0.0:
        return 0.0             # x itself; pow(x, +-0) == 1 exactly (IEEE 754, CUDA)
    if y == 0.5:
        return SQRT_REL        # sqrt(x) for x >= 0; a NaN otherwise, on both sides
    return POW_REL


def _exact_pow(x, y):
    """ref_pow(x, y) where it is exact: (value, mask of the entries where it is)."""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(all="ignore"):
        if y == 1.0:
            return x.copy(), np.ones(x.shape, bool)
        if y == 0.0:
            return np.ones_like(x), np.ones(x.shape, bool)
        if y == 0.5:
            return np.where(x >= 0.0, np.sqrt(np.maximum(x, 0.0)), np.nan), np.ones(x.shape, bool)
        v = np.power(x, y)
        # pow(1, y) == 1 and pow(NaN, y != 0) == NaN exactly; pow(0, y > 0) == 0 exactly
        exact = (x == 1.0) | np.isnan(x) | ((x == 0.0) & (y > 0.0))
        return np.where(x == 1.0, 1.0, v), exact


def length_score(length):
    """read.cpp:241-244 (double)."""
    return 100.0 * (1.0 + (-5000.0 / (np.asarray(length, dtype=np.float64) + 5000.0)))


def rescale(mean, window, length, summary, lw, mw, ww):
    """k_norm_apply + final_score (main.cpp:202-208, read.cpp:241-264) from the device's statistics.

    Returns a dict with `length_score`, `norm_mean`, `norm_window` (float64, exactly the device's operations),
    `final` (np.longdouble: the device's double result wherever every pow() of the row is exact, else the
    same expression with each inexact pow() evaluated in long double and nothing rounded after it but what
    the device also rounds) and `exact` (bool per row: every pow() exact, so `final` must match bit for bit).
    """
    mean = np.asarray(mean, dtype=np.float64)
    window = np.asarray(window, dtype=np.float64)
    f = np.float64
    mq_mean, sd, minz, maxz = f(summary.mean_q), f(summary.stdev_q), f(summary.min_z), f(summary.max_z)
    lw, mw, ww = f(lw), f(mw), f(ww)
    with np.errstate(all="ignore"):
        span = maxz - minz
        ratio = window / mean                                           # main.cpp:203-205
        ratio = np.where(ratio > 1.0, 1.0, ratio)                       # (NaN stays NaN)
        z = (mean - mq_mean) / sd                                       # main.cpp:206
        nm = 100.0 * (z - minz) / span                                  # main.cpp:207: (100 * (z - minz)) / span
        nw = nm * ratio                                                 # main.cpp:208
        ls = length_score(length)
        # read.cpp:249-267, in the device's order
        t = f(1.0) / (lw + mw)
        p1, e1 = _exact_pow(ls, lw)
        p2, e2 = _exact_pow(nm, mw)
        product = p1 * p2
        fs, e3 = _exact_pow(product, t)
        r = nw / nm
        sf = np.where(nm > 0.0, np.where(1.0 < r, 1.0, r), 1.0)         # std::min(r, 1.0): NaN stays NaN
        wf = ww / (lw + mw + ww)
        nwf = f(1.0) - wf
        sf = nwf + (sf * wf)
        final_d = fs * sf
        exact = e1 & e2 & e3
        final = final_d.astype(np.longdouble)
        if not exact.all():
            ld = np.longdouble
            P = np.power(ls.astype(ld), ld(lw)) * np.power(nm.astype(ld), ld(mw))
            fs_ld = np.power(P, ld(t))
            final = np.where(exact, final, fs_ld * sf.astype(ld))
    return dict(length_score=ls, norm_mean=nm, norm_window=nw, final=final, exact=exact)


def final_ulp_bound(lw, mw):
    """How far the device's final score may lie from `rescale`'s long-double value, in ulps of the double.

    The device computes fs = pow(fl(pow(ls, lw) * pow(nm, mw)), t) with t = fl(1 / (lw + mw)), then
    fl(fs * sf), where sf is computed identically on both sides. With a_w the relative error of ref_pow
    for exponent w (0 when exact, u for sqrt, 4u for CUDA's <= 2 ulp pow; u = 2^-53):
      product = P (1 + d),      |d| <= a_lw + a_mw + u            (first order)
      fs      = P^t (1 + d)^t (1 + a_t) = P^t (1 + e),  |e| <= t |d| + a_t
      final   = P^t sf (1 + e) (1 + r),                  |r| <= u
    so |final - P^t sf| <= (t (a_lw + a_mw + u) + a_t + u) |P^t sf|. Since ulp(x) > u |x|, the bound in
    ulps is that coefficient divided by u. One more ulp covers the second-order terms and the long-double
    reference's own rounding (2^-64 relative per operation). Rows whose pow()s are all exact are compared
    bit for bit instead."""
    with np.errstate(all="ignore"):
        t = float(np.float64(1.0) / (np.float64(lw) + np.float64(mw)))
    if not math.isfinite(t):
        return 1               # lw = mw = 0: product = 1 and pow(1, inf) = 1, all exact
    coef = t * (_pow_rel_err(lw) + _pow_rel_err(mw) + U) + _pow_rel_err(t) + U
    return math.ceil(coef / U) + 1


def check_final(got, want, lw, mw, what="final_score"):
    """`got` (float64, the device) against rescale()'s `final` / `exact`: bit-identical where exact, else
    within final_ulp_bound ulps. NaN must be NaN on both sides."""
    got = np.asarray(got, dtype=np.float64)
    fin, exact = want["final"], want["exact"]
    want_d = fin.astype(np.float64)
    nan_g, nan_w = np.isnan(got), np.isnan(want_d)
    bad = np.nonzero(nan_g != nan_w)[0]
    assert bad.size == 0, (what, "NaN", bad[:10], got[bad[:5]], want_d[bad[:5]])
    fin_ok = ~nan_g
    ex = exact & fin_ok
    bad = np.nonzero(got[ex].view(np.uint64) != want_d[ex].view(np.uint64))[0]
    assert bad.size == 0, (what, "bits", np.nonzero(ex)[0][bad[:10]], got[ex][bad[:5]], want_d[ex][bad[:5]])
    inex = ~exact & fin_ok
    if inex.any():
        k = final_ulp_bound(lw, mw)
        err = np.abs(got[inex].astype(np.longdouble) - fin[inex])
        lim = k * np.spacing(np.abs(got[inex])).astype(np.longdouble)
        bad = np.nonzero(err > lim)[0]
        assert bad.size == 0, (what, "ulp bound %d" % k, np.nonzero(inex)[0][bad[:10]], (err[bad[:5]] / lim[bad[:5]] * k))
    return int(inex.sum())


def expected_cut(final, passed, length, target, status):
    """main.cpp:247-257: sort descending by score (stable: equal keys keep row order; NaN first, -0 == +0,
    which is the library's order, fl_select.cu score_key), then keep passed rows while the bases kept so far
    are below the SIGNED target. Returns (passed_final as uint8, keeping)."""
    passed = np.asarray(passed).astype(bool)
    length = np.asarray(length, dtype=np.int64)
    if status != 3:
        return passed.astype(np.uint8), 0
    key = score_keys(final)
    order = np.lexsort((np.arange(key.size), key))          # by key, then by global row
    p = passed[order]
    lens = np.where(p, length[order], 0)
    before = np.cumsum(lens) - lens                          # passed bases ranked strictly before
    keep_sorted = p & (before < int(target))
    out = np.zeros(key.size, dtype=np.uint8)
    out[order] = keep_sorted
    return out, int(length[out.astype(bool)].sum())


# ---------------------------------------------------------------------------------------------
# global statistics (main.cpp:170-196) against the exact values
# ---------------------------------------------------------------------------------------------
RED_THREADS, RED_BLOCKS = 256, 1024          # fl_select.cu's reduction shape


def sum_depth(n, nranks=1):
    """Longest chain of additions in fl_select.cu's sum of n values (k_norm_p1 / k_norm_p2 + the final
    kernel): a thread's strided part of its block's chunk, two 32-lane warp trees, the same over the block
    partials, then the ranks combined one after another."""
    nb = min(max(-(-n // (RED_THREADS * 4)), 1), RED_BLOCKS)
    chunk = -(-n // nb) if n else 0
    return -(-chunk // RED_THREADS) + 10 + -(-nb // RED_THREADS) + 10 + nranks


def _gamma(h):
    return h * U / (1 - h * U)


def exact_moments(x):
    """(sum, mean, variance) of doubles x as exact Fractions (the variance is the population one, /n)."""
    x = np.asarray(x, dtype=np.float64)
    m, e = np.frexp(x)                                          # x = m 2^e, 0.5 <= |m| < 1
    mi = (m * 2.0 ** 53).astype(np.int64)                       # exact
    e = e.astype(np.int64) - 53
    k = int(-e.min()) if x.size else 0
    N = [int(a) << int(b + k) for a, b in zip(mi.tolist(), e.tolist())]
    n = len(N)
    S = sum(N)
    Q = sum(v * v for v in N)
    scale = Fraction(1, 1 << k)
    s = Fraction(S) * scale
    var = Fraction(n * Q - S * S, n * n) * scale * scale
    return s, s / n, var


_moments = {}      # the last row set's exact moments: a sweep re-checks the same rows many times


def check_stats(summary, means, nranks=1):
    """mean_q and stdev_q of fl_select_summary against the exact mean / standard deviation of the rows'
    raw means, within the error bound of fl_select.cu's summation tree; min_q / max_q bit-exact (a NaN
    never updates them, main.cpp:175-178).

    With h the depth of the tree and g = h u / (1 - h u) (Higham, "Accuracy and Stability", 4.2):
      |S' - S| <= g sum|x|,                 mean' = fl(S' / n)  ->  |mean' - mean| <= g sum|x| / n + u |mean'|
      sq' = sum fl(fl(x - mean')^2) = (1 + th) sum (x - mean')^2,  |th| <= g_{h+3},
      sum (x - mean')^2 = n var + n (mean - mean')^2           (exactly, since sum (x - mean) = 0),
      stdev' = fl(sqrt(fl(sq' / n)))  ->  stdev'^2 in [var (1 - g') (1 - u)^3, (var + E^2) (1 + g') (1 + u)^3],
    E being the bound on |mean' - mean|."""
    x = np.asarray(means, dtype=np.float64)
    n = x.size
    fin = x[~np.isnan(x)]
    lo, hi = 100.0, 0.0
    if fin.size:
        lo, hi = min(lo, float(fin.min())), max(hi, float(fin.max()))
    assert summary.min_q == lo and summary.max_q == hi, ((summary.min_q, lo), (summary.max_q, hi))
    if fin.size != n:                   # a NaN mean makes the sums NaN on both sides
        assert math.isnan(summary.mean_q) and math.isnan(summary.stdev_q)
        return
    digest = hashlib.sha1(x.tobytes()).digest()
    if digest not in _moments:
        _moments.clear()
        _moments[digest] = exact_moments(x)
    _, mean, var = _moments[digest]
    h = sum_depth(n, nranks)
    g = _gamma(h)
    E = g * float(np.abs(x).sum()) * (1 + 1e-12) / n + U * abs(summary.mean_q)
    E = E * (1 + 4 * U) + 2.0 ** -1074
    assert abs(Fraction(summary.mean_q) - mean) <= Fraction(E), (summary.mean_q, float(mean), E)
    g2 = _gamma(h + 3)
    sd2 = Fraction(summary.stdev_q) ** 2
    lo2 = var * Fraction((1 - g2) * (1 - U) ** 3 * (1 - 1e-12))
    hi2 = (var + Fraction(E) ** 2) * Fraction((1 + g2) * (1 + U) ** 3 * (1 + 1e-12))
    assert lo2 <= sd2 <= hi2, (summary.stdev_q, math.sqrt(var), math.sqrt(float(lo2)), math.sqrt(float(hi2)))

"""Comparison helpers shared by the GPU parity tests."""
import math
import struct

import numpy as np

from tests import select_model as sm

SCORE_RTOL = 1e-5      # north star: combined float scores within 1e-5 relative
TIE_RTOL = 1e-9        # rows this close at the cut-off are a tie class (SURVEY H1/H2)


def bits(x):
    return struct.pack("<d", float(x))


def same(a, b):
    return bits(a) == bits(b) or (a != a and b != b)


def close(a, b, rtol=SCORE_RTOL):
    if a != a or b != b:
        return a != a and b != b
    if a == b:
        return True
    return abs(a - b) <= rtol * max(abs(a), abs(b))


def check_reads_vs_oracle(rr, sc):
    """rr: Context.read_results(); sc: oracle Scored. Everything per-read is bit-exact."""
    n = len(sc.parents)
    assert len(rr["length"]) == n
    for i, (p, bad, kids) in enumerate(zip(sc.parents, sc.bad, sc.children)):
        assert rr["length"][i] == p.length
        assert same(rr["mean_q"][i], p.mean_q), ("mean", i, rr["mean_q"][i], p.mean_q)
        assert same(rr["window_q"][i], p.window_q), ("window", i, rr["window_q"][i], p.window_q)
        assert same(rr["length_score"][i], p.length_score), ("lscore", i)
        assert rr["passed"][i] == p.passed, ("passed", i)
        assert rr["first_base_in_kmer"][i] == p.first and rr["last_base_in_kmer"][i] == p.last, ("first/last", i)
        assert rr["n_bad"][i] == p.n_bad, ("n_bad", i, rr["n_bad"][i], p.n_bad)
        assert rr["n_child"][i] == p.n_child, ("n_child", i)


def check_rows_vs_oracle(rw, rr, sc, summary):
    """rw: Context.row_results(); sc: finalized oracle Scored."""
    assert len(rw["parent"]) == len(sc.rows), (len(rw["parent"]), len(sc.rows))
    row = 0
    for i, (p, kids) in enumerate(zip(sc.parents, sc.children)):
        assert rr["row_start"][i] == row
        row += max(len(kids), 1)
    for i, r in enumerate(sc.rows):
        assert rw["parent"][i] == r.parent, ("parent", i)
        assert (rw["start"][i], rw["end"][i]) == (r.start, r.end), ("range", i)
        assert same(rw["mean_q"][i], r.mean_q), ("row mean", i, rw["mean_q"][i], r.mean_q)
        assert same(rw["window_q"][i], r.window_q), ("row window", i, rw["window_q"][i], r.window_q)
        assert same(rw["length_score"][i], r.length_score)
        assert rw["passed"][i] == r.passed, ("row passed", i)
        assert close(rw["norm_mean"][i], r.norm_mean), ("norm_mean", i, rw["norm_mean"][i], r.norm_mean)
        assert close(rw["norm_window"][i], r.norm_window), ("norm_window", i)
        assert close(rw["final_score"][i], r.final_score), ("final", i, rw["final_score"][i], r.final_score)
    s, o = summary, sc.summary
    for k in ("min_q", "max_q"):
        assert same(getattr(s, k), getattr(o, k)), k
    assert close(s.mean_q, o.mean_q, 1e-12)
    if o.min_q != o.max_q:
        # (with every mean quality identical the stdev is 0 or a last-bit residue of the summation
        # order -- in the reference too -- and every score is NaN either way, main.cpp:188-207)
        for k in ("stdev_q", "min_z", "max_z"):
            assert close(getattr(s, k), getattr(o, k), 1e-12), k
    assert s.status == o.status
    if o.status:
        assert s.target == o.target and s.passed_bases == o.passed_bases
    check_selection([int(x) for x in rw["passed_final"]], [r.passed_final for r in sc.rows],
                    [r.final_score for r in sc.rows], [r.length for r in sc.rows])
    if o.status == 3:
        assert s.keeping == o.keeping, (s.keeping, o.keeping)


def check_selection(got, want, ref_scores, lengths):
    """Selected IDs must match exactly, except inside the (near-)tie class at the cut-off, where
    the reference's unstable std::sort / last-bit noise decides (SURVEY H1/H2): there the kept
    base total must still agree."""
    diff = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    if not diff:
        return
    sc = [ref_scores[i] for i in diff]
    lo, hi = min(sc), max(sc)
    assert all(not math.isnan(x) for x in sc) or all(math.isnan(x) for x in sc)
    if not math.isnan(lo):
        assert hi - lo <= TIE_RTOL * max(abs(hi), 1e-300), "selection differs outside a tie class: %r" % (diff[:10],)
    assert sum(l for l, g in zip(lengths, got) if g) == sum(l for l, w in zip(lengths, want) if w)


# ---------------------------------------------------------------------------------------------
# exact checks of the last stage against the device's own statistics (tests/select_model.py)
# ---------------------------------------------------------------------------------------------
def _same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return (a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))


def row_lengths(rw):
    return (np.asarray(rw["end"], np.int64) - np.asarray(rw["start"], np.int64))


def check_rescale_exact(rw, summary, params, nranks=1):
    """rw: Context.row_results() (all ranks' rows, in order); summary: the fl_summary of that finalize.
    length_score, norm_mean and norm_window bit-identical to the restatement fed with the summary's
    statistics; final_score too where every pow() is exact, else within select_model.final_ulp_bound;
    min_q / max_q bit-exact, mean_q / stdev_q within the summation tree's bound of the exact values;
    passed and row bases exact."""
    length = row_lengths(rw)
    lw, mw, ww = params.length_weight, params.mean_q_weight, params.window_q_weight
    want = sm.rescale(rw["mean_q"], rw["window_q"], length, summary, lw, mw, ww)
    for k in ("length_score", "norm_mean", "norm_window"):
        ok = _same_bits(rw[k], want[k])
        bad = np.nonzero(~ok)[0]
        assert bad.size == 0, (k, bad[:10], rw[k][bad[:5]], want[k][bad[:5]])
    sm.check_final(rw["final_score"], want, lw, mw)
    sm.check_stats(summary, rw["mean_q"], nranks)
    passed = np.asarray(rw["passed"]).astype(bool)
    assert summary.passed_bases == int(length[passed].sum())
    assert summary.rows_bases == int(length.sum())


def check_selection_exact(rw, summary, params):
    """The device's pass flags, kept bases, target and status must be exactly the stable sort + signed
    prefix walk over its own final scores (NaN first, equal keys in row order: the library's rule)."""
    length = row_lengths(rw)
    passed = np.asarray(rw["passed"]).astype(bool)
    target, status = sm.target_and_status(params, summary.total_bases, int(length[passed].sum()))
    assert (summary.target, summary.status) == (target, status), ((summary.target, summary.status), (target, status))
    want, keeping = sm.expected_cut(rw["final_score"], passed, length, target, status)
    got = np.asarray(rw["passed_final"], np.uint8)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, ("passed_final", bad.size, bad[:10])
    assert summary.keeping == keeping, (summary.keeping, keeping)

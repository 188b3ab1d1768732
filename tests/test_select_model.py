"""CPU tests of tests/select_model.py, the exact restatement of the cut that the GPU tests judge the device by.

The oracle sorts with a stable merge sort, so `expected_cut` applied to the oracle's own final scores must
give the oracle's pass flags, kept bases, target and status EXACTLY: no tie slack. So must the split-phase
numpy restatement (tests/numpy_phases.py) on one and two ranks, applied to its own scores."""
import threading

import numpy as np
import pytest
import torch

from filtlong_b200 import sharding
from oracle import oracle as orc
from tests import select_model as sm
from tests import util
from tests.numpy_phases import NumpyPhases


def _reads(kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "plain":                                  # no ties
        genome = util.rand_seq(rng, 30000)
        return [(s, q) for _, s, q in util.long_reads(rng, genome, 300, max_len=5000)]
    if kind == "dups":                                   # exact duplicates
        genome = util.rand_seq(rng, 30000)
        reads = [(s, q) for _, s, q in util.long_reads(rng, genome, 60, max_len=5000)]
        return [reads[i] for i in rng.permutation(np.repeat(np.arange(60), 5))]
    if kind == "near":
        # one length <= window_size (window == mean, ratio 1) and permutations of one quality multiset: the raw
        # means differ only in summation order, so the scores share every digit but the last one or two
        base = np.frombuffer(util.rand_qual(rng, 200, mean_q=12), np.uint8)
        reads = [(b"A" * 200, rng.permutation(base).tobytes()) for _ in range(400)]
        genome = util.rand_seq(rng, 20000)
        reads += [(s, q) for _, s, q in util.long_reads(rng, genome, 40, max_len=3000)]
        return [reads[i] for i in rng.permutation(len(reads))]
    if kind == "identical":                              # stdev 0: every score NaN, kept in row order
        return [(b"ACGT" * 50, b"5" * 200) for _ in range(30)]
    raise ValueError(kind)


def _oracle(reads, opts):
    p = orc.make_params(**opts)
    return orc.finalize(orc.score(reads, p, None), p), p


def _rows(sc):
    r = sc.rows
    return (np.array([x.final_score for x in r]), np.array([x.passed for x in r], bool),
            np.array([x.length for x in r], np.int64), np.array([x.passed_final for x in r], np.uint8))


def _boundaries(final, passed, length):
    """Inclusive prefix sums of passed bases along the stable descending order."""
    order = np.lexsort((np.arange(final.size), sm.score_keys(final)))
    lens = np.where(passed[order], length[order], 0)
    return np.unique(np.cumsum(lens)[lens > 0])


class _ThreadDist:
    """torch.distributed's all_reduce for ranks that are threads of one process (sum in rank order)."""

    class ReduceOp:
        SUM, MIN, MAX = "sum", "min", "max"

    def __init__(self, world):
        self.world, self.bar, self.slots = world, threading.Barrier(world), [None] * world
        self.local = threading.local()

    def all_reduce(self, t, op="sum"):
        r = self.local.rank
        self.slots[r] = t.clone()
        self.bar.wait()
        st = torch.stack(self.slots)
        red = st.sum(0) if op == "sum" else (st.min(0).values if op == "min" else st.max(0).values)
        self.bar.wait()
        t.copy_(red)


def _numpy_phases(sc, p, world):
    """The split-phase protocol over `world` ranks (threads); returns (final, passed_final, summaries)."""
    rows = sc.rows
    cuts = sharding.shard_by_bases([r.length for r in rows], world)
    out = [None] * world
    dist = _ThreadDist(world) if world > 1 else None
    errors = []

    def run(rank):
        try:
            if dist:
                dist.local.rank = rank
            lo, hi = cuts[rank]
            mine = rows[lo:hi]
            ph = NumpyPhases([r.mean_q for r in mine], [r.window_q for r in mine], [r.length for r in mine],
                             [r.passed for r in mine], p)
            s = sharding.sharded_finalize(ph, dist, sharding.Buffers(torch, "cpu", world), rank, world, sc.total_bases)
            out[rank] = (ph.final, ph.pfinal.astype(np.uint8), s)
        except BaseException as e:          # surfaced below
            errors.append(e)
            if dist:
                dist.bar.abort()

    ts = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    return (np.concatenate([o[0] for o in out]), np.concatenate([o[1] for o in out]), [o[2] for o in out])


def _check(reads, opts, expect_status=None):
    sc, p = _oracle(reads, opts)
    final, passed, length, want = _rows(sc)
    passed_bases = int(length[passed].sum())
    target, status = sm.target_and_status(p, sc.total_bases, passed_bases)
    if p.target_bases_set or p.keep_percent_set:
        assert (target, status) == (sc.summary.target, sc.summary.status)
    if expect_status is not None:
        assert status == expect_status
    got, keeping = sm.expected_cut(final, passed, length, target, status)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]
    assert keeping == sc.summary.keeping
    for world in (1, 2):
        f2, pf2, summaries = _numpy_phases(sc, p, world)
        g2, k2 = sm.expected_cut(f2, passed, length, target, status)
        assert np.array_equal(pf2, g2), (world, np.nonzero(pf2 != g2)[0][:10])
        for s in summaries:
            assert (s.status, s.target, s.keeping) == (status, target, k2), world
    return final, passed, length, status


@pytest.mark.parametrize("kind,opts", [
    ("plain", dict(target_bases=300000)),
    ("plain", dict(keep_percent=55.0, min_length=400)),
    ("dups", dict(keep_percent=45.0)),
    ("dups", dict(target_bases=200000, min_mean_q=80.0)),          # ties mixed with failed rows
    ("dups", dict(keep_percent=60.0, min_length=1500)),
    ("near", dict(keep_percent=50.0)),
    ("near", dict(keep_percent=70.0, window_q_weight=0.0, length_weight=2.0)),
    ("identical", dict(target_bases=1000)),
])
def test_expected_cut_equals_oracle(kind, opts):
    _check(_reads(kind, 5), opts, expect_status=3)


@pytest.mark.parametrize("kind", ["plain", "dups", "near"])
def test_targets_at_prefix_boundaries(kind):
    """Targets at an inclusive prefix boundary of the sorted walk, and one base either side of it."""
    reads = _reads(kind, 9)
    opts = dict(min_mean_q=75.0) if kind == "dups" else {}
    final, passed, length, _ = _check(reads, dict(opts, target_bases=10 ** 5))
    b = _boundaries(final, passed, length)
    rng = np.random.default_rng(3)
    picks = sorted(set([int(b[0]), int(b[1]), int(b[len(b) // 2])] + [int(x) for x in rng.choice(b[:-1], 6)]))
    for B in picks:
        for t in (B - 1, B, B + 1):
            if 0 < t < int(length[passed].sum()):
                _check(reads, dict(opts, target_bases=t), expect_status=3)


def test_targets_near_the_totals():
    reads = _reads("dups", 11)
    sc, _ = _oracle(reads, dict(min_length=2000, target_bases=1))
    passed = int(sum(r.length for r in sc.rows if r.passed))
    total = sc.total_bases
    assert 0 < passed < total
    _check(reads, dict(min_length=2000, target_bases=passed - 1), expect_status=3)
    _check(reads, dict(min_length=2000, target_bases=passed), expect_status=2)
    _check(reads, dict(min_length=2000, target_bases=total - 1), expect_status=2)
    _check(reads, dict(min_length=2000, target_bases=total), expect_status=1)


@pytest.mark.parametrize("opts", [dict(keep_percent=1e-9), dict(target_bases=0), dict(target_bases=-5),
                                  dict(keep_percent=-3.0), dict(target_bases=-(1 << 40), min_length=2000)])
def test_target_at_or_below_zero_keeps_nothing(opts):
    """A target <= 0 (0 from a tiny --keep_percent; negative only through the C ABI) keeps no row, status 3."""
    final, passed, length, status = _check(_reads("dups", 13), opts, expect_status=3)
    got, keeping = sm.expected_cut(final, passed, length, -1, 3)
    assert not got.any() and keeping == 0


def test_score_keys_order():
    x = np.array([np.nan, 3.0, -0.0, 0.0, 1e-300, -1.0, np.inf, 2.5, np.nan, 5e-324])
    k = sm.score_keys(x)
    assert k[0] == k[8] == 0 and k[2] == k[3]
    order = np.lexsort((np.arange(x.size), k))
    assert list(order) == [0, 8, 6, 1, 7, 4, 9, 2, 3, 5]


def test_exact_moments_and_rescale_sanity():
    rng = np.random.default_rng(1)
    x = rng.uniform(0.0, 60.0, size=1000)
    s, mean, var = sm.exact_moments(x)
    assert float(mean) == pytest.approx(np.mean(x), rel=1e-15) and float(var) == pytest.approx(np.var(x), rel=1e-12)
    # t = 1 / (lw + mw); (2, 0.5): 0.4 (4u + u + u) + 4u + u = 7.4u; (1, 3): 0.25 (0 + 4u + u) + 4u + u = 6.25u
    assert (sm.final_ulp_bound(2.0, 0.5), sm.final_ulp_bound(1.0, 3.0), sm.final_ulp_bound(1.0, 1.0)) == (9, 8, 4)

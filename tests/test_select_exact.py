"""The last stage, judged exactly: normalisation, final score and the cut of fl_select.cu against the plain
restatement of tests/select_model.py, fed with the device's own statistics (fl_select_summary) and scores.

Each case pushes its reads once, then sweeps targets and weight sets with fl_ctx_set_params + fl_finalize on
the same context, and with the split-phase fl_norm_* / fl_select_* protocol on 1, 2 and 3 contexts (hand-made
all-reduces, shard cuts inside the tie class at the cut-off). For every combination:
* length_score, norm_mean, norm_window bit-identical; final_score bit-identical where every pow() is exact
  (default weights, (0, 1, 0), (1, 0, 0), lw = mw = 0), else within select_model.final_ulp_bound ulps of the
  long-double value (the derivation from CUDA's <= 2 ulp pow is in that function's docstring);
* min_q / max_q bit-exact, mean_q / stdev_q within the summation tree's bound of the exact values
  (select_model.check_stats), passed and row bases exact;
* pass flags, kept bases, target and status exactly the stable descending sort + signed prefix walk, NaN rows
  first and equal keys in row order (the library's rule; the reference leaves that order unspecified)."""
import time

import numpy as np
import pytest

from filtlong_b200 import api
from tests import parity, util
from tests import select_model as sm

pytestmark = pytest.mark.gpu

EXACT_WEIGHTS = [(1.0, 1.0, 1.0), (0.0, 1.0, 0.0), (1.0, 0.0, 0.0), (0.0, 0.0, 1.0)]
POW_WEIGHTS = [(2.0, 0.5, 3.0), (1.0, 3.0, 1.0)]


def _params(base, w, tgt):
    """tgt: dict, or a tuple of its items (combos are hashable)."""
    return api.make_params(**base, length_weight=w[0], mean_q_weight=w[1], window_q_weight=w[2], **dict(tgt))


def T(**kw):
    return tuple(sorted(kw.items()))


def _rows(ctxs):
    rs = [c.row_results() for c in ctxs]
    return {k: np.concatenate([r[k] for r in rs]) for k in rs[0]}


def _check(rw, summ, p, nranks=1):
    parity.check_rescale_exact(rw, summ, p, nranks)
    parity.check_selection_exact(rw, summ, p)
    if (p.length_weight, p.mean_q_weight) in [w[:2] for w in EXACT_WEIGHTS]:       # every pow() exact: bits compared
        assert sm.rescale(rw["mean_q"], rw["window_q"], parity.row_lengths(rw), summ, *(
            p.length_weight, p.mean_q_weight, p.window_q_weight))["exact"].all()


def _cut_class_shards(rw, summ, bounds):
    """Number of shards holding passed rows of the key class at which the walk crosses the target."""
    if summ.status != 3 or summ.target <= 0:
        return 0
    key = sm.score_keys(rw["final_score"])
    passed = rw["passed"].astype(bool)
    length = parity.row_lengths(rw)
    order = np.lexsort((np.arange(key.size), key))
    lens = np.where(passed[order], length[order], 0)
    incl = np.cumsum(lens)
    j = int(np.searchsorted(incl, summ.target, side="left"))
    if j >= key.size:
        return 0
    rows = np.nonzero(passed & (key == key[order[j]]))[0]
    return len({int(np.searchsorted(bounds, r, side="right")) for r in rows})


class Case:
    """One read set pushed once into a context for fl_finalize and into 2- and 3-context shards."""

    def __init__(self, base, push, worlds=(2, 3)):
        self.base, self.push = base, push
        p = api.make_params(**base)
        self.one = api.Context(p)
        self.total = push(self.one, None)
        self.shards = {}
        for world in worlds:
            ctxs = [api.Context(p) for _ in range(world)]
            for rank, c in enumerate(ctxs):
                push(c, (rank, world))
            self.shards[world] = ctxs

    def close(self):
        for c in [self.one] + [c for cs in self.shards.values() for c in cs]:
            c.close()


def _sweep(case, combos, split):
    """combos: [(weights, target items)]: fl_finalize on the one context; the combos whose index is in `split`
    also through the split-phase protocol on 1, 2 and 3 contexts. Returns (number of final scores checked
    against the ulp bound, most shards holding the key class at the cut)."""
    inexact, straddled = 0, 0
    first = True
    for i, (w, tgt) in enumerate(combos):
        p = _params(case.base, w, tgt)
        case.one.set_params(p)
        summ = case.one.finalize(case.total)
        rw = case.one.row_results()
        _check(rw, summ, p)
        inexact += int((~sm.rescale(rw["mean_q"], rw["window_q"], parity.row_lengths(rw), summ, *w)["exact"]).sum())
        if first:                       # a re-finalized context computes what a fresh one does
            first = False
            fresh = api.Context(p)
            case.push(fresh, None)
            s2 = fresh.finalize(case.total)
            r2 = fresh.row_results()
            fresh.close()
            for k in rw:
                assert np.array_equal(np.asarray(rw[k]).view(np.uint8), np.asarray(r2[k]).view(np.uint8)), k
            assert bytes(summ) == bytes(s2)
        if i not in split:
            continue
        for world, ctxs in [(1, [case.one])] + sorted(case.shards.items()):
            for c in ctxs:
                c.set_params(p)
            sums = util.split_phase_finalize(ctxs, case.total)
            rs = _rows(ctxs)
            for s in sums:
                assert bytes(s) == bytes(sums[0])
            _check(rs, sums[0], p, nranks=world)
            if world > 1:
                counts = np.cumsum([c.counts()[1] for c in ctxs])[:-1]
                straddled = max(straddled, _cut_class_shards(rs, sums[0], counts))
    return inexact, straddled


def _host_push(reads):
    """push(ctx, shard) for a list of (seq, qual): shard = (rank, world) cuts the reads by count into
    contiguous ranges, so that the cuts fall inside interleaved tie classes."""
    def push(ctx, shard):
        lo, hi = 0, len(reads)
        if shard is not None:
            rank, world = shard
            lo, hi = len(reads) * rank // world, len(reads) * (rank + 1) // world
        part = reads[lo:hi]
        if part:
            ctx.push(api.HostBatch([r[0] for r in part], [r[1] for r in part], want_seq=False))
        return sum(len(r[0]) for r in reads)
    return push


def _targets_through(rw, summ_passed, classes=None, limit=60):
    """Targets at the prefix boundaries of the sorted walk among `classes` rows, and one base either side:
    every boundary between two key classes (up to `limit`), and `limit` // 4 inside the classes."""
    key = sm.score_keys(rw["final_score"])
    passed = rw["passed"].astype(bool)
    length = parity.row_lengths(rw)
    order = np.lexsort((np.arange(key.size), key))
    lens = np.where(passed[order], length[order], 0)
    incl = np.cumsum(lens)
    sel = (np.ones(key.size, bool) if classes is None else classes[order]) & (lens > 0)
    ks = key[order]
    last_of_class = np.append(ks[1:] != ks[:-1], True)
    b = np.unique(incl[sel & last_of_class])
    if b.size > limit:
        b = b[np.linspace(0, b.size - 1, limit).astype(int)]
    inner = np.unique(incl[sel & ~last_of_class])
    if inner.size > limit // 4:
        inner = inner[np.linspace(0, inner.size - 1, limit // 4).astype(int)]
    b = np.concatenate([b, inner])
    out = []
    for B in b.tolist():
        out += [t for t in (B - 1, B, B + 1) if 0 < t < summ_passed]
    return sorted(set(out))


def _timed(name, fn):
    t0 = time.time()
    r = fn()
    print("%s: %.2f s" % (name, time.time() - t0))
    return r


def test_near_ties_every_boundary():
    """Thousands of reads of one length <= window_size (window == mean, ratio 1) whose qualities are
    permutations of one multiset: their raw means differ only in summation order, so their keys share every
    digit but the last one or two. The target sweeps every prefix boundary inside that cluster."""
    rng = np.random.default_rng(2024)
    base = np.frombuffer(util.rand_qual(rng, 240, mean_q=13), np.uint8)
    reads = [(b"A" * 240, rng.permutation(base).tobytes()) for _ in range(3000)]
    genome = util.rand_seq(rng, 30000)
    reads += [(s, q) for _, s, q in util.long_reads(rng, genome, 300, max_len=4000)]
    reads = [reads[i] for i in rng.permutation(len(reads))]
    case = Case(dict(), _host_push(reads))
    try:
        p = _params({}, (1.0, 1.0, 1.0), T(target_bases=10 ** 5))
        case.one.set_params(p)
        summ = case.one.finalize(case.total)
        rw = case.one.row_results()
        cluster = parity.row_lengths(rw) == 240
        fs = rw["final_score"][cluster]
        assert np.unique(fs).size > 5 and (fs.max() - fs.min()) < 1e-10 * fs.max()      # near, not exact, ties
        targets = _targets_through(rw, summ.passed_bases, cluster, limit=300)
        assert len(targets) > 100
        combos = [((1.0, 1.0, 1.0), T(target_bases=t)) for t in targets]
        combos += [(w, T(target_bases=targets[len(targets) // 2])) for w in EXACT_WEIGHTS[1:] + POW_WEIGHTS]
        combos += [((1.0, 1.0, 0.0), T(keep_percent=k)) for k in (30.0, 50.0)]
        split = set(range(0, len(combos), 40)) | set(range(len(combos) - 8, len(combos)))
        inexact, straddled = _timed("near ties", lambda: _sweep(case, combos, split))
        assert inexact > 0 and straddled >= 2
    finally:
        case.close()


def test_exact_ties_zero_scores_and_failed_rows():
    """Duplicates that straddle the cut, interleaved with failed rows (min_mean_q, min_length), and reads of
    all '!' (mean 0: a normalised mean and final score of exactly 0) among valid reads."""
    rng = np.random.default_rng(7)
    genome = util.rand_seq(rng, 30000)
    uniq = [(s, q) for _, s, q in util.long_reads(rng, genome, 120, max_len=5000)]
    uniq += [(util.rand_seq(rng, 900), b"!" * 900), (util.rand_seq(rng, 700), b"!" * 700)]
    reads = [uniq[i] for i in rng.permutation(np.repeat(np.arange(len(uniq)), 6))]
    case = Case(dict(min_length=600), _host_push(reads))
    try:
        p = _params(dict(min_length=600), (1.0, 1.0, 1.0), T(target_bases=10 ** 5))
        case.one.set_params(p)
        summ = case.one.finalize(case.total)
        rw = case.one.row_results()
        assert np.any(rw["final_score"] == 0.0) and not rw["passed"].all()
        targets = _targets_through(rw, summ.passed_bases, limit=25)
        # inside the zero-score class (the last of the walk) and across the passed total
        zero_lo = int(parity.row_lengths(rw)[rw["passed"].astype(bool) & (rw["final_score"] != 0.0)].sum())
        targets += [zero_lo + 1, zero_lo + 950, summ.passed_bases - 1, summ.passed_bases, summ.total_bases - 1,
                    summ.total_bases]
        combos = [((1.0, 1.0, 1.0), T(target_bases=t)) for t in targets]
        combos += [(w, T(keep_percent=k)) for w in EXACT_WEIGHTS + POW_WEIGHTS for k in (20.0, 55.0)]
        combos += [((1.0, 1.0, 1.0), T(keep_percent=1e-9)), ((1.0, 1.0, 1.0), T(target_bases=0)),
                   ((1.0, 1.0, 1.0), T(target_bases=-5)), ((2.0, 0.5, 3.0), T(keep_percent=-1.0))]
        split = set(range(0, len(combos), 6)) | set(range(len(combos) - 5, len(combos)))
        inexact, straddled = _timed("exact ties", lambda: _sweep(case, combos, split))
        assert inexact > 0 and straddled >= 2
    finally:
        case.close()
    # ties among rows that fail min_mean_q
    case = Case(dict(min_mean_q=80.0), _host_push(reads), worlds=(3,))
    try:
        combos = [((1.0, 1.0, 1.0), T(keep_percent=k)) for k in (10.0, 35.0, 60.0)]
        _sweep(case, combos, set(range(len(combos))))
    finally:
        case.close()


def test_target_at_or_below_zero_keeps_nothing():
    """A target <= 0 keeps no row (main.cpp:252: 0 < target is false for the first row), with status 3 and
    keeping 0, through fl_finalize and the split-phase calls. The C ABI accepts these parameters."""
    rng = np.random.default_rng(11)
    genome = util.rand_seq(rng, 20000)
    reads = [(s, q) for _, s, q in util.long_reads(rng, genome, 80, max_len=3000)]
    case = Case(dict(), _host_push(reads))
    try:
        combos = [((1.0, 1.0, 1.0), T(target_bases=-5)), ((1.0, 1.0, 1.0), T(target_bases=0)),
                  ((1.0, 1.0, 1.0), T(keep_percent=-3.0)), ((1.0, 1.0, 1.0), T(keep_percent=1e-9)),
                  ((1.0, 1.0, 1.0), T(target_bases=-(1 << 40), keep_percent=50.0))]
        _sweep(case, combos, set(range(len(combos))))
        case.one.set_params(_params({}, (1.0, 1.0, 1.0), T(target_bases=-5)))
        s = case.one.finalize(case.total)
        assert (s.status, s.target, s.keeping) == (3, -5, 0)
        assert not case.one.row_results()["passed_final"].any()
    finally:
        case.close()


def test_kmer_mode_children_and_zero_means():
    """--trim --split: child rows, and rows of mean 0 (no 16-mer of the assembly)."""
    from tests.test_gpu_parity import make_kmer_case
    rng, genome, genome_n, reads = make_kmer_case(61, n_reads=200)
    reads = [(s, None) for s, _ in reads] + [(util.rand_seq(rng, 800), None) for _ in range(10)]
    base = dict(trim=True, split=120)

    def push(ctx, shard):
        ctx.kmers_add([genome_n[:30000], genome_n[30000:]], False)
        ctx.kmers_count()
        lo, hi = 0, len(reads)
        if shard is not None:
            rank, world = shard
            lo, hi = len(reads) * rank // world, len(reads) * (rank + 1) // world
        if hi > lo:
            ctx.push(api.HostBatch([r[0] for r in reads[lo:hi]], None))
        return sum(len(r[0]) for r in reads)

    case = Case(base, push)
    try:
        p = _params(base, (1.0, 1.0, 1.0), T(keep_percent=50.0))
        case.one.set_params(p)
        case.one.finalize(case.total)
        rw = case.one.row_results()
        assert len(rw["parent"]) > len(reads) and np.any(rw["mean_q"] == 0.0)
        combos = [(w, T(keep_percent=k)) for w in EXACT_WEIGHTS + POW_WEIGHTS for k in (25.0, 70.0)]
        combos += [((1.0, 1.0, 1.0), T(target_bases=t)) for t in (1, 40000, 200000)]
        _sweep(case, combos, set(range(0, len(combos), 3)))
    finally:
        case.close()


def test_nan_scores_rank_first_in_row_order():
    """Identical reads: stdev 0, every score NaN, kept in row order. An all-'!' read next to reads with
    invalid quality bytes (negative means): its normalised mean is > 0 and its window/mean ratio 0/0, a NaN
    among finite scores, which the library ranks first as well."""
    seq = b"ACGT" * 100
    same = [(seq, b"5" * 400) for _ in range(40)]
    case = Case(dict(), _host_push(same))
    try:
        combos = [((1.0, 1.0, 1.0), T(target_bases=t)) for t in (1, 400, 401, 4000, 15999)]
        combos += [((2.0, 0.5, 3.0), T(target_bases=2000))]
        _sweep(case, combos, set(range(len(combos))))
        rw = case.one.row_results()
        assert np.isnan(rw["final_score"]).all()
    finally:
        case.close()
    rng = np.random.default_rng(5)
    mixed = [(util.rand_seq(rng, 500), util.rand_qual(rng, 500, mean_q=rng.uniform(6, 25))) for _ in range(60)]
    mixed.insert(17, (b"A" * 400, bytes(rng.integers(1, 33, size=400).astype(np.uint8))))      # negative mean
    for at in (5, 33, 50):
        mixed.insert(at, (b"A" * 300, b"!" * 300))
    case = Case(dict(), _host_push(mixed))
    try:
        case.one.set_params(_params({}, (1.0, 1.0, 1.0), T(keep_percent=50.0)))
        case.one.finalize(case.total)
        rw = case.one.row_results()
        nan = np.isnan(rw["final_score"])
        assert 0 < nan.sum() < nan.size
        combos = [((1.0, 1.0, 1.0), T(target_bases=t)) for t in (1, 300, 301, 600, 601, 900, 901, 5000)]
        combos += [(w, T(keep_percent=40.0)) for w in EXACT_WEIGHTS + POW_WEIGHTS]
        _sweep(case, combos, set(range(len(combos))))
    finally:
        case.close()


def test_scale_past_one_scan_pass():
    """4.4 M rows: more than SCAN_TILE x SCAN_THREADS = 4,194,304, so k_scan_sums carries across
    iterations, and past 1,048,576, where the reductions stop adding blocks. One in seven rows is a copy of
    one read (~630 k rows, interleaved with the rest and on both sides of the shard cut); the target cuts
    that tie class in its middle."""
    import torch
    dev = torch.device("cuda", 0)
    n = 4_400_000
    g = torch.Generator(device=dev)
    g.manual_seed(99)
    length = torch.randint(20, 65, (n,), generator=g, device=dev, dtype=torch.int32)
    qual = torch.randint(33 + 4, 33 + 30, (n, 64), generator=g, device=dev, dtype=torch.uint8)
    tie = torch.arange(n, device=dev) % 7 == 3
    length[tie] = 48
    qual[tie] = torch.randint(33 + 14, 33 + 20, (64,), generator=g, device=dev, dtype=torch.uint8)
    off = torch.arange(n, device=dev, dtype=torch.int64) * 64
    total = int(length.sum())

    def push(ctx, shard):
        lo, hi = 0, n
        if shard is not None:
            rank, world = shard
            lo, hi = n * rank // world, n * (rank + 1) // world
        rel = (off[lo:hi] - off[lo]).contiguous()
        ctx.push_device(api.device_batch(hi - lo, (hi - lo) * 64, rel, length[lo:hi].contiguous(),
                                         qual=qual.view(-1)[lo * 64:]))
        ctx.sync()
        return total

    t0 = time.time()
    case = Case(dict(), push, worlds=(2,))
    try:
        p = _params({}, (1.0, 1.0, 1.0), T(target_bases=10 ** 9))
        case.one.set_params(p)
        summ = case.one.finalize(total)
        rw = case.one.row_results()
        key = sm.score_keys(rw["final_score"])
        tie_np = tie.cpu().numpy()
        tk = key[tie_np][0]
        assert (key[tie_np] == tk).all() and (key == tk).sum() == tie_np.sum() >= 500_000
        better = int(parity.row_lengths(rw)[rw["passed"].astype(bool) & (key < tk)].sum())
        tie_bases = int(tie_np.sum()) * 48
        assert better > 0 and better + tie_bases < summ.passed_bases
        mid = better + tie_bases // 2
        combos = [((1.0, 1.0, 1.0), T(target_bases=t)) for t in (mid, mid + 1, better + 48 * 600_000 + 1)]
        combos += [((2.0, 0.5, 3.0), T(keep_percent=50.0)), ((1.0, 1.0, 1.0), T(target_bases=-1))]
        inexact, straddled = _sweep(case, combos, {0})
        assert straddled == 2
    finally:
        case.close()
    print("scale case: %.2f s" % (time.time() - t0))

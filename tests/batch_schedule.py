"""Seeded batch schedules for tests/test_gpu_batching.py: one read set cut into batches in many ways, each batch pushed
through one of the library's entry points, with result calls between batches.

A schedule is a list of steps:
  ("batch", path, lo, hi)   push reads[lo:hi] through `path` (lo == hi: an empty batch)
  ("observe", what)          call one of OBSERVERS; each finishes a batch whose second half fl_reads_push deferred
The batches of a schedule cover the reads in order, so every schedule must give the results of the one-batch run.

Besides the generator this module holds the read set and, per scoring mode, what the models say about each read (its
children, whether a contaminant set removes it): the generator cuts at those seams, and seams_of() names the seams a
schedule crosses, so the CPU tests can check that every mode's schedules cross all of them."""
import numpy as np

from oracle import oracle as orc
from tests import contam_k_model as km
from tests import qtrim_model as qm
from tests import util

PATHS = ("push", "push_text", "push_bam", "push_device")      # push_text is FASTQ
FASTA = "push_fasta"                                            # push_text with FASTA: k-mer modes only
OBSERVERS = ("counts", "read_results", "row_results", "contam_results", "kmers_count")
SEEDS = (11, 12, 13)
MANY_CHILDREN = 1000
ALLOC_FLOOR = 1024          # the fewest elements DevVec::reserve allocates: arrays grow only past it
SHORT = 16
P_CONTAM = 50.0

# scoring modes: make_params keywords, the k-mer set (an assembly or none), the contaminant set's k (or none)
MODES = {
    "phred": dict(kw=dict(keep_percent=80.0, min_mean_q=9.0)),
    "trimq10_trim_split500": dict(kw=dict(trim_q=10, trim=True, split=500, keep_percent=80.0)),
    "trimq20_split1": dict(kw=dict(trim_q=20, split=1, keep_percent=70.0)),
    "kmer": dict(kw=dict(keep_percent=80.0), kmer=True),
    "kmer_trim_split100": dict(kw=dict(trim=True, split=100, keep_percent=80.0), kmer=True),
    "phred_contam16": dict(kw=dict(keep_percent=80.0, min_mean_q=9.0), contam=16),
    "trimq10_trim_split500_contam16": dict(kw=dict(trim_q=10, trim=True, split=500, keep_percent=80.0), contam=16),
    "kmer_trim_split100_contam16": dict(kw=dict(trim=True, split=100, keep_percent=80.0), kmer=True, contam=16),
    "kmer_trim_split100_contam24": dict(kw=dict(trim=True, split=100, keep_percent=80.0), kmer=True, contam=24),
}


def paths_of(mode):
    return PATHS + (FASTA,) if MODES[mode].get("kmer") else PATHS


# ---- the read set -----------------------------------------------------------------------------------------------------
def read_set(seed=2024):
    """dict(genome, contam, reads): test_contam.make_inputs's reads in upper case (BAM carries no lower case), and,
    kept together so that a batch can hold just them: reads shorter than 16 bases, wholly contaminant reads, a read with no
    children next to two reads of about 600 children each with --split 100 or --split 1 (genome 20-mers between junk runs
    of 110 bases with Phred 2), another next to two reads of about 520 children each with --split 500 too (genome 24-mers
    between junk runs of 500 bases); then reads longer than PH_LONG (24,576 bases), reads of 16 and 17 bases, a read with
    N every 500 bases, a read that --trim cuts into one child, and one empty read. Besides, 1,400 short genome reads (30 to
    400 bases), half after the reads shorter than 16 and half at the end: with them the reads and the rows of every mode
    pass ALLOC_FLOOR, so per-read and per-row arrays must grow, keeping what earlier batches wrote."""
    from tests.test_contam import make_inputs
    genome, contam, base = make_inputs(seed)
    rng = np.random.default_rng(seed + 1)
    cont = contam.upper().replace(b"N", b"A")
    G = len(genome)

    def g(n):
        s = int(rng.integers(0, G - n))
        return genome[s:s + n]

    def q(n, mean_q=20.0, lo=1):
        return util.rand_qual(rng, n, mean_q=mean_q, lo=lo)

    base = [(n, s.upper(), ql) for n, s, ql in base]
    short = [("short_%d" % L, g(L), q(L)) for L in (1, 15, 7, 3, 12)]
    removed = []
    for i, L in enumerate((2500, 4000, 1800, 5200)):                 # exact contaminant sequence: c = 100
        s = 2000 + 3000 * i
        removed.append(("whole_contam_%d" % i, cont[s:s + L], q(L)))
    comb = []
    for i in range(2):
        seq, qual = [], []
        for _ in range(600):
            seq += [g(20), util.rand_seq(rng, 110)]
            qual += [b"I" * 20, b"#" * 110]
        comb.append(("comb_%d" % i, b"".join(seq), b"".join(qual)))
    childless = [("childless_%d" % i, g(4000), b"I" * 4000) for i in range(2)]
    comb_q = []
    for i in range(2):
        seq, qual = [], []
        for _ in range(520):
            seq += [g(24), util.rand_seq(rng, 500)]
            qual += [q(24, mean_q=30, lo=11), b"#" * 500]
        comb_q.append(("comb_q_%d" % i, b"".join(seq), b"".join(qual)))
    one_child = ("one_child", util.rand_seq(rng, 200) + g(2800), b"#" * 200 + b"I" * 2800)
    long = [("long_%d" % L, g(L), q(L, mean_q=15)) for L in (26000, 45000, 30001)]
    edges = [("len_%d" % L, g(L), q(L)) for L in (16, 17)]
    nread = bytearray(g(5000))
    nread[::500] = b"N" * len(nread[::500])
    with_n = ("with_n", bytes(nread), q(5000))
    empty = ("empty", b"", b"")
    cheap = []
    for i in range(1400):
        L = int(rng.integers(30, 401))
        cheap.append(("cheap_%d" % i, g(L), q(L, mean_q=25)))
    reads = (base[:60] + short + cheap[:700] + base[60:120] + removed + base[120:180] + childless[:1] + comb + base[180:200]
             + [empty] + base[200:240] + childless[1:] + comb_q + [one_child] + edges + [with_n] + base[240:300] + long
             + base[300:] + cheap[700:])
    return dict(genome=genome, contam=contam, reads=reads)


# ---- what the models say per read, per mode ---------------------------------------------------------------------------
def assembly_kmers(genome):
    k = orc.Kmers()
    k.add_assembly([genome])
    return k


def contam_percentages(data, k):
    """per read: the percentage of its bases in contaminant k-mers -- the oracle's k-mer-mode mean for 16-mers, the
    numpy model for longer k-mers"""
    seqs = [r[1] for r in data["reads"]]
    if k == 16:
        ck = assembly_kmers(data["contam"])
        sc = orc.score([(s, None) for s in seqs], orc.make_params(), ck)
        return np.array([p.mean_q for p in sc.parents], dtype=np.float64)
    members = km.kmer_set([data["contam"]], k)[0]
    return km.percents(seqs, members, k)


def scored(data, mode, kmers=None):
    """the oracle's finalised Scored of the mode without its contaminant set (--trim_q by tests/qtrim_model.py)"""
    kw = dict(MODES[mode]["kw"])
    Q = kw.pop("trim_q", 0)
    pairs = [(r[1], r[2]) for r in data["reads"]]
    if Q:
        return qm.score_rows(pairs, Q, kw)
    op = orc.make_params(**kw)
    if MODES[mode].get("kmer") and kmers is None:
        kmers = assembly_kmers(data["genome"])
    return orc.finalize(orc.score(pairs, op, kmers if MODES[mode].get("kmer") else None), op)


def attrs(data, mode, sc=None, pct=None):
    """dict(length, n_child, removed) per read: what the schedules cut at"""
    sc = sc if sc is not None else scored(data, mode)
    k = MODES[mode].get("contam")
    n = len(data["reads"])
    if k:
        pct = pct if pct is not None else contam_percentages(data, k)
        removed = pct > P_CONTAM
    else:
        removed = np.zeros(n, dtype=bool)
    return dict(length=np.array([len(r[1]) for r in data["reads"]], dtype=np.int64),
                n_child=np.array([len(c) for c in sc.children], dtype=np.int64), removed=removed)


# ---- the generator ----------------------------------------------------------------------------------------------------
def _longest_run(flags):
    """[a, b) of the longest run of True"""
    best, a = (0, 0), None
    for i, f in enumerate(list(flags) + [False]):
        if f and a is None:
            a = i
        elif not f and a is not None:
            if i - a > best[1] - best[0]:
                best = (a, i)
            a = None
    return best


def _many_children_window(n_child):
    """[a, b): the shortest run of reads with more than MANY_CHILDREN children, preceded by a read with none (or None)"""
    best = None
    for a in range(1, len(n_child)):
        if n_child[a - 1] != 0:
            continue
        s = 0
        for b in range(a, len(n_child)):
            s += n_child[b]
            if s > MANY_CHILDREN:
                if best is None or b + 1 - a < best[1] - best[0]:
                    best = (a, b + 1)
                break
    return best


def _batches(cuts, paths_cycle, length):
    """batch steps over consecutive cuts; a batch holding an empty read goes through push (the other paths take none)"""
    out = []
    for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        p = paths_cycle[i % len(paths_cycle)]
        if b > a and (length[a:b] == 0).any():
            p = "push"
        out.append(("batch", p, int(a), int(b)))
    return out


def _with_observers(rng, steps, rate=0.3, force=()):
    """observers after some batches (the ones in `force` after the first batches, in order)"""
    out, forced = [], list(force)
    for st in steps:
        out.append(st)
        if st[0] != "batch":
            continue
        if forced:
            out.append(("observe", forced.pop(0)))
        elif rng.random() < rate:
            out.append(("observe", OBSERVERS[int(rng.integers(0, len(OBSERVERS)))]))
    return out


def schedules(a, paths):
    """{name: steps} for a mode whose per-read attrs are `a` and whose push paths are `paths` (push first)"""
    length, n_child, removed = a["length"], a["n_child"], a["removed"]
    n = len(length)
    others = [p for p in paths if p != "push"]
    out = {"one_batch": [("batch", "push", 0, n)]}
    out["one_per_batch"] = _batches(np.arange(n + 1), list(paths), length)

    # one read into each staging slot, then a batch past ALLOC_FLOOR into the first slot while the second is held: the
    # slot's arrays, the per-read arrays and the per-row arrays all grow
    big = 2 + ALLOC_FLOOR + 100
    rest = np.unique(np.concatenate(([1, 2, big], np.random.default_rng(1).integers(big + 1, n, 8), [n])))
    out["grow"] = _batches(np.concatenate(([0], rest)), ["push"] * 3 + list(paths), length)

    cycle = ["push"] + others
    steps = [("batch", "push", 0, 0)]                                     # before any read
    for i, st in enumerate(_batches(np.linspace(0, n, 7).astype(int), ["push"], length)):
        steps += [st, ("batch", cycle[i % len(cycle)], st[3], st[3])]     # each deferred push, then an empty batch
    out["empty"] = steps

    seam_cuts = {0, n}
    sa, sb = _longest_run((length < SHORT) & (length > 0))
    seam_cuts |= {sa, sb}
    if removed.any():
        ra, rb = _longest_run(removed)
        seam_cuts |= {ra, rb}
    w = _many_children_window(n_child)
    if w is not None:
        seam_cuts |= {w[0] - 1, w[0], w[1]}
    seam_cuts |= set(int(x) for x in np.random.default_rng(2).integers(1, n, 6))
    out["seams"] = _with_observers(np.random.default_rng(3), _batches(np.array(sorted(seam_cuts)), list(reversed(paths)), length),
                                   force=OBSERVERS)

    alt = []
    for i in range(len(others) * 3):
        alt += ["push", others[i % len(others)]]
    out["alternating"] = _with_observers(np.random.default_rng(4), _batches(np.arange(0, n + 20, 20).clip(max=n), alt, length))

    for s in SEEDS:
        r = np.random.default_rng(s)
        k = int(r.integers(3, 40))
        cuts = np.unique(np.concatenate(([0, n], r.integers(0, n + 1, k))))
        seq = [paths[int(i)] for i in r.integers(0, len(paths), len(cuts))]
        out["random_%d" % s] = _with_observers(r, _batches(cuts, seq, length))
    return out


# ---- what a schedule crosses ------------------------------------------------------------------------------------------
def check_cover(steps, n):
    """the batches cover reads 0..n in order"""
    at = 0
    for st in steps:
        if st[0] == "batch":
            assert st[2] == at and st[3] >= st[2], st
            at = st[3]
    assert at == n


def seams_of(steps, a):
    """the names of the seams `steps` crosses"""
    length, n_child, removed = a["length"], a["n_child"], a["removed"]
    batches = [st for st in steps if st[0] == "batch"]
    full = [b for b in batches if b[3] > b[2]]
    got = set()
    if len(full) == 1 and len(batches) == 1 and full[0][1] == "push":
        got.add("one_batch")
    if len(full) > 1 and all(b[3] - b[2] == 1 for b in full):
        got.add("one_per_batch")
    for x, y, z in zip(full[:-2], full[1:-1], full[2:]):
        if x[1] == y[1] == z[1] == "push" and max(x[3] - x[2], y[3] - y[2]) <= ALLOC_FLOOR < z[3] - z[2]:
            got.add("grow_staging")
    rows = np.concatenate(([0], np.cumsum(np.maximum(n_child, 1))))
    if full and full[0][3] < ALLOC_FLOOR and rows[full[0][3]] < ALLOC_FLOOR and full[-1][3] > ALLOC_FLOOR \
            and rows[full[-1][3]] > ALLOC_FLOOR:
        got.add("grow_arrays")                   # the first batch allocates ALLOC_FLOOR reads and rows; a later one grows them
    for x, y in zip(full[:-1], full[1:]):
        if x[1] == "push" and y[1] != "push":
            got.add("after_deferred:" + y[1])
        kids = sorted((int(n_child[x[2]:x[3]].sum()), int(n_child[y[2]:y[3]].sum())))
        if kids[0] == 0 and kids[1] > MANY_CHILDREN:
            got.add("childless_next_to_many")
    for i, b in enumerate(batches):
        if b[3] == b[2]:
            got.add("empty:" + b[1])
            prev = [x for x in batches[:i] if x[3] > x[2]]
            if b[1] == "push" and prev and prev[-1][1] == "push":
                got.add("empty_push_after_push")
        elif (length[b[2]:b[3]] < SHORT).all():
            got.add("short_only")
        if b[3] > b[2] and removed[b[2]:b[3]].all():
            got.add("all_removed")
    for st in steps:
        if st[0] == "observe":
            got.add("observe:" + st[1])
    return got


def required_seams(a, paths):
    """the seams every mode's schedules must cross between them"""
    need = {"one_batch", "one_per_batch", "grow_staging", "grow_arrays", "short_only", "empty_push_after_push"}
    need |= {"empty:" + p for p in paths} | {"after_deferred:" + p for p in paths if p != "push"}
    need |= {"observe:" + o for o in OBSERVERS}
    if a["removed"].any():
        need.add("all_removed")
    if a["n_child"].sum() > MANY_CHILDREN:
        need.add("childless_next_to_many")
    return need

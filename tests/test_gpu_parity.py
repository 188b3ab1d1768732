"""GPU parity tests: the CUDA path (through the C ABI) against the oracle on the same seeded
inputs. Per-read values (raw mean / window quality, first/last base, bad and child ranges, hard
pass flags) must be bit-identical; normalised / final scores within 1e-5 relative (north star);
selected row IDs identical (modulo the tie class at the cut-off, tests/parity.py). Judged by the
device's own statistics instead, the rescaling and the cut are exact (tests/select_model.py)."""
import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import parity, util

pytestmark = pytest.mark.gpu


def run_both(reads, opts, assembly=None, short=None, cap=4096):
    """the oracle and the device on the same reads; `cap` bounds the oracle's bad ranges and children per read"""
    p, op = api.make_params(**opts), orc.make_params(**opts)
    ok = None
    if assembly or short:
        ok = orc.Kmers()
        if assembly:
            ok.add_assembly(assembly)
        for f in short or []:
            ok.add_short_reads(f)
    sc = orc.finalize(orc.score(reads, op, ok, cap=cap), op)
    ctx, summ = api.score_and_filter(reads, p, assembly=assembly, short_reads=short)
    return ctx, summ, sc, ok


def full_check(ctx, summ, sc):
    rr, rw = ctx.read_results(), ctx.row_results()
    parity.check_reads_vs_oracle(rr, sc)
    parity.check_rows_vs_oracle(rw, rr, sc, summ)
    # and exactly, against the device's own statistics and scores
    parity.check_rescale_exact(rw, summ, ctx.params)
    parity.check_selection_exact(rw, summ, ctx.params)


PHRED_CASES = [
    (1, dict(target_bases=400000)),
    (2, dict(keep_percent=70.0, min_length=500)),
    (3, dict(keep_percent=85.0, min_mean_q=80.0, window_size=100)),
    (4, dict(target_bases=250000, length_weight=2.0, mean_q_weight=0.5, window_q_weight=3.0)),
    (5, dict(min_length=1, keep_percent=90.0, window_size=16)),
    (6, dict(min_length=1, keep_percent=50.0, window_size=1)),
    (7, dict(min_window_q=85.0, max_length=6000, window_size=251)),
    (8, dict(target_bases=10 ** 12)),                 # "not enough reads to reach target"
    (9, dict(target_bases=1000, min_length=100000)),  # "reads already fall below target"
]


@pytest.mark.parametrize("seed,opts", PHRED_CASES)
def test_phred_random(seed, opts):
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, 50000)
    reads = [(s, q) for _, s, q in util.long_reads(rng, genome, 300, max_len=12000)]
    reads.append((b"ACGTACGTAC", b"IIIIIIIIII"))
    reads.append((util.rand_seq(rng, 300), bytes(rng.integers(33, 127, size=300).astype(np.uint8))))
    reads.append((util.rand_seq(rng, 251), b"5" * 251))
    reads.append((util.rand_seq(rng, 250), b"+" * 250))
    reads.append((util.rand_seq(rng, 1), b"#"))
    # bytes outside the printable range exercise the signed-char indexing of read.cpp:271
    reads.append((util.rand_seq(rng, 400), bytes(rng.integers(0, 256, size=400).astype(np.uint8).clip(1, 255))))
    ctx, summ, sc, _ = run_both(reads, opts)
    full_check(ctx, summ, sc)
    ctx.close()


def test_phred_long_reads_and_batches():
    """Reads up to 300 kb, pushed as several batches: results must not depend on batching."""
    rng = np.random.default_rng(42)
    reads = []
    for L in [300000, 150001, 99999, 65536, 4097, 4096, 4095, 17, 16, 15, 2]:
        reads.append((util.rand_seq(rng, L), util.rand_qual(rng, L, mean_q=rng.uniform(6, 28))))
    opts = dict(keep_percent=60.0)
    p, op = api.make_params(**opts), orc.make_params(**opts)
    sc = orc.finalize(orc.score(reads, op, None), op)
    ctx = api.Context(p)
    total = 0
    for i in range(0, len(reads), 4):
        hb = api.HostBatch([r[0] for r in reads[i:i + 4]], [r[1] for r in reads[i:i + 4]], want_seq=False)
        ctx.push(hb)
        total += hb.total_bases
    summ = ctx.finalize(-1)
    assert summ.total_bases == total
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", [250, 16, 1000])
def test_phred_long_read_segment_prediction_and_fallback(ws):
    """Under the work-item kernels (fl_phred.cu), long reads are cut into segments whose entry value of
    the window recurrence is PREDICTED and then verified. These reads make the prediction fail on
    purpose -- the window quality crosses binades (0.99 -> 0.2 -> 0.99), bytes outside the Phred
    range -- so the serial re-score path must produce the reference's bits too. Only ws = 1000 takes
    that path: 250 and 16 are scored by the lattice kernels (k_phred_sum / k_phred_win) and check
    those on the same reads. tests/test_gpu_phred_items.py aims at the work-item path's seams."""
    rng = np.random.default_rng(99)
    reads = []
    reads.append((b"A" * 120000, b"I" * 50000 + b"#" * 30000 + b"I" * 40000))                  # binade crossings
    reads.append((b"A" * 90000, bytes(rng.integers(33, 43, size=90000).astype(np.uint8))))      # w around 0.3-0.6
    reads.append((b"A" * 70000, bytes(rng.integers(1, 256, size=70000).astype(np.uint8))))      # garbage bytes
    reads.append((b"A" * 200000, util.rand_qual(rng, 200000, mean_q=12)))                       # well behaved
    # (no all-'!' read here: with the garbage-byte read above its normalised mean is > 0 while its
    # window/mean ratio is 0/0, i.e. a NaN score among finite ones -- std::sort order is then
    # unspecified in the reference itself; only invalid quality bytes can produce that mix)
    reads.append((b"A" * 60001, b'"' * 60001))                                                  # Q1 everywhere
    reads.append((b"A" * 45000, b"5" * 45000))                                                  # constant quality
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=50.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", [250, 16, 33, 64, 65, 128, 129, 200, 256, 257])
def test_phred_tile_kernel_edges(ws):
    """k_phred_tile (one warp per read, one window length per step): read lengths around multiples of
    the window, every chunk width (window sizes 16..256; 257 takes the work-item kernels), sums that
    cross binades inside a step, qualities whose window stays near 1.0 (Q40+, PacBio '~'), near and
    below 0.5 (rejected -> serial kernel), tie-prone window sizes (200: Q9 ties on the 2^-53 grid),
    all-'!' reads (sum stays 0) and bytes outside the Phred range."""
    rng = np.random.default_rng(1000 + ws)
    reads = []
    for L in [ws + 1, ws + 2, 2 * ws - 1, 2 * ws, 2 * ws + 1, 3 * ws, 5 * ws + 7, 9 * ws - 1, 33 * ws + 3, 1023, 1024, 1025,
              2047, 2048, 2049, 4100, 8200, 16390, 40000]:
        if L > ws:
            reads.append((b"A" * L, util.rand_qual(rng, L, mean_q=rng.uniform(5, 30))))
    reads.append((b"A" * 30000, util.rand_qual(rng, 30000, mean_q=45, sd=3, hi=60)))          # w ~ 0.9999
    reads.append((b"A" * 25000, b"~" * 25000))                                                 # Q93 everywhere
    reads.append((b"A" * 25000, bytes(rng.choice(np.frombuffer(b"~}|{", np.uint8), size=25000))))
    reads.append((b"A" * 20000, util.rand_qual(rng, 20000, mean_q=3.2, sd=1.5)))              # w around 0.5
    reads.append((b"A" * 20000, util.rand_qual(rng, 20000, mean_q=2, sd=1)))                  # w below 0.5
    # (no all-'!' read: next to the invalid-byte reads below its score would be NaN among finite ones)
    reads.append((b"A" * 9000, b"!" * 4000 + b"I" * 5000))                                     # q = 0: the sum stays 0 for 16 steps
    reads.append((b"A" * 12000, b"I" * 6000 + b"!" * 300 + b"I" * 5700))                       # window dips to 0
    reads.append((b"A" * 12000, util.rand_qual(rng, 6000, mean_q=20) + bytes([200]) + util.rand_qual(rng, 5999, mean_q=20)))
    reads.append((b"A" * 12000, util.rand_qual(rng, 6000, mean_q=20) + bytes([12]) + util.rand_qual(rng, 5999, mean_q=20)))
    reads.append((b"A" * 7000, bytes(rng.integers(33 + 40, 33 + 50, size=7000).astype(np.uint8))))   # Q44 ties while the sum is in [512, 1024)
    reads.append((b"A" * 7000, bytes(rng.integers(33 + 75, 33 + 93, size=7000).astype(np.uint8))))   # Q79 / Q89 tie in [128, 512)
    reads.append((b"A" * 150000, util.rand_qual(rng, 150000, mean_q=17)))
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


def test_phred_tile_kernel_many_reads():
    """A few thousand ordinary reads (default window): every warp of the grid takes several reads."""
    rng = np.random.default_rng(77)
    reads = []
    for _ in range(3000):
        L = int(np.clip(rng.lognormal(7.5, 1.0), 20, 60000))
        reads.append((b"A" * L, util.rand_qual(rng, L, mean_q=float(np.clip(rng.normal(14, 4), 5, 30)))))
    ctx, summ, sc, _ = run_both(reads, dict(target_bases=3000000))
    full_check(ctx, summ, sc)
    ctx.close()


def make_kmer_case(seed, n_reads=150, genome_len=60000, max_len=9000):
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, genome_len)
    ga = np.frombuffer(genome, dtype=np.uint8).copy()
    ga[1000:1005] = ord("N")
    ga[20000] = ord("R")
    genome_n = ga.tobytes()
    reads = [(s, q) for _, s, q in util.long_reads(rng, genome, n_reads, max_len=max_len)]
    reads.append((genome[200:215], b"I" * 15))
    reads.append((genome[300:316], b"I" * 16))
    reads.append((util.rand_seq(rng, 700), b"5" * 700))
    reads.append((genome[5000:5400].lower(), b"5" * 400))
    one_n = bytearray(genome[7000:7400]); one_n[200] = ord("N")
    reads.append((bytes(one_n), b"5" * 400))
    reads.append((util.rand_seq(rng, 100) + genome[9000:9400] + util.rand_seq(rng, 30), b"5" * 530))
    reads.append((util.rand_seq(rng, 10) + genome[11000:11200] + util.rand_seq(rng, 60) + genome[12000:12200], b"5" * 470))
    return rng, genome, genome_n, reads


KMER_CASES = [
    (11, dict(keep_percent=90.0)),
    (12, dict(keep_percent=80.0, trim=True, split=100)),
    (13, dict(target_bases=300000, split=30)),
    (14, dict(trim=True)),
    (15, dict(keep_percent=90.0, trim=True, split=250, min_window_q=50.0)),
    (16, dict(min_length=1000, min_mean_q=60.0, window_size=50, split=16)),
    (17, dict(keep_percent=75.0, trim=True, split=1, window_size=20)),
    (18, dict(min_window_q=80.0, split=50, trim=True)),
]


@pytest.mark.parametrize("seed,opts", KMER_CASES)
def test_kmer_assembly_random(seed, opts):
    rng, genome, genome_n, reads = make_kmer_case(seed)
    assembly = [genome_n[:30000], genome_n[30000:], b"ACGT"]
    ctx, summ, sc, ok = run_both(reads, opts, assembly=assembly)
    assert ctx.kmers_count() == len(ok)
    assert np.array_equal(ctx.kmers_export(), ok.dump())
    probe = np.concatenate([ok.dump()[:500], rng.integers(0, 2 ** 32, size=500, dtype=np.uint64).astype(np.uint32)])
    assert list(ctx.kmers_contains(probe)) == [int(k) in ok for k in probe]
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.parametrize("ws", [17, 100, 250, 256, 333, 470, 1000])
def test_kmer_window_kernel_window_sizes_and_long_rows(ws):
    """k_kmer_window on rows from a few bases to > 100 kbases (many 1024-step iterations per warp), clean and
    junk-ridden, for window sizes with different tie binades: every raw mean / window quality bit-exact."""
    rng = np.random.default_rng(1000 + ws)
    genome = util.rand_seq(rng, 300000)
    reads = []
    for i in range(60):
        L = int([50, ws, ws + 1, 2000, 20000, 120000][i % 6] * rng.uniform(0.9, 1.1))
        s = int(rng.integers(0, len(genome) - L))
        seq = util.mutate(rng, genome[s:s + L], [0.0, 0.03, 0.08, 0.12, 0.16][i % 5])
        if i % 4 == 1 and L > 3000:
            cut = int(rng.integers(500, L - 500))
            seq = seq[:cut] + util.rand_seq(rng, int(rng.integers(200, 2500))) + seq[cut:]
        if i % 7 == 3:
            seq = util.rand_seq(rng, int(rng.integers(1, 90))) + seq + util.rand_seq(rng, int(rng.integers(1, 90)))
        reads.append((seq, b"I" * len(seq)))
    for opts in (dict(keep_percent=80.0, window_size=ws), dict(keep_percent=80.0, window_size=ws, trim=True, split=400, min_window_q=40.0)):
        ctx, summ, sc, ok = run_both(reads, opts, assembly=[genome])
        full_check(ctx, summ, sc)
        ctx.close()


@pytest.mark.parametrize("seed,opts", [(21, dict(keep_percent=85.0, trim=True, split=120)),
                                       (22, dict(target_bases=200000))])
def test_kmer_short_reads_random(seed, opts):
    rng, genome, genome_n, reads = make_kmer_case(seed, n_reads=80, genome_len=30000, max_len=5000)
    r1, r2 = util.short_reads(rng, genome, 5000)
    short = [[r[1] for r in r1] + [b"ACGTACG", b"N" * 40], [r[1] for r in r2]]
    ctx, summ, sc, ok = run_both(reads, opts, short=short)
    assert ctx.kmers_count() == len(ok)
    assert np.array_equal(ctx.kmers_export(), ok.dump())
    full_check(ctx, summ, sc)
    ctx.close()


def test_kmer_assembly_then_short_reads():
    """-a and -1/-2 together: assembly k-mers are in the set first and are skipped by the
    multiple-copy rule (kmers.cpp:144-145, main.cpp:55-58)."""
    rng, genome, genome_n, reads = make_kmer_case(31, n_reads=60, genome_len=30000, max_len=4000)
    r1, r2 = util.short_reads(rng, genome, 3000)
    asm = [genome_n[:12000]]
    short = [[r[1] for r in r1], [r[1] for r in r2]]
    ctx, summ, sc, ok = run_both(reads, dict(keep_percent=80.0, trim=True, split=60), assembly=asm, short=short)
    assert np.array_equal(ctx.kmers_export(), ok.dump())
    full_check(ctx, summ, sc)
    ctx.close()


def test_empty_kmer_set_falls_back_to_phred_mode():
    """H5: the mode is decided by kmers.empty(), not by flags (read.cpp:35, main.cpp:103)."""
    rng = np.random.default_rng(5)
    reads = [(util.rand_seq(rng, 500), util.rand_qual(rng, 500)) for _ in range(20)]
    ctx, summ, sc, ok = run_both(reads, dict(keep_percent=50.0), assembly=[b"ACGTACGTACG"])   # < 16 bp: no k-mers
    assert ctx.kmers_count() == 0 and len(ok) == 0
    full_check(ctx, summ, sc)
    ctx.close()


def test_all_identical_reads_give_nan_scores():
    """H3: stdev == 0 -> every normalised quality and final score is NaN; selection then keeps
    rows in file order."""
    seq = b"ACGT" * 100
    reads = [(seq, b"5" * 400) for _ in range(6)]
    ctx, summ, sc, _ = run_both(reads, dict(target_bases=1000))
    rw = ctx.row_results()
    assert all(np.isnan(rw["final_score"]))
    full_check(ctx, summ, sc)
    assert [int(x) for x in rw["passed_final"]] == [1, 1, 1, 0, 0, 0]
    ctx.close()


def test_fasta_without_reference_is_rejected():
    ctx = api.Context(api.make_params(min_length=1))
    hb = api.HostBatch([b"ACGT" * 10], None)
    with pytest.raises(api.FLError) as e:
        ctx.push(hb)
    assert "FASTA input not supported without an external reference" in str(e.value)   # main.cpp:104
    ctx.close()


@pytest.mark.parametrize("mode", ["phred", "assembly", "short"])
def test_against_the_real_reference_harness(mode, tmp_path):
    """Same inputs through the UNMODIFIED reference objects (oracle/_ref/refdump, replayed from tests/golden) and the CUDA path."""
    rng, genome, genome_n, reads = make_kmer_case(77, n_reads=120)
    named = [("r%d" % i, s, q) for i, (s, q) in enumerate(reads)]
    fq = util.write_fastq(tmp_path / "reads.fastq", named)
    opts = dict(keep_percent=80.0) if mode == "phred" else dict(keep_percent=80.0, trim=True, split=90)
    p = api.make_params(**opts)
    cli = orc.params_to_cli(orc.make_params(**opts))
    asm = short = None
    if mode == "assembly":
        fa = util.write_fasta(tmp_path / "asm.fasta", [("c1", genome_n)], width=80)
        cli += ["-a", fa]
        asm = [genome_n]
    elif mode == "short":
        r1, r2 = util.short_reads(rng, genome, 8000)
        cli += ["-1", util.write_fastq(tmp_path / "s1.fastq", r1), "-2", util.write_fastq(tmp_path / "s2.fastq", r2)]
        short = [[r[1] for r in r1], [r[1] for r in r2]]
    ref = orc.run_refdump(cli + [fq])
    ctx, summ = api.score_and_filter(reads, p, assembly=asm, short_reads=short)
    if mode != "phred":
        assert ctx.kmers_count() == ref["n_kmers"]
    rr, rw = ctx.read_results(), ctx.row_results()
    row = 0
    for i, r in enumerate(ref["reads"]):
        assert parity.same(rr["mean_q"][i], r["mean_q"]) and parity.same(rr["window_q"][i], r["window_q"])
        assert (rr["first_base_in_kmer"][i], rr["last_base_in_kmer"][i]) == (r["first"], r["last"])
        assert rr["n_bad"][i] == r["n_bad"] and rr["n_child"][i] == r["n_child"]
        for c in r["children"]:
            assert (rw["start"][row], rw["end"][row]) == (c["start"], c["end"])
            assert parity.same(rw["mean_q"][row], c["mean_q"]) and parity.same(rw["window_q"][row], c["window_q"])
            row += 1
        if not r["children"]:
            row += 1
    assert row == len(ref["rows"]) == len(rw["parent"])
    for i, fr in enumerate(ref["rows"]):
        assert parity.close(rw["final_score"][i], fr["final_score"])
    parity.check_selection([int(x) for x in rw["passed_final"]], [fr["passed_final"] for fr in ref["rows"]],
                           [fr["final_score"] for fr in ref["rows"]], [fr["length"] for fr in ref["rows"]])
    assert summ.keeping == ref["tail"]["keeping"] and summ.target == ref["tail"]["target"]
    ctx.close()


def test_bloom_false_positive_kat_912k_reads():
    """Bloom false-positive path at scale (SURVEY 7.3-H4, Appendix D recipe): 912,000 random 100-bp
    reads passed as -1, with 2,000 reads present three times late in the stream, when the
    reference's Bloom filter is ~65 % full. The unmodified reference (oracle/_ref/refdump, run in
    the build container on exactly this input) logs `25,225 16-mers`; the C restatement gives the
    same. A 16-mer with exactly 3 sightings is in the set only if its FIRST sighting hit a Bloom
    false positive (kmers.cpp:142-166), so a plain ">= 4 copies" rule undercounts by several
    hundred here. Checks the device's closed-form, order-free multiple-copy build."""
    rng = np.random.default_rng(99)
    main = rng.integers(0, 4, size=(900000, 100), dtype=np.int64)
    A = rng.integers(0, 4, size=(2000, 100), dtype=np.int64)
    B = rng.integers(0, 4, size=(2000, 100), dtype=np.int64)
    lut = np.frombuffer(b"ACGT", dtype=np.uint8)
    order = [B, main, A, A, B, A, B]
    seqs = []
    for blk in order:
        arr = lut[blk]
        seqs.extend(bytes(row) for row in arr)
    assert len(seqs) == 912000
    ctx = api.Context(api.make_params(min_length=1))
    ctx.kmers_add(seqs, True)
    n = ctx.kmers_count()
    ctx.kmers_release_build_state()
    ctx.close()
    assert n == 25225


def test_prefilter_flavour_follows_the_set_size_and_all_flavours_agree(monkeypatch):
    """fl_kmers_recount picks the pre-filter's flavour from the number of members (one word per table group of four 16-mers for
    small sets, per pair of neighbours, per 16-mer); forcing each of them (FL_FILTER_KIND), or no filter, must not change a bit."""
    rng, genome, genome_n, reads = make_kmer_case(77, n_reads=120)
    opts = dict(keep_percent=85.0, trim=True, split=120)
    outs = {}
    for tag, env in (("auto", {}), ("group", {"FL_FILTER_KIND": "22"}), ("pair", {"FL_FILTER_KIND": "26"}), ("single", {"FL_FILTER_KIND": "18"}),
                     ("two_bits", {"FL_FILTER_KIND": "2"}), ("none", {"FL_FILTER": "0"}), ("pair_forced_by_size", {"FL_FILTER_G4_MAX": "10"})):
        for k in ("FL_FILTER_KIND", "FL_FILTER", "FL_FILTER_G4_MAX"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ctx = api.Context(api.make_params(**opts))
        ctx.kmers_add([genome_n], False)
        info = ctx.kmers_probe_info()
        hb = api.HostBatch([r[0] for r in reads], [r[1] for r in reads])
        ctx.push(hb)
        summ = ctx.finalize(hb.total_bases)
        rw = ctx.row_results()
        outs[tag] = (info, summ.keeping, {k: v.tobytes() for k, v in rw.items()})
        ctx.close()
    assert outs["auto"][0]["pre_filter"] and outs["auto"][0]["filter_kind"] & 4          # 120 k members: keyed by table group
    assert outs["pair_forced_by_size"][0]["filter_kind"] & 8
    assert not outs["none"][0]["pre_filter"]
    assert all(i["anchored"] for i, _, _ in outs.values())
    ref = outs["none"]
    for tag, o in outs.items():
        assert o[1:] == ref[1:], tag


def test_kmer_results_do_not_depend_on_batching():
    """fl_reads_push double-buffers its staging (copy of batch i+1 overlaps the kernels of batch
    i): pushing the same reads as 1, 3 or 7 batches must give identical rows."""
    rng, genome, genome_n, reads = make_kmer_case(55, n_reads=90)
    opts = dict(keep_percent=80.0, trim=True, split=100)
    outs = []
    for n_batches in (1, 3, 7):
        ctx = api.Context(api.make_params(**opts))
        ctx.kmers_add([genome_n], False)
        step = (len(reads) + n_batches - 1) // n_batches
        total = 0
        for i in range(0, len(reads), step):
            hb = api.HostBatch([r[0] for r in reads[i:i + step]], [r[1] for r in reads[i:i + step]])
            ctx.push(hb)
            total += hb.total_bases
        summ = ctx.finalize(total)
        rw = ctx.row_results()
        outs.append((summ.keeping, summ.target, {k: v.tobytes() for k, v in rw.items()}))
        ctx.close()
    assert outs[0] == outs[1] == outs[2]


@pytest.mark.parametrize("opts,dup", [(dict(keep_percent=60.0), False), (dict(target_bases=250000, min_length=300), False),
                                      (dict(keep_percent=40.0), True)])
def test_sharded_split_phase_protocol_on_device(opts, dup):
    """Two contexts, each holding a contiguous shard of the reads, driven through the split-phase C
    ABI (fl_norm_* / fl_select_*) with hand-made all-reduces: the union of their pass flags must
    equal the single-context fl_finalize and the oracle. `dup` repeats reads so that an exact tie
    class straddles the cut-off AND the shard boundary."""
    from filtlong_b200 import sharding
    rng = np.random.default_rng(123)
    genome = util.rand_seq(rng, 30000)
    reads = [(s, q) for _, s, q in util.long_reads(rng, genome, 200, max_len=5000)]
    if dup:
        reads = reads[:50] * 4
    p, op = api.make_params(**opts), orc.make_params(**opts)
    sc = orc.finalize(orc.score(reads, op, None), op)
    total = sum(len(r[0]) for r in reads)
    cuts = sharding.shard_by_bases([len(r[0]) for r in reads], 2)
    ctxs = []
    for lo, hi in cuts:
        c = api.Context(p)
        c.push(api.HostBatch([r[0] for r in reads[lo:hi]], [r[1] for r in reads[lo:hi]], want_seq=False))
        ctxs.append(c)
    summaries = util.split_phase_finalize(ctxs, total)
    got = []
    rows = [c.row_results() for c in ctxs]
    for r in rows:
        got += [int(x) for x in r["passed_final"]]
    cat = {k: np.concatenate([r[k] for r in rows]) for k in rows[0]}
    parity.check_rescale_exact(cat, summaries[0], p, nranks=2)
    parity.check_selection_exact(cat, summaries[0], p)
    parity.check_selection(got, [r.passed_final for r in sc.rows], [r.final_score for r in sc.rows], [r.length for r in sc.rows])
    for s in summaries:
        assert s.status == sc.summary.status
        if s.status == 3:
            assert (s.keeping, s.target) == (sc.summary.keeping, sc.summary.target)
    # and the one-GPU convenience call agrees
    one, summ = api.score_and_filter(reads, p)
    assert [int(x) for x in one.row_results()["passed_final"]] == got
    for c in ctxs + [one]:
        c.close()

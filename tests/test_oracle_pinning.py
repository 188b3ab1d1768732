"""Pins oracle/filtlong_oracle.c (our C restatement) against the REAL reference.

Runs on CPU. The runs of oracle/_ref (the unmodified reference compiled by oracle/Makefile) are
replayed from tests/golden/reference_runs.json.xz; the reference's own fixtures are the copies under
tests/golden/ref_fixtures. Every double is compared bit-for-bit (the restatement follows the
reference's operation order, so anything else is a restatement bug).
"""
import hashlib
import os
import struct

import numpy as np
import pytest

from oracle import oracle as orc
from tests import util

def bits(x):
    return struct.pack("<d", x)


def same(a, b):
    return bits(a) == bits(b) or (a != a and b != b)


def compare(ref, sc, p, check_rows=True):
    """ref: run_refdump() result; sc: finalized oracle Scored."""
    assert len(ref["reads"]) == len(sc.parents)
    for r, row, bad, kids in zip(ref["reads"], sc.parents, sc.bad, sc.children):
        assert r["length"] == row.length
        assert same(r["mean_q"], row.mean_q), (r["name"], r["mean_q"], row.mean_q)
        assert same(r["window_q"], row.window_q), (r["name"], r["window_q"], row.window_q)
        assert same(r["length_score"], row.length_score)
        assert r["passed"] == row.passed
        assert (r["first"], r["last"]) == (row.first, row.last)
        assert r["bad"] == bad
        assert len(r["children"]) == len(kids)
        for c, k in zip(r["children"], kids):
            assert (c["start"], c["end"]) == (k.start, k.end)
            assert same(c["mean_q"], k.mean_q) and same(c["window_q"], k.window_q)
            assert same(c["length_score"], k.length_score)
            assert c["passed"] == k.passed
            assert c["n_bad"] == 0 and c["n_child"] == 0      # no grandchildren (SURVEY 8a-R7)
            assert k.n_bad == 0 and k.n_child == 0
    g, s = ref["global"], sc.summary
    for key in ("min_q", "max_q", "mean_q", "stdev_q", "min_z", "max_z"):
        assert same(g[key], getattr(s, key)), key
    t = ref["tail"]
    assert t["status"] == s.status
    if s.status:
        assert (t["target"], t["passed_bases"]) == (s.target, s.passed_bases)
    if s.status == 3:
        assert t["keeping"] == s.keeping
    if not check_rows:
        return
    assert len(ref["rows"]) == len(sc.rows)
    flips = []
    for i, (fr, row) in enumerate(zip(ref["rows"], sc.rows)):
        assert same(fr["norm_mean"], row.norm_mean)
        assert same(fr["norm_window"], row.norm_window)
        assert same(fr["final_score"], row.final_score), (fr, row.final_score)
        if fr["passed_final"] != row.passed_final:
            flips.append(i)
    if flips:
        # only legal inside the tie class at the cut-off (unstable std::sort, SURVEY H2)
        scores = {bits(sc.rows[i].final_score) for i in flips}
        assert len(scores) == 1, "selection differs outside a tie class"
        assert sum(r["length"] * r["passed_final"] for r in ref["rows"]) == \
            sum(r.length * r.passed_final for r in sc.rows)


def oracle_kmers(assembly=None, short=None):
    k = orc.Kmers()
    if assembly:
        k.add_assembly([r[1] for r in assembly])
    if short:
        for f in short:
            k.add_short_reads([r[1] for r in f])
    return k


# --------------------------------------------------------------------------------------------
# Bloom constants and hash closed form (SURVEY 8a-K5) against the vendored filter itself
# --------------------------------------------------------------------------------------------
def test_bloom_closed_form():
    keys = [0, 1, 0xDEADBEEF, 0xFFFFFFFF, 0x12345678, 0x80000000]
    ref = orc.run_refdump_bloom(keys)
    L = orc.lib()
    assert ref["k"] == 13 and ref["bits"] == L.orc_bloom_table_bits() == 1917295480
    for k in keys:
        for j in range(13):
            h, idx = ref["hashes"][(k, j)]
            assert L.orc_bloom_hash(k, j) == h
            assert h % ref["bits"] == idx


# --------------------------------------------------------------------------------------------
# The reference's own fixtures (known answers of test/test_sort.py, test_trim.py, test_split.py)
# --------------------------------------------------------------------------------------------
T = util.REF_FIXTURES


# the first 1500 pairs of the reference's test_reference_{1,2}.fastq.gz (all 20,000 are too large to store)
S1, S2 = T + "/test_reference_1_first1500.fastq.gz", T + "/test_reference_2_first1500.fastq.gz"


def test_kmer_counts_match_reference_log_lines():
    # SURVEY section 4 KAT: 199,964 16-mers from the assembly; 23,368 from the stored short-read sample (the
    # reference's log line on exactly these files; 204,833 on all 20,000 pairs)
    asm = util.read_fastx(T + "/test_reference.fasta")
    k = oracle_kmers(assembly=asm)
    assert len(k) == 199964
    k2 = oracle_kmers(short=[util.read_fastx(S1), util.read_fastx(S2)])
    assert len(k2) == 23368


@pytest.mark.parametrize("mode", ["phred", "assembly", "short"])
@pytest.mark.parametrize("opts", [
    dict(min_length=1, keep_percent=90.0),           # BASELINE config 1
    dict(target_bases=10000),
    dict(target_bases=5001),
    dict(target_bases=5000),
    dict(keep_percent=50.0),
    dict(min_mean_q=90.0, min_window_q=80.0),
])
def test_sort_fixture(mode, opts, tmp_path):
    p = orc.make_params(**opts)
    reads = util.read_fastx(T + "/test_sort.fastq")
    cli = orc.params_to_cli(p)
    kmers = None
    if mode == "assembly":
        cli += ["-a", T + "/test_reference.fasta"]
        kmers = oracle_kmers(assembly=util.read_fastx(T + "/test_reference.fasta"))
    elif mode == "short":
        cli += ["-1", S1, "-2", S2]
        kmers = oracle_kmers(short=[util.read_fastx(S1), util.read_fastx(S2)])
    ref = orc.run_refdump(cli + [T + "/test_sort.fastq"])
    sc = orc.finalize(orc.score([(r[1], r[2]) for r in reads], p, kmers), p)
    if kmers is not None:
        assert ref["n_kmers"] == len(kmers)
    compare(ref, sc, p)
    if opts == dict(min_length=1, keep_percent=90.0):
        assert (sc.summary.target, sc.summary.keeping) == (13500, 15000)


@pytest.mark.parametrize("fixture,opts", [
    ("test_trim.fastq", dict(trim=True)),
    ("test_trim.fastq", dict(trim=True, split=20)),
    ("test_split.fastq", dict(split=250)),
    ("test_split.fastq", dict(split=201)),
    ("test_split.fastq", dict(split=200)),
    ("test_split.fastq", dict(split=75)),
    ("test_split.fastq", dict(split=50, trim=True)),
    ("test_split.fastq", dict(split=25, min_window_q=80.0)),     # drifted 79.999999999999986
    ("test_split.fastq", dict(min_length=1, min_window_q=80.0)),
    ("test_split.fastq", dict(min_length=1, min_window_q=79.9999)),
])
def test_trim_split_fixtures(fixture, opts, tmp_path):
    p = orc.make_params(**opts)
    reads = util.read_fastx(T + "/" + fixture)
    kmers = oracle_kmers(assembly=util.read_fastx(T + "/test_reference.fasta"))
    ref = orc.run_refdump(orc.params_to_cli(p) + ["-a", T + "/test_reference.fasta", T + "/" + fixture])
    sc = orc.finalize(orc.score([(r[1], r[2]) for r in reads], p, kmers), p)
    compare(ref, sc, p)


def test_window_drift_golden():
    """SURVEY section 4: window quality 79.999999999999986 (not 80) for test_split_2 under -a."""
    p = orc.make_params(min_length=1)
    reads = util.read_fastx(T + "/test_split.fastq")
    kmers = oracle_kmers(assembly=util.read_fastx(T + "/test_reference.fasta"))
    sc = orc.score([(r[1], r[2]) for r in reads], p, kmers)
    assert sc.parents[1].window_q == float.fromhex("0x1.3ffffffffffffp+6")
    assert sc.parents[2].window_q == float.fromhex("0x1.dfffffffffffbp+5")
    assert sc.parents[3].window_q == float.fromhex("0x1.3ffffffffffecp+4")


# --------------------------------------------------------------------------------------------
# Randomised differential tests (inputs generated here, reference run here)
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,opts", [
    (1, dict(target_bases=200000)),
    (2, dict(keep_percent=70.0, min_length=500)),
    (3, dict(keep_percent=85.0, min_mean_q=80.0, window_size=100)),
    (4, dict(target_bases=150000, length_weight=2.0, mean_q_weight=0.5, window_q_weight=3.0)),
])
def test_random_phred(seed, opts, tmp_path):
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, 50000)
    reads = util.long_reads(rng, genome, 120, max_len=8000)
    reads.append(("tiny", b"ACGTACGTAC", b"IIIIIIIIII"))
    reads.append(("weird_q", util.rand_seq(rng, 300), bytes(rng.integers(33, 127, size=300).astype(np.uint8))))
    fq = util.write_fastq(tmp_path / "r.fastq", reads)
    p = orc.make_params(**opts)
    ref = orc.run_refdump(orc.params_to_cli(p) + [fq])
    sc = orc.finalize(orc.score([(r[1], r[2]) for r in reads], p, None), p)
    compare(ref, sc, p)


@pytest.mark.parametrize("seed,opts,use_short", [
    (11, dict(keep_percent=90.0), False),
    (12, dict(keep_percent=80.0, trim=True, split=100), False),
    (13, dict(target_bases=300000, split=30), False),
    (14, dict(trim=True), False),
    (15, dict(keep_percent=90.0, trim=True, split=250, min_window_q=50.0), True),
    (16, dict(min_length=1000, min_mean_q=60.0, window_size=50, split=16), True),
])
def test_random_kmer(seed, opts, use_short, tmp_path):
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, 60000)
    ga = np.frombuffer(genome, dtype=np.uint8).copy()
    ga[1000:1005] = ord("N")                 # non-ACGT in the reference (kmers.cpp:176-219 asymmetry)
    genome_n = ga.tobytes()
    reads = util.long_reads(rng, genome, 100, max_len=6000)
    reads.append(("short15", genome[200:215], b"I" * 15))
    reads.append(("exact16", genome[300:316], b"I" * 16))
    reads.append(("junk", util.rand_seq(rng, 700), b"5" * 700))
    fq = util.write_fastq(tmp_path / "r.fastq", reads)
    p = orc.make_params(**opts)
    cli = orc.params_to_cli(p)
    if use_short:
        r1, r2 = util.short_reads(rng, genome, 9000)
        f1 = util.write_fastq(tmp_path / "s1.fastq", r1)
        f2 = util.write_fastq(tmp_path / "s2.fastq.gz", r2)
        cli += ["-1", f1, "-2", f2]
        kmers = oracle_kmers(short=[r1, r2])
    else:
        fa = util.write_fasta(tmp_path / "asm.fasta", [("c1", genome_n[:30000]), ("c2", genome_n[30000:]),
                                                      ("tiny", b"ACGT")], width=70)
        cli += ["-a", fa]
        kmers = oracle_kmers(assembly=[("c1", genome_n[:30000]), ("c2", genome_n[30000:])])
    ref = orc.run_refdump(cli + [fq], kmers_out=True)
    assert ref["n_kmers"] == len(kmers)
    assert ref["kmers_sha256"] == hashlib.sha256(kmers.dump().astype("<u4").tobytes()).hexdigest()
    sc = orc.finalize(orc.score([(r[1], r[2]) for r in reads], p, kmers), p)
    compare(ref, sc, p)


def test_harness_selection_matches_reference_cli(tmp_path):
    """The harness restates main.cpp:136-261; pin that restatement on the real CLI's output."""
    rng = np.random.default_rng(21)
    genome = util.rand_seq(rng, 40000)
    reads = util.long_reads(rng, genome, 150, max_len=5000, lower_frac=0, n_frac=0)
    fq = util.write_fastq(tmp_path / "r.fastq", reads)
    fa = util.write_fasta(tmp_path / "a.fasta", [("g", genome)])
    for extra in (["--keep_percent", "60"], ["-a", fa, "--target_bases", "120000", "--trim", "--split", "80"]):
        ref = orc.run_refdump(extra + [fq])
        rc, out, err = orc.run_refcli(extra + [fq])
        assert rc == 0
        cli_names = orc.fastq_names(out)
        # reads2 rows in file order; child rows carry the child name
        kept = [r["name"] for r in ref["rows"] if r["passed_final"]]
        assert cli_names == kept
        if ref["tail"]["status"] == 3:
            assert ("keeping %d bp" % ref["tail"]["keeping"]) in err

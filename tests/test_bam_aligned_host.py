"""Aligned BAM input (--aligned) on the CPU: the aligned walker's index and follower join against the model of
tests/aligned_bam_util.py on a coordinate-sorted file cut into 1 MiB chunks, each new record check on a file built to fail
it next to its valid neighbour, the uncompressed BAM that pass 2 writes for given pass flags, and the option's refusals."""
import os
import subprocess

import numpy as np
import pytest

from tests import aligned_bam_util as au
from tests import bam_util as bu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "filtlong_b200")
HOST_LIB = os.path.join(PKG, "libfiltlong_host.a")
CLI = os.path.join(PKG, "bin", "filtlong")
pytestmark = pytest.mark.skipif(not os.path.exists(HOST_LIB), reason="host library not built")


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("bam_aligned") / "bam_aligned_dump")
    cmd = ["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "bam_aligned_dump.cpp"), HOST_LIB, "-L" + PKG, "-lfiltlong_b200",
           "-lz", "-lpthread", "-Wl,-rpath," + PKG, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def run(dumper, *args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([dumper] + [str(a) for a in args], capture_output=True, env=e)


def parse_index(stdout):
    lines = stdout.decode().splitlines()
    get = lambda tag: [tuple(int(x) for x in l.split()[1:]) for l in lines if l.startswith(tag + " ")]
    return get("C"), get("R"), get("F")


@pytest.fixture(scope="module")
def sorted_file(tmp_path_factory):
    """a seeded coordinate-sorted aligned BAM of over 4 MiB, its records and the BAM file"""
    rng = np.random.default_rng(21)
    recs = au.aligned_reads(rng, bu.random_reads(rng, 2400, hi=2500))
    raw = au.sorted_bam(recs)
    path = tmp_path_factory.mktemp("sorted") / "in.bam"
    path.write_bytes(bu.bgzf(raw))
    return raw, path


@pytest.mark.parametrize("parts", [1, 3])
def test_index_and_join_equal_the_model_across_chunk_cuts(dumper, sorted_file, parts):
    raw, path = sorted_file
    assert len(raw) > 4 << 20
    r = run(dumper, "index", path, env={"FL_CHUNK_MB": "1", "FL_DUMP_PARTS": str(parts)})
    assert r.returncode == 0, r.stderr
    chunks, reads, followers = parse_index(r.stdout)
    want_reads, want_followers = au.model_index(raw)
    assert reads == want_reads
    assert followers == want_followers
    assert r.stderr.decode().strip() == "orphans 0"
    # the file holds what the walker must handle: both strands, unmapped reads, hard-clipped supplementary records,
    # secondary records without SEQ, followers before and after their read, and in another chunk than their read
    recs = bu.records(raw)
    flags = [x["flag"] for x in recs]
    assert any(f & 0x910 == 0x10 for f in flags) and any(f & 0x914 == 0 for f in flags) and any(f & 4 for f in flags)
    assert any(f & 0x800 for f in flags) and any(f & 0x100 and x["len"] == 0 for f, x in zip(flags, recs))
    chunk_of = lambda off: next(k for k, (b, e) in enumerate(chunks) if b <= off < e)
    before = [f for f in followers if f[1] <= f[3]]
    after = [f for f in followers if f[1] > f[3]]
    assert before and after
    assert any(chunk_of(f[0]) != chunk_of(reads[f[3]][0]) for f in followers) and len(chunks) > 4


def test_orphans_are_followers_without_a_read(dumper, tmp_path):
    rng = np.random.default_rng(22)
    recs = au.aligned_reads(rng, bu.random_reads(rng, 300, hi=800))
    raw = au.sorted_bam(recs)
    # a region subset: drop a few reads' read records, keep their followers
    names = [x["name"] for x in bu.records(raw) if not au.is_read(x)][:40:4]
    kept = [x for x in bu.records(raw) if not (au.is_read(x) and x["name"] in names)]
    raw = raw[:bu.header_end(raw)] + b"".join(raw[x["start"]:x["start"] + x["size"]] for x in kept)
    path = tmp_path / "subset.bam"
    path.write_bytes(bu.bgzf(raw))
    r = run(dumper, "index", path)
    assert r.returncode == 0, r.stderr
    _, reads, followers = parse_index(r.stdout)
    want_reads, want_followers = au.model_index(raw)
    assert (reads, followers) == (want_reads, want_followers)
    n_orphans = sum(1 for f in want_followers if f[3] < 0)
    assert n_orphans >= len(set(names)) and r.stderr.decode().strip() == "orphans %d" % n_orphans


GOOD_SEQ, GOOD_QUAL = b"ACGTNACGTA", bytes([20] * 10)


def bad_cases():
    """(case id, the second record when bad, the same record when valid, the message)"""
    rec = lambda flag=0, **kw: bu.record(b"read_2", GOOD_SEQ, GOOD_QUAL, bu.aux_z(b"RG", b"rg1"), flag=flag, ref_id=0, pos=10, **kw)
    return [
        ("hard_clipped_primary", rec(cigar=au.cigar("3H10M")), rec(cigar=au.cigar("3S7M")), "BAM read read_2: its primary record is hard-clipped"),
        ("hard_clipped_reverse_primary", rec(flag=0x10, cigar=au.cigar("10M2H")), rec(flag=0x10, cigar=au.cigar("10M2D")),
         "BAM read read_2: its primary record is hard-clipped"),
        ("query_length_short", rec(cigar=au.cigar("4S5M")), rec(cigar=au.cigar("4S6M")), "the query length of its CIGAR (9) is not its l_seq (10)"),
        ("query_length_long", rec(cigar=au.cigar("5M2I3=1X")), rec(cigar=au.cigar("5M1I3=1X")), "the query length of its CIGAR (11) is not its l_seq (10)"),
        ("no_cigar_when_mapped", rec(), rec(cigar=au.cigar("10M")), "the query length of its CIGAR (0) is not its l_seq (10)"),
        ("primary_without_seq", bu.record(b"read_2", b"", b"", flag=0, ref_id=0, pos=10, cigar=au.cigar("10M")),
         bu.record(b"read_2", GOOD_SEQ, GOOD_QUAL, flag=0, ref_id=0, pos=10, cigar=au.cigar("10M")), "BAM read read_2 has no sequence"),
        ("unmapped_without_seq", bu.record(b"read_2", b"", b""), bu.record(b"read_2", GOOD_SEQ, GOOD_QUAL), "BAM read read_2 has no sequence"),
        ("follower_name_bytes", bu.record(b"read 2", b"", b"", flag=0x100, ref_id=0, pos=10, cigar=au.cigar("10M")),
         bu.record(b"read_2", b"", b"", flag=0x100, ref_id=0, pos=10, cigar=au.cigar("10M")), "outside '!'..'~'"),
    ]


@pytest.mark.parametrize("case,bad,good,message", bad_cases(), ids=[c[0] for c in bad_cases()])
def test_every_new_check_rejects_its_file_and_accepts_the_valid_neighbour(dumper, tmp_path, case, bad, good, message):
    first = bu.record(b"read_1", b"ACGT", bytes([30] * 4), flag=0, cigar=au.cigar("4M"), ref_id=0, pos=5)
    third = bu.record(b"read_3", b"GGGCC", None, bu.aux_f(b"qs", 9.5), flag=0x14)
    sup = bu.record(b"read_1", b"AC", bytes([30] * 2), flag=0x800, cigar=au.cigar("2M2H"), ref_id=0, pos=50)
    hdr = bu.header(refs=[(b"chr1", 1000)])
    (tmp_path / "bad.bam").write_bytes(bu.bgzf(hdr + first + bad + third + sup))
    r = run(dumper, "index", tmp_path / "bad.bam")
    assert r.returncode == 1, (r.returncode, r.stderr)
    err = r.stderr.decode().splitlines()
    assert len(err) == 1 and err[0].startswith("Error: ") and message in err[0], err
    (tmp_path / "good.bam").write_bytes(bu.bgzf(hdr + first + good + third + sup))
    r = run(dumper, "index", tmp_path / "good.bam")
    assert r.returncode == 0, r.stderr
    _, reads, followers = parse_index(r.stdout)
    n_follow = 2 if case == "follower_name_bytes" else 1
    assert len(reads) == 4 - n_follow and len(followers) == n_follow


@pytest.mark.parametrize("parts", [1, 3])
@pytest.mark.parametrize("want", [1, 0])
def test_pass2_stream_equals_the_model(dumper, sorted_file, tmp_path, parts, want):
    raw, path = sorted_file
    rng = np.random.default_rng(23)
    reads = [x for x in bu.records(raw) if au.is_read(x)]
    flags = [int(rng.random() < 0.6) for _ in reads]
    spec = tmp_path / "spec"
    spec.write_text(" ".join(str(f) for f in flags))
    r = run(dumper, "write", path, spec, want, env={"FL_CHUNK_MB": "1", "FL_DUMP_PARTS": str(parts)})
    assert r.returncode == 0, r.stderr
    passed = {x["name"]: f for x, f in zip(reads, flags)}
    assert r.stdout == au.expected_output(raw, passed, bool(want))


def test_pass2_orphans_go_to_failed_only(dumper, tmp_path):
    sup = lambda name, pos: bu.record(name, b"ACG", bytes([9] * 3), flag=0x800, cigar=au.cigar("3M5H"), ref_id=0, pos=pos)
    recs = [sup(b"lost", 1), bu.record(b"a", b"ACGTACGT", bytes([20] * 8), flag=0, cigar=au.cigar("8M"), ref_id=0, pos=2), sup(b"a", 3),
            sup(b"lost", 4), bu.record(b"b", b"ACGTACGT", bytes([20] * 8), flag=0x10, cigar=au.cigar("8M"), ref_id=0, pos=5), sup(b"b", 6)]
    raw = bu.header(refs=[(b"chr1", 100)]) + b"".join(recs)
    (tmp_path / "o.bam").write_bytes(bu.bgzf(raw))
    for flags in ("1 1", "0 0", "1 0"):
        (tmp_path / "spec").write_text(flags)
        passed = dict(zip((b"a", b"b"), (int(x) for x in flags.split())))
        for want in (1, 0):
            r = run(dumper, "write", tmp_path / "o.bam", tmp_path / "spec", want)
            assert r.returncode == 0, r.stderr
            assert r.stdout == au.expected_output(raw, passed, bool(want))


def cli(*args):
    p = subprocess.run([CLI] + [str(a) for a in args], capture_output=True)
    return p.returncode, p.stdout, p.stderr.decode()


@pytest.mark.skipif(not os.path.exists(CLI), reason="CLI not built")
@pytest.mark.parametrize("args", [["--trim"], ["--split", "100"], ["--trim", "--split", "100"], ["--trim_q", "10", "--trim"],
                                  ["--trim", "--keep_mods"]], ids=lambda a: " ".join(a))
def test_aligned_refuses_trim_and_split(tmp_path, args):
    (tmp_path / "a.fasta").write_bytes(b">c\nACGTACGTACGTACGTACGT\n")
    (tmp_path / "x.bam").write_bytes(bu.bgzf(bu.bam_of([(b"r", b"ACGT", bytes([9] * 4), b"")])))
    ref = [] if "--trim_q" in args else ["-a", tmp_path / "a.fasta"]
    rc, out, err = cli("--aligned", *args, *ref, tmp_path / "x.bam")
    assert (rc, out, err) == (1, b"", "Error: --aligned cannot be used with --trim or --split\n")


@pytest.mark.skipif(not os.path.exists(CLI), reason="CLI not built")
def test_help_lists_aligned():
    rc, _, err = cli("--help")
    assert rc == 0 and "--aligned" in err
    assert err.index("other:") < err.index("--aligned") < err.index("--help")

"""Unaligned BAM input on the CPU (filtlong_b200/csrc/host/bam.h, survivors.h): the walker's chunk plan and record index
against the Python reader of tests/bam_util.py, every record check on a file built to fail it next to its valid
neighbour, the uncompressed BAM that pass 2 writes against bam_util.expected_output, and the shared name hash."""
import os
import subprocess

import numpy as np
import pytest

from tests import bam_util as bu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "filtlong_b200")
HOST_LIB = os.path.join(PKG, "libfiltlong_host.a")
pytestmark = pytest.mark.skipif(not os.path.exists(HOST_LIB), reason="host library not built")


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("bam") / "bam_dump")
    cmd = ["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "bam_dump.cpp"), HOST_LIB, "-L" + PKG, "-lfiltlong_b200",
           "-lz", "-lpthread", "-Wl,-rpath," + PKG, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def run(dumper, *args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([dumper] + [str(a) for a in args], capture_output=True, env=e)


def write_bam(path, raw):
    path.write_bytes(bu.bgzf(raw))
    return path


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_index_equals_the_python_reader_with_records_across_chunk_cuts(dumper, tmp_path, seed):
    rng = np.random.default_rng(seed)
    reads = bu.random_reads(rng, 1500, hi=2500, no_qual_every=7 if seed == 2 else 0)
    reads.insert(700, (b"long_one", bu.SEQ_CODES[1:5] * 300000, None, bu.aux_z(b"RG", b"rg1")))     # a chunk of its own at 1 MB
    hdr = bu.header(refs=[(b"chr1", 1000), (b"chr2", 20)] if seed == 3 else ())
    raw = bu.bam_of(reads, hdr)
    assert len(raw) > 4 << 20
    path = write_bam(tmp_path / "in.bam", raw)
    r = run(dumper, "index", path, env={"FL_CHUNK_MB": "1"})
    assert r.returncode == 0, r.stderr
    lines = r.stdout.decode().splitlines()
    chunks = [tuple(int(x) for x in l.split()[1:]) for l in lines if l.startswith("C ")]
    got = [tuple(int(x) for x in l.split()[1:]) for l in lines if l.startswith("R ")]
    recs = bu.records(raw)
    want = [(x["name_off"], x["name_len"], x["seq_off"], x["qual_off"], x["len"], bu.name_hash(x["name"])) for x in recs]
    assert got == want
    # the chunks tile the records, cut at record starts, at most 1 MiB unless one record is larger
    starts = {x["start"]: x["size"] for x in recs}
    assert chunks[0][0] == bu.header_end(raw) and chunks[-1][1] == len(raw) and len(chunks) > 4
    for (b0, e0), (b1, _) in zip(chunks, chunks[1:]):
        assert e0 == b1
    for b, e in chunks:
        assert b in starts
        assert e - b <= 1 << 20 or starts[b] == e - b
    assert any(starts[b] > 1 << 20 for b, _ in chunks)
    # the records of a chunk's last bytes straddle the 1 MiB mark: the cuts are not at fixed positions
    assert any(b % (1 << 20) for b, _ in chunks[1:])


def test_a_header_without_records(dumper, tmp_path):
    raw = bu.header(refs=[(b"c", 5)])
    r = run(dumper, "index", write_bam(tmp_path / "empty.bam", raw))
    assert r.returncode == 0 and r.stdout == b""


GOOD = (b"good_2", b"ACGTNACGTA", bytes([20] * 10), bu.aux_z(b"RG", b"rg1"))


def bad_cases():
    """(case id, the second record's bytes or a whole stream, the message)"""
    rec = lambda **kw: bu.record(GOOD[0], GOOD[1], GOOD[2], GOOD[3], **kw)
    return [
        ("block_size_below_32", bu.struct.pack("<I", 20) + b"\0" * 20, "has block_size < 32"),
        ("record_past_the_end", "truncate", "runs past the end of the file"),
        ("header_text_past_the_end", "header_text", "malformed BAM header"),
        ("reference_entries_past_the_end", "header_refs", "malformed BAM header"),
        ("l_read_name_1", bu.record(b"", GOOD[1], GOOD[2]), "does not end with its NUL"),
        ("no_nul_at_the_name_end", rec(l_read_name=len(GOOD[0])), "does not end with its NUL"),
        ("fields_past_block_size", rec(l_seq=40), "do not fit in its block_size"),
        ("aux_without_nul", bu.record(GOOD[0], GOOD[1], GOOD[2], b"RGZrg1"), "do not parse up to its end"),
        ("aux_unknown_type", bu.record(GOOD[0], GOOD[1], GOOD[2], b"XXq\x01"), "do not parse up to its end"),
        ("aux_array_too_long", bu.record(GOOD[0], GOOD[1], GOOD[2], b"fiBS" + bu.struct.pack("<I", 9) + b"\0\0"), "do not parse up to its end"),
        ("mapped", rec(flag=0), "BAM input must be unaligned: read good_2"),
        ("reverse", rec(flag=4 | 16), "BAM input must be unaligned: read good_2"),
        ("secondary", rec(flag=4 | 0x100), "BAM input must be unaligned: read good_2"),
        ("supplementary", rec(flag=4 | 0x800), "BAM input must be unaligned: read good_2"),
        ("cigar", rec(cigar=(10 << 4,)), "BAM input must be unaligned: read good_2"),
        ("empty_sequence", bu.record(b"good_2", b"", b""), "has no sequence"),
        ("space_in_the_name", bu.record(b"good 2", GOOD[1], GOOD[2]), "outside '!'..'~'"),
        ("nul_in_the_name", bu.record(b"go\0d_2", GOOD[1], GOOD[2]), "outside '!'..'~'"),
    ]


@pytest.mark.parametrize("case,second,message", bad_cases(), ids=[c[0] for c in bad_cases()])
def test_every_check_rejects_its_file_and_accepts_the_valid_neighbour(dumper, tmp_path, case, second, message):
    first = bu.record(b"good_1", b"ACGT", bytes([30] * 4))
    third = bu.record(b"good_3", b"GGGCC", None, bu.aux_f(b"qs", 9.5))
    good = bu.header() + first + bu.record(*GOOD) + third
    if second == "truncate":
        bad = good[:-3]
    elif second == "header_text":
        bad = b"BAM\1" + bu.struct.pack("<I", 10 ** 6) + b"@HD\n"
    elif second == "header_refs":
        bad = bu.header() [:-4] + bu.struct.pack("<I", 3) + bu.struct.pack("<I", 5) + b"chr1\0" + bu.struct.pack("<I", 9)
    else:
        bad = bu.header() + first + second + third
    r = run(dumper, "index", write_bam(tmp_path / "bad.bam", bad))
    assert r.returncode == 1, (r.returncode, r.stderr)
    err = r.stderr.decode().splitlines()
    assert len(err) == 1 and err[0].startswith("Error: ") and message in err[0], err
    r = run(dumper, "index", write_bam(tmp_path / "good.bam", good))
    assert r.returncode == 0, r.stderr
    assert len([l for l in r.stdout.splitlines() if l.startswith(b"R ")]) == 3


def test_the_first_bad_record_is_reported(dumper, tmp_path):
    recs = [bu.record(b"r%d" % i, b"ACGT" * 100, bytes([9] * 400)) for i in range(3000)]
    recs[1800] = bu.record(b"r1800", b"ACGT", bytes([9] * 4), flag=0)
    recs[2500] = bu.record(b"", b"ACGT", bytes([9] * 4))
    r = run(dumper, "index", write_bam(tmp_path / "two_bad.bam", bu.header() + b"".join(recs)), env={"FL_CHUNK_MB": "1"})
    assert r.returncode == 1 and "read r1800" in r.stderr.decode()


def make_results(rng, reads):
    """kept and dropped reads, and reads with children: kept, dropped, of length 0, at odd and even starts"""
    results = []
    for i, (_, seq, _, _) in enumerate(reads):
        L = len(seq)
        if i % 4 < 2 or L < 10:
            results.append((0, [(0, L, int(rng.random() < 0.6))]))
        else:
            cuts = sorted(set(int(c) for c in rng.integers(0, L + 1, size=5)))
            rows = [(a, b, int(rng.random() < 0.7)) for a, b in zip(cuts[:-1], cuts[1:])]
            rows += [(cuts[0], cuts[0], 1), (1, L, 1), (2, L - 1, 1)]          # length 0; odd and even starts and ends
            results.append((len(rows), rows))
    return results


@pytest.mark.parametrize("no_qual_every", [0, 1, 4])
def test_pass2_stream_equals_the_expected_output(dumper, tmp_path, no_qual_every):
    rng = np.random.default_rng(60 + no_qual_every)
    reads = bu.random_reads(rng, 600, hi=4000, no_qual_every=no_qual_every)
    if no_qual_every == 1:
        reads = [(n, s, None, a) for n, s, _, a in reads]
    raw = bu.bam_of(reads)
    path = write_bam(tmp_path / "in.bam", raw)
    results = make_results(rng, reads)
    spec = tmp_path / "spec"
    spec.write_text("".join("%d " % n + " ".join("%d %d %d" % row for row in rows) + "\n" for n, rows in results))
    r = run(dumper, "write", path, spec)
    assert r.returncode == 0, r.stderr
    want = bu.expected_output(raw, results)
    assert r.stdout == want
    # the children carry RG and nothing else of the parent's aux fields
    out = bu.records(r.stdout)
    children = [x for x in out if b"_" in x["name"][5:]]
    assert children and all([t for t, _ in bu.aux_fields(x["aux"])] in ([], [b"RG"]) for x in children)
    assert any(x["aux"] for x in children)


def test_name_hash_is_the_text_paths(dumper):
    names = [b"a", b"read_1", b"read_2", b"0a7c9e3f-1b2d-4c5e-8f90-123456789abc", b"m64011_190830_220126/1/ccs", b"~!" * 60]
    r = run(dumper, "hash", *[n.decode() for n in names])
    assert r.returncode == 0
    assert [int(x) for x in r.stdout.split()] == [bu.name_hash(n) for n in names]

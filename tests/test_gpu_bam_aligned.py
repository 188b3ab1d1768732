"""Aligned BAM input (--aligned) on the GPU: fl_reads_push_bam_strand with mixed strands against fl_reads_push of the
FASTQ equivalent, bit for bit, in Phred and k-mer mode; and the CLI with --aligned on an aligned BAM against the CLI on
its FASTQ equivalent (tests/aligned_bam_util.py): the same log, the kept reads' records byte for byte in input order,
--failed the complement, orphans to --failed only."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from filtlong_b200 import api
from tests import aligned_bam_util as au
from tests import bam_util as bu
from tests import bgzf_util, util

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def strand_reads(rng, mode):
    """(name, seq, qual or None, reverse): every length from 1 to 80 and lengths around multiples of 32, 64 and 1024,
    names of four lengths (SEQ at every byte alignment), IUPAC codes, no-quality records in k-mer mode, mixed strands"""
    lengths = list(range(1, 81)) + [m * k + d for m in (32, 64, 1024) for k in (1, 2, 3, 5) for d in (-1, 0, 1)] + \
        [int(x) for x in rng.integers(100, 6000, size=300)]
    acgt = np.frombuffer(b"ACGT", np.uint8)
    out = []
    for i, L in enumerate(lengths):
        seq = bytearray(acgt[rng.integers(0, 4, size=L)].tobytes())
        if i % 3 == 0:
            for p in rng.integers(0, L, size=max(1, L // 20)):
                seq[p] = bu.SEQ_CODES[int(rng.integers(0, 16))]
        qual = bytes(rng.integers(1, 50, size=L).astype(np.uint8))
        if mode == "kmer" and i % 7 == 3:
            qual = None
        out.append((b"r%d" % i + b"x" * (i % 4), bytes(seq), qual, bool(rng.random() < 0.5) or i == 0))
    return out


def push_both(mode, reads, genome=None, cuts=()):
    """reads through fl_reads_push_bam_strand (their records in chunks cut before the given read indexes; a chunk starts
    at its first record's SEQ, so that a reverse first record's loads reach before the chunk) and their FASTQ
    equivalent through fl_reads_push; returns the two contexts"""
    opts = dict(keep_percent=70.0) if mode == "phred" else dict(keep_percent=70.0, trim=True, split=100)
    a, b = api.Context(api.make_params(**opts)), api.Context(api.make_params(**opts))
    if mode == "kmer":
        for c in (a, b):
            c.kmers_add([genome], False)
            c.kmers_count()
    recs_in = [bu.record(n, au.revcomp(s) if rev else s, None if q is None else (q[::-1] if rev else q), flag=0x10 if rev else 0,
                         cigar=au.cigar("%dM" % len(s)), ref_id=0, pos=i)
               for i, (n, s, q, rev) in enumerate(reads)]
    raw = bu.header(refs=[(b"chr1", 10 ** 7)]) + b"".join(recs_in)
    recs = bu.records(raw)
    bounds = [0] + list(cuts) + [len(recs)]
    for lo, hi in zip(bounds, bounds[1:]):
        part = recs[lo:hi]
        start = part[0]["seq_off"]
        end = part[-1]["start"] + part[-1]["size"]
        a.push_bam(raw[start:end], [r["seq_off"] - start for r in part], [r["qual_off"] - start for r in part], [r["len"] for r in part],
                   reverse=[rev for _, _, _, rev in reads[lo:hi]])
    quals = [None if q is None else bytes(x + 33 for x in q) for _, _, q, _ in reads]
    b.push(api.HostBatch([s for _, s, _, _ in reads], quals if mode == "phred" else None, want_seq=(mode == "kmer")))
    return a, b, recs


def assert_same(a, b):
    assert a.counts() == b.counts()
    s1, s2 = a.finalize(-1), b.finalize(-1)
    assert (s1.status, s1.target, s1.keeping, s1.total_bases) == (s2.status, s2.target, s2.keeping, s2.total_bases)
    for x, y in ((a.read_results(), b.read_results()), (a.row_results(), b.row_results())):
        for k in x:
            assert np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)), k


@pytest.mark.parametrize("mode", ["phred", "kmer"])
def test_push_bam_strand_equals_the_fastq_equivalent(mode):
    rng = np.random.default_rng(31 if mode == "phred" else 32)
    genome = util.rand_seq(rng, 200000)
    reads = strand_reads(rng, mode)
    if mode == "kmer":                       # reads from the genome, on either strand, so that k-mers hit
        for i, (n, s, q, rev) in enumerate(reads):
            if len(s) > 40 and i % 3:
                p = int(rng.integers(0, len(genome) - len(s)))
                g = util.mutate(rng, genome[p:p + len(s)], 0.04)
                reads[i] = (n, au.revcomp(g) if i % 2 else g, q, rev)
    for i in range(2):                       # two reverse reads of 1 Mbase
        L = 1_000_000 + i
        reads.insert(150 + 200 * i, (b"mega_%d" % i, util.rand_seq(rng, L), bytes(rng.integers(1, 50, L).astype(np.uint8)), True))
    cuts = (97, 151, 260)                    # chunks whose first record is reverse, and short
    for c in cuts:
        n, s, q, _ = reads[c]
        L = int(rng.integers(1, 31))
        reads[c] = (n, s[:L], None if q is None else q[:L], True)
    a, b, recs = push_both(mode, reads, genome, cuts)
    assert len({r["seq_off"] % 4 for r in recs}) == 4 and {len(r["seq"]) % 2 for r in recs} == {0, 1}
    assert sum(rev for *_, rev in reads) > 100 and sum(not rev for *_, rev in reads) > 100
    assert_same(a, b)
    a.close(); b.close()


def test_push_bam_strand_without_flags_is_push_bam():
    rng = np.random.default_rng(33)
    reads = [(n, s, q, False) for n, s, q, _ in strand_reads(rng, "phred")]
    a, b, _ = push_both("phred", reads)
    assert_same(a, b)
    a.close(); b.close()


# ---- the CLI ----
def run(cmd, env=None, stdin=None):
    e = dict(os.environ, LC_ALL="C")
    e.pop("LANG", None)
    e.update(env or {})
    p = subprocess.run(cmd, capture_output=True, env=e, stdin=stdin)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("bamaligned")
    rng = np.random.default_rng(41)
    genome = util.rand_seq(rng, 50000)
    reads = []
    for i, (name, seq, qual) in enumerate(util.long_reads(rng, genome, 320, max_len=12000)):
        aux = (bu.aux_z(b"RG", b"rg1") if i % 3 else b"") + bu.aux_f(b"qs", 12.5) + bu.aux_z(b"MM", b"C+m?,0,1;") + \
            bu.aux_b(b"ML", b"C", [200, 10])
        reads.append((name.encode(), seq.upper(), bytes(x - 33 for x in qual), aux))
    raw = au.sorted_bam(au.aligned_reads(rng, reads))
    (d / "in.bam").write_bytes(bu.bgzf(raw))
    (d / "in.fastq").write_bytes(au.to_fastq(raw))
    fa = util.write_fasta(d / "asm.fasta", [("contig_1", genome[:30000]), ("contig_2", genome[30000:])], width=60)
    ct = util.write_fasta(d / "contam.fasta", [("host", genome[5000:15000])])
    return dict(dir=d, raw=raw, fa=fa, ct=ct)


CASES = [
    ["-p", "90"],
    ["-t", "300000"],
    ["-l", "2000", "-p", "80"],
    ["-q", "12", "--min_window_q", "9", "--window_size", "100"],
    ["-a", "FA", "-p", "80"],
    ["--contam", "CT"],
]


def fastq_names(fq):
    return [l[1:].split(b" ")[0] for l in fq.split(b"\n")[0::4] if l]


@pytest.mark.parametrize("case", CASES, ids=lambda c: " ".join(c))
def test_cli_aligned_equals_cli_on_the_fastq_equivalent(case, files):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    d, raw = files["dir"], files["raw"]
    args = [files["fa"] if a == "FA" else (files["ct"] if a == "CT" else a) for a in case]
    rc_f, out_f, err_f = run([CLI] + args + ["--failed", d / "failed.fastq", d / "in.fastq"])
    rc_b, out_b, err_b = run([CLI, "--aligned"] + args + ["--failed", d / "failed.bam", d / "in.bam"])
    assert rc_b == rc_f == 0, err_b[-2000:]
    assert err_b == err_f
    m = bgzf_util.members(out_b)
    assert out_b[m[-1][0]:] == bgzf_util.EOF_MEMBER
    raw_out = gzip.decompress(out_b)
    kept = set(fastq_names(out_f))
    passed = {r["name"]: r["name"] in kept for r in bu.records(raw) if au.is_read(r)}
    assert kept
    assert raw_out == au.expected_output(raw, passed, True)
    assert au.to_fastq(raw_out) == out_f
    failed = gzip.decompress((d / "failed.bam").read_bytes())
    assert failed == au.expected_output(raw, passed, False)
    assert au.to_fastq(failed) == (d / "failed.fastq").read_bytes()
    if case not in (CASES[0], CASES[4]):
        return
    # the same bytes with small chunks and several readers, with --bgzip, from standard input, over two GPUs
    variants = [({"FL_CHUNK_MB": "1", "FL_READERS": "3"}, [], None), ({}, ["--bgzip"], None), ({}, [], "stdin")]
    import torch
    if torch.cuda.device_count() >= 2:
        variants.append(({"FL_CHUNK_MB": "1", "NCCL_DEBUG": "VERSION"}, ["--gpus", "2"], None))
    for env, extra, how in variants:
        if how == "stdin":
            with open(d / "in.bam", "rb") as f:
                rc, out, err = run([CLI, "--aligned"] + extra + args + ["-"], env, stdin=f)
        else:
            rc, out, err = run([CLI, "--aligned"] + extra + args + [d / "in.bam"], env)
        assert rc == 0 and out == out_b, (env, extra, how, err[-2000:])


def test_orphans_go_to_failed_only_and_are_counted(files, tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    raw = files["raw"]
    recs = bu.records(raw)
    lost = sorted({r["name"] for r in recs if not au.is_read(r)})[:6]
    sub = raw[:bu.header_end(raw)] + b"".join(raw[r["start"]:r["start"] + r["size"]] for r in recs if not (au.is_read(r) and r["name"] in lost))
    n_orphans = sum(1 for r in recs if not au.is_read(r) and r["name"] in lost)
    (tmp_path / "sub.bam").write_bytes(bu.bgzf(sub))
    (tmp_path / "sub.fastq").write_bytes(au.to_fastq(sub))
    rc_f, out_f, err_f = run([CLI, "-p", "90", tmp_path / "sub.fastq"])
    rc, out, err = run([CLI, "--aligned", "-p", "90", "--failed", tmp_path / "f.bam", tmp_path / "sub.bam"])
    assert rc == rc_f == 0, err
    line = "  secondary or supplementary records without their read in the input: %d (not written to stdout)\n" % n_orphans
    assert line in err and err.replace(line, "") == err_f
    kept = set(fastq_names(out_f))
    passed = {r["name"]: r["name"] in kept for r in bu.records(sub) if au.is_read(r)}
    assert gzip.decompress(out) == au.expected_output(sub, passed, True)
    failed = gzip.decompress((tmp_path / "f.bam").read_bytes())
    assert failed == au.expected_output(sub, passed, False)
    assert sum(1 for r in bu.records(failed) if r["name"] in lost) == n_orphans


def test_cli_errors(files, tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    raw = files["raw"]
    recs = bu.records(raw)
    first_read = next(r for r in recs if au.is_read(r))
    dup = raw + raw[first_read["start"]:first_read["start"] + first_read["size"]]
    (tmp_path / "dup.bam").write_bytes(bu.bgzf(dup))
    (tmp_path / "dup.fastq").write_bytes(au.to_fastq(dup))
    rc_b, out_b, err_b = run([CLI, "--aligned", "-p", "90", tmp_path / "dup.bam"])
    rc_f, out_f, err_f = run([CLI, "-p", "90", tmp_path / "dup.fastq"])
    assert (rc_b, out_b) == (rc_f, out_f) == (1, b"")
    assert "Error: duplicate read name: " + first_read["name"].decode() in err_b and err_b == err_f
    # without --aligned the file is refused as before; --aligned needs BAM input
    rc, out, err = run([CLI, "-p", "90", files["dir"] / "in.bam"])
    assert rc == 1 and out == b"" and "BAM input must be unaligned: read " in err
    rc, out, err = run([CLI, "--aligned", "-p", "90", files["dir"] / "in.fastq"])
    assert rc == 1 and out == b"" and [l for l in err.splitlines() if l.startswith("Error")] == ["Error: --aligned needs BAM input"]

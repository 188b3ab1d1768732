"""Unaligned BAM input on the GPU: fl_reads_push_bam against the packed-arena path, and the CLI on a BAM file against the
same CLI on the file's FASTQ equivalent (tests/bam_util.py): the same log, the same reads kept, trimmed and split, the
output a BGZF-compressed BAM whose header and whole records are the input's bytes."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from filtlong_b200 import api
from tests import bam_util as bu
from tests import bgzf_util, util

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def push_both(mode, reads, genome=None):
    """the reads through fl_reads_push_bam and through fl_reads_push; returns the two contexts, finalised"""
    opts = dict(keep_percent=70.0) if mode == "phred" else dict(keep_percent=70.0, trim=True, split=100)
    a, b = api.Context(api.make_params(**opts)), api.Context(api.make_params(**opts))
    if mode == "kmer":
        for c in (a, b):
            c.kmers_add([genome], False)
            c.kmers_count()
    raw = bu.bam_of(reads)
    recs = bu.records(raw)
    # two chunks of whole records, the second not starting on a 4-byte boundary of the stream
    cut = recs[len(recs) // 2]["start"]
    for lo, hi, part in ((0, cut, recs[:len(recs) // 2]), (cut, len(raw), recs[len(recs) // 2:])):
        a.push_bam(raw[lo:hi], [r["seq_off"] - lo for r in part], [r["qual_off"] - lo for r in part], [r["len"] for r in part])
    quals = [None if q is None else bytes(x + 33 for x in q) for _, _, q, _ in reads]
    b.push(api.HostBatch([r["seq"] for r in recs], quals if mode == "phred" else None, want_seq=(mode == "kmer")))
    return a, b


@pytest.mark.parametrize("mode", ["phred", "kmer"])
def test_push_bam_equals_the_packed_path(mode):
    rng = np.random.default_rng(5 if mode == "phred" else 6)
    genome = util.rand_seq(rng, 200000)
    reads = bu.random_reads(rng, 1500, lo=1, hi=5000)
    if mode == "kmer":                       # reads from the genome, so that k-mers hit
        reads = [(n, util.mutate(rng, genome[s:s + len(q)], 0.05) if len(q) < 150000 else q, qual, a)
                 for (n, q, qual, a), s in zip(reads, rng.integers(0, 40000, size=len(reads)))]
    for i in range(2):                       # a few 1 Mbase reads
        reads.insert(300 + 600 * i, (b"mega_%d" % i, util.rand_seq(rng, 1_000_000 + i), bytes(rng.integers(1, 50, 1_000_000 + i).astype(np.uint8)),
                                     bu.aux_z(b"RG", b"rg1")))
    assert len({r["seq_off"] % 4 for r in bu.records(bu.bam_of(reads))}) == 4          # SEQ at every byte alignment
    a, b = push_both(mode, reads, genome)
    assert a.counts() == b.counts()
    s1, s2 = a.finalize(-1), b.finalize(-1)
    assert (s1.status, s1.target, s1.keeping, s1.total_bases) == (s2.status, s2.target, s2.keeping, s2.total_bases)
    for x, y in ((a.read_results(), b.read_results()), (a.row_results(), b.row_results())):
        for k in x:
            assert np.array_equal(x[k].view(np.uint8), y[k].view(np.uint8)), k
    a.close(); b.close()


def run(cmd, env=None):
    e = dict(os.environ, LC_ALL="C")
    e.pop("LANG", None)
    e.update(env or {})
    p = subprocess.run(cmd, capture_output=True, env=e)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("bamcli")
    rng = np.random.default_rng(11)
    genome = util.rand_seq(rng, 50000)
    reads = []
    for i, (name, seq, qual) in enumerate(util.long_reads(rng, genome, 300, max_len=12000)):
        aux = (bu.aux_z(b"RG", b"rg1") if i % 3 else b"") + bu.aux_f(b"qs", 12.5) + bu.aux_z(b"MM", b"C+m?,0,1;") + \
            bu.aux_b(b"ML", b"C", [200, 10]) + (bu.aux_b(b"fi", b"S", list(range(len(seq)))) if i % 7 == 0 else b"")
        reads.append((name.encode(), seq.upper(), bytes(x - 33 for x in qual), aux))
    out = {}
    for kind, rs in (("q", reads), ("noq", [(n, s, None, a) for n, s, _, a in reads])):
        raw = bu.bam_of(rs, bu.header(refs=[(b"chr1", 50000)]))
        (d / ("%s.bam" % kind)).write_bytes(bu.bgzf(raw))
        (d / ("%s.fastq" % kind)).write_bytes(bu.to_fastq(raw))
        out[kind] = raw
    fa = util.write_fasta(d / "asm.fasta", [("contig_1", genome[:30000]), ("contig_2", genome[30000:])], width=60)
    return dict(dir=d, raw=out, fa=fa)


CASES = [
    ["-p", "90", "Q"],
    ["-t", "300000", "Q"],
    ["-l", "2000", "-p", "80", "Q"],
    ["-q", "12", "--min_window_q", "9", "--window_size", "100", "Q"],
    ["-a", "FA", "--trim", "--split", "1", "Q"],
    ["-a", "FA", "-p", "80", "--trim", "--split", "16", "Q"],
    ["-a", "FA", "--trim", "--split", "500", "-t", "250000", "Q"],
    ["-a", "FA", "-p", "70", "--trim", "--split", "80", "NOQ"],
]


def check_output(raw_in, out):
    """the BAM output's structure: BGZF members ending with the EOF member, readable by gzip; the input's header; whole
    records byte for byte as in the input; children with only RG of the aux fields"""
    m = bgzf_util.members(out)
    assert out[m[-1][0]:] == bgzf_util.EOF_MEMBER
    raw_out = gzip.decompress(out)
    h = bu.header_end(raw_in)
    assert raw_out[:h] == raw_in[:h]
    by_name = {r["name"]: r for r in bu.records(raw_in)}
    for r in bu.records(raw_out):
        if r["name"] in by_name:
            p = by_name[r["name"]]
            assert raw_out[r["start"]:r["start"] + r["size"]] == raw_in[p["start"]:p["start"] + p["size"]]
        else:
            parent = by_name[r["name"].rsplit(b"_", 1)[0]]
            s, e = (int(x) for x in r["name"].rsplit(b"_", 1)[1].split(b"-"))
            assert raw_out[r["start"]:r["start"] + r["size"]] == bu.child_record(raw_in, parent, s - 1, e)
            assert [t for t, _ in bu.aux_fields(r["aux"])] in ([], [b"RG"])
    return raw_out


@pytest.mark.parametrize("case", CASES, ids=lambda c: " ".join(c))
def test_cli_on_bam_equals_cli_on_its_fastq_equivalent(case, files):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    d = files["dir"]
    kind = "noq" if "NOQ" in case else "q"
    sub = lambda path: [files["fa"] if a == "FA" else (str(path) if a in ("Q", "NOQ") else a) for a in case]
    rc_f, out_f, err_f = run([CLI] + sub(d / ("%s.fastq" % kind)))
    rc_b, out_b, err_b = run([CLI] + sub(d / ("%s.bam" % kind)))
    assert rc_b == rc_f == 0, err_b[-2000:]
    assert err_b == err_f
    raw_out = check_output(files["raw"][kind], out_b)
    assert bu.to_fastq(raw_out) == out_f and len(out_f) > 0
    # the same bytes with small chunks, with --bgzip, and over two GPUs
    variants = [({"FL_CHUNK_MB": "1", "FL_READERS": "3"}, []), ({}, ["--bgzip"]), ({"FL_HOST_PARSER": "1"}, [])]
    import torch
    if torch.cuda.device_count() >= 2:
        variants.append(({"FL_CHUNK_MB": "1", "NCCL_DEBUG": "VERSION"}, ["--gpus", "2"]))
    for env, extra in variants:
        rc, out, err = run([CLI] + extra + sub(d / ("%s.bam" % kind)), env)
        assert rc == 0 and out == out_b, (env, extra, err[-2000:])


def test_cli_on_a_bam_without_records(tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    raw = bu.header(refs=[(b"chr1", 100)])
    (tmp_path / "empty.bam").write_bytes(bu.bgzf(raw))
    (tmp_path / "empty.fastq").write_bytes(b"")
    rc_f, out_f, err_f = run([CLI, "-p", "90", str(tmp_path / "empty.fastq")])
    rc_b, out_b, err_b = run([CLI, "-p", "90", str(tmp_path / "empty.bam")])
    assert rc_b == rc_f == 0 and out_f == b""
    assert err_b == err_f
    assert gzip.decompress(out_b) == raw and out_b.endswith(bgzf_util.EOF_MEMBER)


def error_lines(err):
    lines = err.splitlines()
    return [l for i, l in enumerate(lines) if l.startswith("Error") or (i and lines[i - 1].startswith("Error") and l.startswith("  "))]


def test_cli_errors(tmp_path, files):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    good = [(b"r%d" % i, b"ACGT" * 50, bytes([20] * 200), bu.aux_z(b"RG", b"rg1")) for i in range(20)]
    mixed = good[:5] + [(b"r_fasta", b"ACGT" * 50, None, b"")] + good[5:]
    dup = good + [good[7]]
    noq = [(n, s, None, a) for n, s, _, a in good]
    # checks the FASTQ equivalent's run makes too: the same error lines
    for reads, args, message in ((mixed, ["-p", "90"], "could not parse input reads"),
                                 (noq, ["-p", "90"], "FASTA input not supported without an external reference"),
                                 (dup, ["-p", "90"], "duplicate read name: r7")):
        raw = bu.bam_of(reads)
        (tmp_path / "x.bam").write_bytes(bu.bgzf(raw))
        (tmp_path / "x.fastq").write_bytes(bu.to_fastq(raw))
        rc_b, out_b, err_b = run([CLI] + args + [str(tmp_path / "x.bam")])
        rc_f, out_f, err_f = run([CLI] + args + [str(tmp_path / "x.fastq")])
        assert (rc_b, out_b) == (rc_f, out_f) == (1, b""), err_b
        assert error_lines(err_b) == error_lines(err_f) and message in err_b, (err_b, err_f)
        if reads is mixed:
            assert "  problem occurred at read r_fasta" in error_lines(err_b)
    # checks of the BAM file itself
    (tmp_path / "ok.bam").write_bytes(bu.bgzf(bu.bam_of(good)))
    aligned = bu.bam_of(good[:3] + [(b"mapped", b"ACGT", bytes([9] * 4), b"")])
    aligned = aligned[:-len(bu.record(b"mapped", b"ACGT", bytes([9] * 4)))] + bu.record(b"mapped", b"ACGT", bytes([9] * 4), flag=0)
    (tmp_path / "aligned.bam").write_bytes(bu.bgzf(aligned))
    (tmp_path / "short.bam").write_bytes(bu.bgzf(bu.bam_of(good)[:-7]))
    for path, args, env, message in (
            ("aligned.bam", ["-p", "90"], {}, "BAM input must be unaligned: read mapped"),
            ("short.bam", ["-p", "90"], {}, "runs past the end of the file"),
            ("ok.bam", ["--verbose", "-p", "90"], {}, "--verbose is not supported with BAM input"),
            ("ok.bam", ["-p", "90"], {"FL_GZ_HOST": "1"}, "cannot read BAM input")):
        rc, out, err = run([CLI] + args + [str(tmp_path / path)], env)
        assert rc == 1 and out == b"", (path, err)
        errs = [l for l in err.splitlines() if l.startswith("Error")]
        assert len(errs) == 1 and message in errs[0], (path, err)

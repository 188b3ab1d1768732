"""`filtlong ARGS --failed FILE`: the reads that are not kept go to FILE. For every case the run with `--failed` and the run
without it give the same exit code, byte-identical stdout and the same stderr log; and FILE is the complement of stdout
within the all-rows run (the same input, references, --trim and --split, and `--min_length 1` as the only threshold):
that run's records minus stdout's, byte for byte and in order, with the bases of stdout and FILE adding up to its bases.
BAM is compared record by record after inflating, with the headers equal. The argument errors come before any read is
scored and need no GPU."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from tests import bam_util as bu
from tests import bgzf_util, util
from tests.test_cli import CLI, make_inputs, need_cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT = 300


def run(args, stdin_data=None, env_extra=None, stdout=subprocess.PIPE):
    env = dict(os.environ, LC_ALL="C", **(env_extra or {}))
    env.pop("LANG", None)
    p = subprocess.run([CLI] + list(args), input=stdin_data, stdout=stdout, stderr=subprocess.PIPE, env=env, timeout=TIMEOUT)
    return p.returncode, p.stdout, p.stderr


def gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 1


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("failed_cli")
    crlf, fa, s1, s2, fasta_reads = make_inputs(d)
    rng = np.random.default_rng(23)
    genome = util.rand_seq(rng, 200000)
    reads = util.long_reads(rng, genome, 1500, max_len=12000)
    fq = util.write_fastq(d / "lf.fastq", reads)
    text = open(fq, "rb").read()
    files = dict(FQ=fq, FQGZ=util.write_fastq(d / "lf.fastq.gz", reads), CRLF=crlf, FA=fa, S1=s1, S2=s2, FASTA=fasta_reads)
    files["LFA"] = util.write_fasta(d / "lf_asm.fasta", [("contig_1", genome[:120000]), ("contig_2", genome[120000:])], width=60)
    files["BGZF"] = str(d / "lf.bgzf.fastq.gz")
    open(files["BGZF"], "wb").write(bgzf_util.zlib_bgzf(text) + bgzf_util.EOF_MEMBER)
    recs = [(n.encode(), s.upper(), bytes(x - 33 for x in q), (bu.aux_z(b"RG", b"rg1") if i % 3 else b"") + bu.aux_f(b"qs", 11.5) +
             bu.aux_z(b"MM", b"C+m?,0,1;") + bu.aux_b(b"ML", b"C", [200, 10])) for i, (n, s, q) in enumerate(reads[:800])]
    files["BAM"] = str(d / "reads.bam")
    open(files["BAM"], "wb").write(bu.bgzf(bu.bam_of(recs, bu.header(refs=[(b"chr1", 200000)]))))
    return files


def unpack(data, compressed, bam):
    """(BAM header or b"", [(record bytes, bases)]) of an output"""
    if compressed:
        assert data.endswith(bgzf_util.EOF_MEMBER)
        data = gzip.decompress(data)
    if bam:
        return data[:bu.header_end(data)], [(data[r["start"]:r["start"] + r["size"]], r["len"]) for r in bu.records(data)]
    if not data:
        return b"", []
    assert data.endswith(b"\n")
    lines = data[:-1].split(b"\n")
    k = 4 if data[:1] == b"@" else 2
    assert len(lines) % k == 0
    return b"", [(b"\n".join(lines[i:i + k]) + b"\n", len(lines[i + 1])) for i in range(0, len(lines), k)]


def all_rows_args(args):
    """the same references, --trim and --split, and --min_length 1 as the only threshold"""
    out, i = ["--min_length", "1"], 0
    while i < len(args):
        if args[i] in ("-a", "-1", "-2", "--split", "--window_size"):
            out += args[i:i + 2]
            i += 2
            continue
        if args[i] == "--trim":
            out.append(args[i])
        i += 1 + (args[i] in ("-p", "-t", "-l", "-L", "-q", "--min_mean_q", "--min_window_q", "--gpus", "--length_weight",
                               "--mean_q_weight", "--window_q_weight"))
    return out


_all_rows = {}


def check(inputs, args, key, tmp_path, stdin=False, env=None):
    """the two runs, and FILE against the all-rows run; returns FILE's bytes"""
    path = inputs[key]
    data = open(path, "rb").read() if stdin else None
    where = "-" if stdin else path
    failed = tmp_path / "failed.out"
    rc0, out0, err0 = run(args + [where], data, env)
    rc1, out1, err1 = run(args + ["--failed", str(failed), where], data, env)
    assert rc0 == rc1 == 0, err1[-2000:]
    assert out1 == out0
    assert err1 == err0
    F = failed.read_bytes()
    plain = all_rows_args(args)
    k = (key, tuple(plain))
    if k not in _all_rows:
        rc, out_all, err = run(plain + [path])
        assert rc == 0, err[-2000:]
        _all_rows[k] = out_all
    bam = key == "BAM"
    compressed = bam or "--bgzip" in args
    h_out, r_out = unpack(out1, compressed, bam)
    h_f, r_f = unpack(F, compressed, bam)
    h_all, r_all = unpack(_all_rows[k], bam, bam)
    assert h_out == h_f == h_all
    kept = {r for r, _ in r_out}
    assert len(kept) == len(r_out)
    assert [r for r, _ in r_all if r not in kept] == [r for r, _ in r_f]
    assert sum(b for _, b in r_out) + sum(b for _, b in r_f) == sum(b for _, b in r_all)
    assert len(r_out) + len(r_f) == len(r_all)
    return F


CASES = [
    ("phred", ["-p", "90"], "FQ"),
    ("target_not_enough", ["-t", "1g"], "FQ"),
    ("target_already_below", ["-t", "1000", "-l", "100000"], "FQ"),
    ("target_keeping", ["-t", "2m"], "FQ"),
    ("min_length", ["-l", "2000"], "FQ"),
    ("max_length", ["-L", "5000"], "FQ"),
    ("min_mean_q", ["-q", "15"], "FQ"),
    ("min_window_q", ["--min_window_q", "9", "--window_size", "100"], "FQ"),
    ("asm_trim_split", ["-a", "LFA", "-p", "80", "--trim", "--split", "100"], "FQ"),
    ("short_trim_split", ["-1", "S1", "-2", "S2", "-p", "85", "--trim", "--split", "250"], "CRLF"),
    ("fasta_reads", ["-a", "FA", "-p", "70"], "FASTA"),
    ("crlf", ["-p", "60", "--min_mean_q", "70"], "CRLF"),
    ("verbose", ["-a", "LFA", "-p", "80", "--verbose"], "FQ"),
    ("gzip", ["-p", "90"], "FQGZ"),
    ("bgzf", ["-p", "50"], "BGZF"),
    ("bam", ["-p", "90"], "BAM"),
    ("bam_trim_split", ["-a", "LFA", "-p", "80", "--trim", "--split", "100"], "BAM"),
]


@need_cli
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_failed_is_the_complement(inputs, case, tmp_path):
    name, args, key = case
    F = check(inputs, [inputs.get(a, a) for a in args], key, tmp_path)
    if name == "target_already_below":
        assert len(F) > 1_000_000
    if key == "BAM":
        assert F[:4] == b"\x1f\x8b\x08\x04"


@need_cli
@pytest.mark.gpu
def test_failed_with_the_input_through_a_pipe(inputs, tmp_path):
    F = check(inputs, ["-p", "90"], "FQ", tmp_path, stdin=True)
    (tmp_path / "file").mkdir()
    assert F == check(inputs, ["-p", "90"], "FQ", tmp_path / "file")


@need_cli
@pytest.mark.gpu
@pytest.mark.parametrize("case", [("mapped", ["-p", "90"], "FQ"), ("reparse", ["-p", "60", "--min_mean_q", "70"], "CRLF")],
                         ids=lambda c: c[0])
def test_bgzip_failed_inflates_to_the_plain_failed(inputs, case, tmp_path):
    """FILE is BGZF with the EOF block; the re-parse path runs two compressors on one context"""
    _, args, key = case
    (tmp_path / "z").mkdir()
    (tmp_path / "p").mkdir()
    Fz = check(inputs, args + ["--bgzip"], key, tmp_path / "z")
    Fp = check(inputs, args, key, tmp_path / "p")
    assert Fz.endswith(bgzf_util.EOF_MEMBER) and len(bgzf_util.members(Fz)) > 1
    assert gzip.decompress(Fz) == Fp and len(Fp) > 0


@need_cli
@pytest.mark.gpu
@pytest.mark.skipif(gpu_count() < 2, reason="needs two GPUs")
def test_failed_over_two_gpus(inputs, tmp_path):
    args = ["-a", inputs["LFA"], "-p", "80", "--trim", "--split", "100"]
    (tmp_path / "one").mkdir()
    F1 = check(inputs, args, "FQ", tmp_path / "one", env={"FL_CHUNK_MB": "1"})
    F2 = check(inputs, args + ["--gpus", "2"], "FQ", tmp_path, env={"FL_CHUNK_MB": "1"})
    assert F1 == F2


@need_cli
@pytest.mark.gpu
def test_nothing_fails(inputs, tmp_path):
    assert check(inputs, ["--min_length", "1"], "FQ", tmp_path) == b""
    F = check(inputs, ["--min_length", "1"], "BAM", tmp_path)
    raw = gzip.decompress(open(inputs["BAM"], "rb").read())
    assert gzip.decompress(F) == raw[:bu.header_end(raw)] and F.endswith(bgzf_util.EOF_MEMBER)


@need_cli
@pytest.mark.gpu
def test_a_failed_write_to_failed(inputs, tmp_path):
    for key in ("FQ", "CRLF"):
        rc0, out0, _ = run(["-p", "80", inputs[key]])
        rc, out, err = run(["-p", "80", "--failed", "/dev/full", inputs[key]])
        assert rc0 == 0 and rc == 1
        assert b"Error: cannot write to file: /dev/full" in err
        assert out in (b"", out0)


# ---- errors found while the arguments are checked: exit 1, nothing on stdout, no read scored ----
@pytest.fixture
def small(tmp_path):
    fq = util.write_fastq(tmp_path / "x.fastq", [("r1", b"ACGT" * 10, b"I" * 40)])
    fa = util.write_fasta(tmp_path / "a.fasta", [("c", b"ACGT" * 30)])
    return fq, fa


def refused(args, stdout=subprocess.PIPE):
    rc, out, err = run(args, stdout=stdout)
    assert rc == 1, err
    assert out in (b"", None)
    lines = err.decode().splitlines()
    assert len(lines) == 1 and lines[0].startswith("Error: "), err
    return lines[0]


@need_cli
def test_failed_dash_is_refused(small):
    assert "standard output" in refused(["-p", "90", "--failed", "-", small[0]])


@need_cli
def test_failed_is_not_an_input(small, tmp_path):
    fq, fa = small
    before = open(fq, "rb").read()
    assert "input file" in refused(["-p", "90", "--failed", fq, fq])
    assert open(fq, "rb").read() == before
    link = tmp_path / "again.fastq"
    os.link(fq, link)                                          # the same file by another name
    assert "input file" in refused(["-p", "90", "--failed", str(link), fq])
    assert "input file" in refused(["-a", fa, "-p", "90", "--failed", fa, fq])
    with open(fq, "rb") as f:                                  # the input read from standard input
        p = subprocess.run([CLI, "-p", "90", "--failed", fq, "-"], stdin=f, capture_output=True, timeout=TIMEOUT)
    assert p.returncode == 1 and p.stdout == b"" and b"input file" in p.stderr
    assert open(fq, "rb").read() == before
    assert open(fa, "rb").read().startswith(b">c\n")


@need_cli
def test_failed_in_a_missing_directory(small, tmp_path):
    path = str(tmp_path / "no" / "such" / "failed.fastq")
    assert refused(["-p", "90", "--failed", path, small[0]]) == "Error: cannot write to file: " + path


@need_cli
def test_failed_is_not_standard_output(small, tmp_path):
    out = tmp_path / "out.fastq"
    with open(out, "wb") as f:
        assert "standard output" in refused(["-p", "90", "--failed", str(out), small[0]], stdout=f)
    assert out.read_bytes() == b""
    with open(out, "wb") as f:
        assert "standard output" in refused(["-p", "90", "--failed", "/dev/stdout", small[0]], stdout=f)

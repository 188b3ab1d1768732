"""`filtlong --bgzip`: stdout compressed as BGZF on the GPU. Inflated, it is the plain run's stdout byte for byte, on every
output path (device feeder to a pipe or a file, host reader for CRLF / --verbose, .gz input, FASTA, k-mer references,
several GPUs); the stderr log is the plain run's; the compressed bytes do not depend on the path, the chunk size or the
GPU count; a run reads its own --bgzip output back as BGZF; and the error exits write what plain output writes."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from tests import bgzf_util as bu
from tests import util
from tests.test_cli import CLI, make_inputs, need_cli

pytestmark = [need_cli, pytest.mark.gpu]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(args, env_extra=None, stdout_path=None):
    env = dict(os.environ, LC_ALL="C", **(env_extra or {}))
    env.pop("LANG", None)
    if stdout_path is None:
        p = subprocess.run([CLI] + list(args), capture_output=True, env=env)
        return p.returncode, p.stdout, p.stderr
    with open(stdout_path, "wb") as f:
        p = subprocess.run([CLI] + list(args), stdout=f, stderr=subprocess.PIPE, env=env)
    out = open(stdout_path, "rb").read() if os.path.isfile(stdout_path) else None
    return p.returncode, out, p.stderr


def gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 1


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("bgzip")
    fq_crlf, fa, s1, s2, fasta_reads = make_inputs(d)
    rng = np.random.default_rng(17)
    genome = util.rand_seq(rng, 200000)
    reads = util.long_reads(rng, genome, 1500, max_len=12000)
    fq = util.write_fastq(d / "lf.fastq", reads)
    fqgz = util.write_fastq(d / "lf.fastq.gz", reads)
    return dict(FQ=fq, FQGZ=fqgz, CRLF=fq_crlf, FA=fa, S1=s1, S2=s2, FASTA=fasta_reads, dir=d, genome=genome)


CASES = [
    ["-p", "80", "FQ"],                                             # Phred mode, device feeder
    ["-a", "FA", "-p", "80", "--trim", "--split", "100", "FQ"],
    ["-1", "S1", "-2", "S2", "-p", "85", "FQ"],
    ["-a", "FA", "-p", "70", "FASTA"],
    ["-p", "80", "FQGZ"],
    ["-p", "60", "--min_mean_q", "70", "CRLF"],                      # host reader
    ["-a", "FA", "-p", "80", "--trim", "--split", "100", "--verbose", "CRLF"],
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: " ".join(c))
def test_bgzip_inflates_to_the_plain_output(inputs, case, tmp_path):
    args = [inputs.get(a, a) for a in case]
    rc, plain, err = run(args)
    assert rc == 0, err[-2000:]
    rc, z, zerr = run(args + ["--bgzip"])
    assert rc == 0, zerr[-2000:]
    assert zerr == err
    assert z.endswith(bu.EOF_MEMBER)
    assert gzip.decompress(z) == plain
    inflated = subprocess.run(["gzip", "-dc"], input=z, capture_output=True)
    assert inflated.returncode == 0 and inflated.stdout == plain
    bu.members(z[:-28])
    # the compressed bytes do not depend on the output path, the chunk size or the GPU count
    variants = [dict(stdout_path=str(tmp_path / "out.gz")), dict(env_extra={"FL_CHUNK_MB": "1"}),
                dict(env_extra={"FL_HOST_PARSER": "1"})]
    if gpu_count() >= 2:
        variants.append(dict(extra=["--gpus", "2"]))
    for v in variants:
        extra = v.pop("extra", [])
        rc, z2, _ = run(args + ["--bgzip"] + extra, **v)
        assert rc == 0 and z2 == z, (case, v, extra)


def test_a_bgzip_output_is_read_back_as_bgzf(inputs, tmp_path):
    rc, plain, _ = run(["-p", "90", inputs["FQ"]])
    assert rc == 0 and len(plain) > 2_000_000
    gz = tmp_path / "a.fastq.gz"
    rc, _, _ = run(["-p", "90", "--bgzip", inputs["FQ"]], stdout_path=str(gz))
    assert rc == 0
    fq = tmp_path / "a.fastq"
    fq.write_bytes(plain)
    rc1, out1, err1 = run(["-p", "50", str(gz)])
    rc2, out2, err2 = run(["-p", "50", str(fq)])
    assert rc1 == rc2 == 0 and out1 == out2 and err1 == err2
    dumper = str(tmp_path / "gzmem_dump")
    host = os.path.join(ROOT, "filtlong_b200", "csrc", "host")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-I", host, os.path.join(ROOT, "tests", "gzmem_dump.cpp"),
                        os.path.join(host, "gzmem.cpp"), "-lz", "-lpthread", "-o", dumper], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([dumper, str(gz), "4"], capture_output=True)
    members, threads, is_bgzf = r.stderr.decode().split()
    assert r.returncode == 0 and r.stdout == plain
    assert is_bgzf == "1" and int(members) > 17 and int(threads) > 1


def test_edge_cases(inputs, tmp_path):
    rc, out, _ = run(["--min_length", "1g", "--bgzip", inputs["FQ"]])
    assert rc == 0 and out == bu.EOF_MEMBER
    good = [("a", b"ACGT" * 30, b"I" * 120), ("b", b"ACGT" * 30, b"I" * 120)]
    dup = util.write_fastq(tmp_path / "dup.fastq", good + [("a", b"ACGT" * 20, b"I" * 80)])
    rc_p, out_p, err_p = run(["-t", "100", dup])
    rc_z, out_z, err_z = run(["-t", "100", "--bgzip", dup])
    assert (rc_z, out_z, err_z) == (rc_p, out_p, err_p) and rc_z == 1 and out_z == b""
    rc, _, _ = run(["-p", "80", "--bgzip", inputs["FQ"]], stdout_path="/dev/full")
    assert rc == 1
    rc, _, _ = run(["-p", "80", "--bgzip", inputs["CRLF"]], stdout_path="/dev/full")
    assert rc == 1
    # plain output from the host reader: the re-parse (CR LF) and the mapped slices fail like the feeder's
    rc, _, _ = run(["-p", "80", inputs["CRLF"]], stdout_path="/dev/full")
    assert rc == 1
    rc, _, _ = run(["-p", "80", inputs["FQ"]], env_extra={"FL_HOST_PARSER": "1"}, stdout_path="/dev/full")
    assert rc == 1

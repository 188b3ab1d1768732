"""`filtlong ARGS -`: the input reads from a pipe, read once into memory. Every case runs the CLI with its input fed through
a real pipe by a writer thread in uneven pieces, and again on the same bytes as a file; the two runs must give the same
exit code, byte-identical stdout and the same stderr log once progress redraws are dropped (the file runs are pinned to
the reference by tests/test_cli.py and the suites after it). Covered: FASTQ and FASTA text scored while it arrives, gzip
in one or several members, BGZF, unaligned BAM, the host reader's inputs (CR LF records, --verbose, FL_HOST_PARSER),
--bgzip, many small chunks, an empty stream, the errors a file gives, /dev/stdin and /dev/fd/N as the path, a regular
file on standard input, and two GPUs."""
import gzip
import os
import re
import subprocess
import tempfile
import threading
import time

import numpy as np
import pytest

from tests import bam_util as bu
from tests import util
from tests.test_cli import CLI, final_lines, make_inputs, need_cli

pytestmark = [need_cli, pytest.mark.gpu]
TIMEOUT = 300


def env_of(extra):
    env = dict(os.environ, LC_ALL="C", **(extra or {}))
    env.pop("LANG", None)
    return env


def run_file(args, path, env_extra=None):
    p = subprocess.run([CLI] + list(args) + [path], capture_output=True, env=env_of(env_extra), timeout=TIMEOUT)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


def run_stream(args, data, env_extra=None, path="-", seed=0, stall_at=None, stall_s=1.0):
    """the CLI with `data` written into a pipe in pieces of 1 B .. 1 MiB (a few short pauses; stall_at: a fraction of the
    data after which the writer pauses stall_s seconds). path "-" or "/dev/stdin": the pipe is standard input; "fd": the
    pipe's read end is passed as /dev/fd/N. The CLI is always waited for, or killed, before this returns."""
    rng = np.random.default_rng(seed)
    rfd = wfd = None
    kw = {}
    if path == "fd":
        rfd, wfd = os.pipe()
        argv = [CLI] + list(args) + ["/dev/fd/%d" % rfd]
        kw = dict(stdin=subprocess.DEVNULL, pass_fds=(rfd,))
    else:
        argv = [CLI] + list(args) + [path]
        kw = dict(stdin=subprocess.PIPE)
    with tempfile.TemporaryFile() as out, tempfile.TemporaryFile() as err:
        p = subprocess.Popen(argv, stdout=out, stderr=err, env=env_of(env_extra), **kw)
        sink = p.stdin if rfd is None else os.fdopen(wfd, "wb")
        if rfd is not None:
            os.close(rfd)

        def writer():
            try:
                pos, stalled = 0, False
                while pos < len(data):
                    n = int(rng.integers(1, 1 << 20))
                    sink.write(data[pos:pos + n])
                    sink.flush()
                    pos += n
                    if rng.random() < 0.02:
                        time.sleep(0.01)
                    if stall_at is not None and not stalled and pos >= stall_at * len(data):
                        stalled = True
                        time.sleep(stall_s)
            except (BrokenPipeError, ValueError, OSError):     # the CLI stopped reading (an error, or killed)
                pass
            finally:
                try:
                    sink.close()
                except OSError:
                    pass

        t = threading.Thread(target=writer)
        t.start()
        try:
            rc = p.wait(timeout=TIMEOUT)
        finally:
            if p.poll() is None:
                p.kill()
                p.wait()
            t.join(timeout=60)
        out.seek(0)
        err.seek(0)
        return rc, out.read(), err.read().decode(errors="replace")


def gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 1


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("stdin")
    crlf, _, _, _, _ = make_inputs(d)
    rng = np.random.default_rng(29)
    genome = util.rand_seq(rng, 200000)
    reads = util.long_reads(rng, genome, 1500, max_len=12000)
    fq = util.write_fastq(d / "lf.fastq", reads)
    text = open(fq, "rb").read()
    fa = util.write_fasta(d / "asm.fasta", [("contig_1", genome[:120000]), ("contig_2", genome[120000:])], width=60)
    fasta = util.write_fasta(d / "reads.fasta", [(n, s) for n, s, _ in reads[:300]], width=80)
    half = text.index(b"\n@read_700\n") + 1
    files = dict(FQ=fq, FA=fa, FASTA=fasta, CRLF=crlf)
    for key, data in (("FQGZ", gzip.compress(text, 6)), ("MEMBERS", gzip.compress(text[:half], 1) + gzip.compress(text[half:], 9)),
                      ("EMPTY", b""), ("DUP", b"@a\n" + b"ACGT" * 30 + b"\n+\n" + b"I" * 120 + b"\n@b\nACGT\n+\nIIII\n@a\nACGT\n+\nIIII\n"),
                      ("MIXED", b"@a\nACGTACGT\n+\nIIIIIIII\n>b\nACGTACGT\n")):
        files[key] = str(d / key)
        open(files[key], "wb").write(data)
    # BGZF: an earlier --bgzip output
    files["BGZF"] = str(d / "bgzf.fastq.gz")
    with open(files["BGZF"], "wb") as f:
        assert subprocess.run([CLI, "-p", "90", "--bgzip", fq], stdout=f, stderr=subprocess.DEVNULL, env=env_of(None), timeout=TIMEOUT).returncode == 0
    # unaligned BAM of the same reads, with tags
    recs = [(n.encode(), s.upper(), bytes(x - 33 for x in q), bu.aux_z(b"RG", b"rg1") + bu.aux_f(b"qs", 11.5)) for n, s, q in reads[:800]]
    files["BAM"] = str(d / "reads.bam")
    open(files["BAM"], "wb").write(bu.bgzf(bu.bam_of(recs, bu.header(refs=[(b"chr1", 200000)]))))
    # over 20 MB, for many 1 MB chunks
    big = util.long_reads(np.random.default_rng(31), genome, 2600, max_len=20000)
    files["BIG"] = util.write_fastq(d / "big.fastq", big)
    assert os.path.getsize(files["BIG"]) >= 20 << 20
    return files


CASES = [
    ("fastq", ["-p", "90"], "FQ", None),
    ("asm_trim_split", ["-a", "FA", "-p", "80", "--trim", "--split", "100"], "FQ", None),
    ("fasta_reads", ["-a", "FA", "-p", "70"], "FASTA", None),
    ("gzip", ["-p", "90"], "FQGZ", None),
    ("gzip_members", ["-p", "85"], "MEMBERS", None),
    ("bgzf", ["-p", "50"], "BGZF", None),
    ("bam", ["-a", "FA", "-p", "80", "--trim", "--split", "100"], "BAM", None),
    ("crlf", ["-p", "60", "--min_mean_q", "70"], "CRLF", None),
    ("verbose", ["-a", "FA", "-p", "80", "--verbose"], "FQ", None),
    ("host_parser", ["-p", "90"], "FQ", {"FL_HOST_PARSER": "1"}),
    ("bgzip", ["-p", "90", "--bgzip"], "FQ", None),
    ("chunk_1mb", ["-p", "90"], "BIG", {"FL_CHUNK_MB": "1"}),
    ("empty", ["-p", "90"], "EMPTY", None),
    ("duplicate_name", ["-t", "100"], "DUP", None),
    ("mixed_fasta_fastq", ["-t", "100"], "MIXED", None),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_stdin_equals_the_file(inputs, case):
    name, args, key, env = case
    args = [inputs.get(a, a) for a in args]
    path = inputs[key]
    data = open(path, "rb").read()
    rc_f, out_f, err_f = run_file(args, path, env)
    rc_s, out_s, err_s = run_stream(args, data, env, seed=len(name))
    assert rc_s == rc_f, (name, err_s[-2000:])
    assert out_s == out_f, name
    assert final_lines(err_s) == final_lines(err_f), name
    if name in ("duplicate_name", "mixed_fasta_fastq"):
        assert rc_s == 1 and out_s == b""
    elif name != "empty":
        assert rc_s == 0 and len(out_s) > 0
    if name == "bam":
        assert out_s[:4] == b"\x1f\x8b\x08\x04"


@pytest.mark.parametrize("how", ["/dev/stdin", "fd", "regular_file_on_stdin"])
def test_other_ways_to_name_a_stream(inputs, how):
    args = ["-a", inputs["FA"], "-p", "80", "--trim", "--split", "100"]
    rc_f, out_f, err_f = run_file(args, inputs["FQ"])
    if how == "regular_file_on_stdin":
        with open(inputs["FQ"], "rb") as f:
            p = subprocess.run([CLI] + args + ["-"], stdin=f, capture_output=True, env=env_of(None), timeout=TIMEOUT)
        rc_s, out_s, err_s = p.returncode, p.stdout, p.stderr.decode(errors="replace")
    else:
        rc_s, out_s, err_s = run_stream(args, open(inputs["FQ"], "rb").read(), path=how, seed=3)
    assert rc_s == rc_f == 0, err_s[-2000:]
    assert out_s == out_f and final_lines(err_s) == final_lines(err_f)


def test_chunks_are_scored_while_the_stream_arrives(inputs):
    """¾ of a many-chunk input, a pause, then the rest: FL_CLI_TIMING's stream line counts the chunks scored before the end"""
    data = open(inputs["BIG"], "rb").read()
    env = {"FL_CHUNK_MB": "1", "FL_CLI_TIMING": "1"}
    rc, out, err = run_stream(["-p", "90"], data, env, seed=11, stall_at=0.75, stall_s=1.5)
    assert rc == 0, err[-2000:]
    m = re.search(r"^\[timing\] stream: (\d+) bytes, (\d+) of (\d+) chunks scored before its end$", err, re.M)
    assert m, err[-2000:]
    assert int(m.group(1)) == len(data) and int(m.group(3)) >= 20 and 1 <= int(m.group(2)) < int(m.group(3))
    rc_f, out_f, _ = run_file(["-p", "90"], inputs["BIG"], {"FL_CHUNK_MB": "1"})
    assert rc_f == 0 and out == out_f


@pytest.mark.skipif(gpu_count() < 2, reason="needs two GPUs")
def test_stdin_over_two_gpus(inputs):
    args = ["-a", inputs["FA"], "-p", "80", "--trim", "--split", "100", "--gpus", "2"]
    env = {"FL_CHUNK_MB": "1"}
    rc_f, out_f, err_f = run_file(args, inputs["BIG"], env)
    rc_s, out_s, err_s = run_stream(args, open(inputs["BIG"], "rb").read(), env, seed=5)
    assert rc_s == rc_f == 0, err_s[-2000:]
    assert out_s == out_f and final_lines(err_s) == final_lines(err_f)

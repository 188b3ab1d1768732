"""`--failed FILE` in the CLI's pass-2 writer (filtlong_b200/csrc/host/survivors.h) on the CPU: with a second output, stdout
still gets exactly the survivors, and the second output gets what stdout would get with every row's pass flag inverted --
on every way the writer has (writev, pwrite groups, the choice between them, the re-parse that feeds both outputs from
one parse), to a pipe and to a regular file that already holds bytes, in one or several parts; a failed write to the
second output is reported while stdout is complete; and BAM writes its header and the failed records to the second
output."""
import os
import subprocess
import threading

import numpy as np
import pytest

from tests import bam_util as bu
from tests.test_bam_host import make_results
from tests.test_survivor_writer import make_case, reference_pass2, write_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "filtlong_b200")
HOST_LIB = os.path.join(PKG, "libfiltlong_host.a")
pytestmark = pytest.mark.skipif(not os.path.exists(HOST_LIB), reason="host library not built")


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("failed") / "failed_dump")
    cmd = ["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "failed_dump.cpp"), HOST_LIB, "-L" + PKG, "-lfiltlong_b200",
           "-lz", "-lpthread", "-Wl,-rpath," + PKG, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def inverted(results):
    return [(n, [(s, e, 1 - p) for s, e, p in rows]) for n, rows in results]


@pytest.fixture(scope="module", params=["fastq", "fasta"])
def case(request, tmp_path_factory):
    fasta = request.param == "fasta"
    d = tmp_path_factory.mktemp("failed_" + request.param)
    text, recs, results = make_case(np.random.default_rng(41 + fasta), fasta)
    inp = d / ("in." + request.param)
    inp.write_bytes(text)
    # flip: the same case with every flag inverted, so that each output once holds the 9 MB read (more than a copy buffer)
    specs, want = {}, {}
    for flip, res in ((False, results), (True, inverted(results))):
        want[flip] = reference_pass2(recs, res, fasta)
        for n_parts in (1, 2):
            specs[flip, n_parts] = str(d / ("%d_%d.spec" % (flip, n_parts)))
            write_spec(specs[flip, n_parts], recs, res, n_parts)
    assert len(want[False]) > 8 << 20 and len(want[True]) > 2 << 20
    return dict(fmt=request.param, input=str(inp), specs=specs, want=want)


def run(dumper, c, mode, lead, n_parts, flip, failed_fd, stdout=subprocess.PIPE):
    r = subprocess.run([dumper, mode, c["fmt"], lead, c["input"], c["specs"][flip, n_parts], str(failed_fd)], stdout=stdout,
                       stderr=subprocess.PIPE, pass_fds=(failed_fd,))
    return r, c["want"][flip], c["want"][not flip]


def modes(pwrite=True):
    return [(m, p) for m in ("auto", "writev") + (("pwrite",) if pwrite else ()) for p in (1, 2)] + [("reparse", 1)]


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("lead", ["0", "1"])
@pytest.mark.parametrize("mode,n_parts", modes(pwrite=False))           # pwrite() needs a regular file
def test_failed_to_a_pipe(dumper, case, mode, n_parts, lead, flip):
    rfd, wfd = os.pipe()
    got = []
    reader = threading.Thread(target=lambda: got.append(b"".join(iter(lambda: os.read(rfd, 1 << 20), b""))))
    reader.start()
    try:
        r, want, want_failed = run(dumper, case, mode, lead, n_parts, flip, wfd)
    finally:
        os.close(wfd)
        reader.join()
        os.close(rfd)
    assert r.returncode == 0, r.stderr
    assert r.stdout == want
    assert got[0] == want_failed


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("lead", ["0", "1"])
@pytest.mark.parametrize("mode,n_parts", modes())
def test_failed_to_a_regular_file_after_existing_bytes(dumper, case, mode, n_parts, lead, flip, tmp_path):
    out = tmp_path / "failed"
    out.write_bytes(b"HEAD\n")
    fd = os.open(out, os.O_WRONLY)
    try:
        os.lseek(fd, 0, os.SEEK_END)
        with open(tmp_path / "out", "wb") as stdout:           # a regular file too: every mode can write stdout there
            r, want, want_failed = run(dumper, case, mode, lead, n_parts, flip, fd, stdout=stdout)
        end = os.lseek(fd, 0, os.SEEK_CUR)                  # left at the end of what was written
    finally:
        os.close(fd)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "out").read_bytes() == want
    assert out.read_bytes() == b"HEAD\n" + want_failed
    assert end == 5 + len(want_failed)


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("mode,n_parts", modes())
def test_a_failed_write_to_failed_is_reported_and_stdout_is_complete(dumper, case, mode, n_parts, flip, tmp_path):
    fd = os.open("/dev/full", os.O_WRONLY)
    try:
        with open(tmp_path / "out", "wb") as out:                # a regular file: every mode can write stdout there
            r, want, _ = run(dumper, case, mode, "1", n_parts, flip, fd, stdout=out)
    finally:
        os.close(fd)
    assert r.returncode == 1 and r.stderr == b"failed\n", r.stderr
    assert (tmp_path / "out").read_bytes() == want


@pytest.mark.parametrize("no_qual_every", [0, 4])
def test_bam_failed_equals_the_expected_output_of_the_inverted_results(dumper, tmp_path, no_qual_every):
    rng = np.random.default_rng(70 + no_qual_every)
    reads = bu.random_reads(rng, 600, hi=4000, no_qual_every=no_qual_every)
    raw = bu.bam_of(reads, bu.header(refs=[(b"chr1", 1000)]))
    path = tmp_path / "in.bam"
    path.write_bytes(bu.bgzf(raw))
    results = make_results(rng, reads)
    spec = tmp_path / "spec"
    spec.write_text("".join("%d " % n + " ".join("%d %d %d" % row for row in rows) + "\n" for n, rows in results))
    failed = tmp_path / "failed.bam"
    fd = os.open(failed, os.O_WRONLY | os.O_CREAT | os.O_TRUNC)
    try:
        r = subprocess.run([dumper, "auto", "bam", "-", str(path), str(spec), str(fd)], capture_output=True, pass_fds=(fd,))
    finally:
        os.close(fd)
    assert r.returncode == 0, r.stderr
    assert r.stdout == bu.expected_output(raw, results)
    got = failed.read_bytes()
    assert got == bu.expected_output(raw, inverted(results))
    h = bu.header_end(raw)
    assert r.stdout[:h] == got[:h] == raw[:h]                 # the header goes to both outputs
    kept = {x["name"] for x in bu.records(r.stdout)}
    dropped = {x["name"] for x in bu.records(got)}
    assert kept and dropped and not kept & dropped


def test_nothing_failed_leaves_failed_empty(dumper, tmp_path):
    text, recs, results = make_case(np.random.default_rng(3), False, n=200)
    results = [(n, [(s, e, 1) for s, e, _ in rows]) for n, rows in results]
    inp = tmp_path / "in.fastq"
    inp.write_bytes(text)
    spec = str(tmp_path / "spec")
    write_spec(spec, recs, results, 1)
    for mode in ("auto", "reparse"):
        out = tmp_path / ("failed_" + mode)
        fd = os.open(out, os.O_WRONLY | os.O_CREAT | os.O_TRUNC)
        try:
            r = subprocess.run([dumper, mode, "fastq", "1", str(inp), spec, str(fd)], capture_output=True, pass_fds=(fd,))
        finally:
            os.close(fd)
        assert r.returncode == 0 and r.stdout == reference_pass2(recs, results, False)
        assert out.read_bytes() == b""

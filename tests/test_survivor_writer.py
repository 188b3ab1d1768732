"""The CLI's pass-2 writer (filtlong_b200/csrc/host/survivors.h) on the CPU: given a table of where each record sits in
the input and the scoring results, every way it has of getting the survivors to stdout -- writev to a pipe, pwrite groups
into a regular file, writev behind O_APPEND, and the buffered re-parse -- prints what the reference's pass 2 prints
(reference src/main.cpp:263-313), and a failed write is reported on each of them."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "filtlong_b200")
HOST_LIB = os.path.join(PKG, "libfiltlong_host.a")
pytestmark = pytest.mark.skipif(not os.path.exists(HOST_LIB), reason="host library not built")


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("surv") / "survivors_dump")
    cmd = ["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "survivors_dump.cpp"), HOST_LIB, "-L" + PKG, "-lfiltlong_b200",
           "-lz", "-lpthread", "-Wl,-rpath," + PKG, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def make_case(rng, fasta, n=1500):
    """(file bytes, records with their offsets, per-read results). Results: kept and dropped reads, and reads with
    children, some of them kept, dropped or of length 0. Long reads make the writers flush mid-run: read 8 alone is more
    than a copy buffer."""
    comments = [b"", b"c1 c2\tc3", b"x", b"", b"tab\tsep"]
    text, recs, results = bytearray(), [], []
    for i in range(n):
        L = 9_000_000 if i == 8 else 3_000_000 if i % 500 == 7 else int(rng.integers(1, 2500))
        name, comment = b"read_%d" % i, comments[i % len(comments)]
        seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=L)].tobytes()
        qual = (rng.integers(33, 75, size=L).astype(np.uint8)).tobytes()
        name_off = len(text) + 1
        text += (b">" if fasta else b"@") + name + ((b" " + comment) if comment else b"") + b"\n"
        seq_off = len(text)
        text += seq + b"\n"
        qual_off = 0
        if not fasta:
            text += b"+\n"
            qual_off = len(text)
            text += qual + b"\n"
        recs.append(dict(name=name, comment=comment, seq=seq, qual=qual, offs=(name_off, len(name), len(comment), seq_off, qual_off, L)))
        kind = i % 4
        if kind < 2 or L < 10:
            results.append((0, [(0, L, int(i == 8 or rng.random() < 0.6))]))
        else:
            cuts = sorted(set(int(c) for c in rng.integers(0, L + 1, size=5)))
            rows = [(a, b, int(rng.random() < 0.7)) for a, b in zip(cuts[:-1], cuts[1:])]
            rows += [(cuts[0], cuts[0], 1)]                                  # a kept child of length 0
            results.append((len(rows), rows))
    return bytes(text), recs, results


def reference_pass2(recs, results, fasta):
    """main.cpp:263-313, restated."""
    out = bytearray()
    lead = b">" if fasta else b"@"
    for r, (n_child, rows) in zip(recs, results):
        tail = (b" " + r["comment"]) if r["comment"] else b""
        if n_child == 0:
            if rows[0][2]:
                out += lead + r["name"] + tail + b"\n" + r["seq"] + b"\n"
                if not fasta:
                    out += b"+\n" + r["qual"] + b"\n"
            continue
        for s, e, passed in rows:
            if passed and e - s > 0:
                out += lead + r["name"] + b"_%d-%d" % (s + 1, e) + tail + b"\n" + r["seq"][s:e] + b"\n"
                if not fasta:
                    out += b"+\n" + r["qual"][s:e] + b"\n"
    return bytes(out)


def write_spec(path, recs, results, n_parts):
    bounds = [len(recs) * k // n_parts for k in range(n_parts + 1)]
    with open(path, "w") as f:
        for k in range(n_parts):
            f.write("P\n")
            for r, (n_child, rows) in zip(recs[bounds[k]:bounds[k + 1]], results[bounds[k]:bounds[k + 1]]):
                f.write("R %d %d %d %d %d %d " % r["offs"] + "%d\n" % n_child)
                f.write("".join("W %d %d %d\n" % row for row in rows))


@pytest.fixture(scope="module", params=["fastq", "fasta"])
def case(request, tmp_path_factory):
    fasta = request.param == "fasta"
    d = tmp_path_factory.mktemp(request.param)
    text, recs, results = make_case(np.random.default_rng(31 + fasta), fasta)
    inp = d / ("in." + request.param)
    inp.write_bytes(text)
    one, two = str(d / "one.spec"), str(d / "two.spec")
    write_spec(one, recs, results, 1)
    write_spec(two, recs, results, 2)
    want = reference_pass2(recs, results, fasta)
    assert len(want) > 8 << 20
    return dict(fmt=request.param, input=str(inp), one=one, two=two, want=want, text=text, dir=d)


def run(dumper, c, mode, lead, stdout, spec=None):
    spec = spec or (c["one"] if mode == "reparse" else c["two"])
    return subprocess.run([dumper, mode, c["fmt"], lead, c["input"], spec], stdout=stdout, stderr=subprocess.PIPE)


@pytest.mark.parametrize("lead", ["0", "1"])
@pytest.mark.parametrize("mode", ["auto", "writev", "reparse"])
def test_pipe(dumper, case, mode, lead):
    r = run(dumper, case, mode, lead, subprocess.PIPE)
    assert r.returncode == 0, r.stderr
    assert r.stdout == case["want"]


@pytest.mark.parametrize("lead", ["0", "1"])
@pytest.mark.parametrize("mode,append", [("auto", False), ("pwrite", False), ("reparse", False), ("auto", True), ("reparse", True)])
def test_regular_file_after_existing_bytes(dumper, case, mode, append, lead, tmp_path):
    out = tmp_path / "out"
    out.write_bytes(b"HEAD\n")
    fd = os.open(out, os.O_WRONLY | (os.O_APPEND if append else 0))
    try:
        os.lseek(fd, 0, os.SEEK_END)
        r = run(dumper, case, mode, lead, fd)
        assert r.returncode == 0, r.stderr
        end = os.lseek(fd, 0, os.SEEK_CUR)                  # the descriptor is left at the end of what was written
    finally:
        os.close(fd)
    assert out.read_bytes() == b"HEAD\n" + case["want"]
    assert end == 5 + len(case["want"])


@pytest.mark.parametrize("mode", ["auto", "writev", "pwrite", "reparse"])
def test_a_failed_write_is_reported(dumper, case, mode):
    with open("/dev/full", "wb") as full:
        r = run(dumper, case, mode, "1", full)
    assert r.returncode == 1, r.stderr


def test_a_table_past_the_end_of_the_input_is_refused(dumper, case):
    short = case["dir"] / "short"
    short.write_bytes(case["text"][:-10])
    r = subprocess.run([dumper, "auto", case["fmt"], "1", str(short), case["one"]], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 4 and r.stdout == b""

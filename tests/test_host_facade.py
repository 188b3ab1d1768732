"""The reference-compatible C++ classes (filtlong_b200/csrc/host: Kmers, Read) used the way the
reference's main uses them -- `Read(name, seq, qscores, length, &kmers, &args)` per record -- against
the unmodified reference objects (oracle/_ref/refdump, replayed from tests/golden). Same public fields, same values."""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "filtlong_b200")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def facade(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("facade") / "facade_dump")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", os.path.join(ROOT, "tests", "facade_dump.cpp"),
           os.path.join(PKG, "libfiltlong_host.a"), "-L" + PKG, "-lfiltlong_b200", "-lz", "-Wl,-rpath," + PKG, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


@pytest.mark.parametrize("opts", [["--min_length", "1"], ["-a", "ASM", "--trim", "--split", "60", "--min_window_q", "50"]])
def test_read_and_kmers_classes_match_reference(facade, opts, tmp_path):
    rng = np.random.default_rng(8)
    genome = util.rand_seq(rng, 30000)
    reads = util.long_reads(rng, genome, 40, max_len=4000)
    reads.append(("mid_junk", genome[100:500] + util.rand_seq(rng, 150) + genome[900:1400], b"5" * 1050))
    fq = util.write_fastq(tmp_path / "r.fastq", reads)
    fa = util.write_fasta(tmp_path / "a.fasta", [("g", genome)], width=60)
    args = [fa if a == "ASM" else a for a in opts] + [fq]
    env = dict(os.environ, LC_ALL="C")
    got = subprocess.run([facade] + args, capture_output=True, text=True, env=env)
    assert got.returncode == 0, got.stderr[-1000:]
    ref = orc.run_refdump(args)
    lines = got.stdout.splitlines()
    assert lines[0] == "K %d" % ref["n_kmers"]
    mine = {"R": [], "B": [], "C": []}
    for l in lines:
        if l[0] in mine:
            mine[l[0]].append(l)
    want_R, want_B, want_C = [], [], []
    for r in ref["reads"]:
        want_R.append((r["idx"], r["name"], r["length"], r["mean_q"], r["window_q"], r["length_score"], r["passed"], r["first"],
                       r["last"], r["n_bad"], r["n_child"]))
        want_B += [(r["idx"], b[0], b[1]) for b in r["bad"]]
        want_C += [(r["idx"], ci, c["name"], c["start"], c["end"], c["mean_q"], c["window_q"], c["length_score"], c["passed"])
                   for ci, c in enumerate(r["children"])]
    got_R = []
    for l in mine["R"]:
        f = l.split()
        got_R.append((int(f[1]), f[2], int(f[3]), float.fromhex(f[4]), float.fromhex(f[5]), float.fromhex(f[6]), int(f[7]), int(f[8]),
                      int(f[9]), int(f[10]), int(f[11])))
    assert got_R == want_R
    assert [tuple(map(int, l.split()[1:])) for l in mine["B"]] == want_B
    got_C = []
    for l in mine["C"]:
        f = l.split()
        got_C.append((int(f[1]), int(f[2]), f[3], int(f[4]), int(f[5]), float.fromhex(f[6]), float.fromhex(f[7]), float.fromhex(f[8]),
                      int(f[9])))
    assert got_C == want_C

"""FastxReader's stream offsets (used by the CLI's pass 2 to copy slices of the input instead of parsing
it again, main.cpp:263-313): for every record it calls `simple`, the file's bytes at the reported
offsets are exactly the name, the comment, the sequence and the quality it parsed; records it cannot vouch for
(multi-line, CR LF) are flagged; gzip input is reported as not plain."""
import gzip
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "filtlong_b200", "csrc", "host")


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("fx") / "fastx_offsets_dump")
    r = subprocess.run(["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "fastx_offsets_dump.cpp"),
                        os.path.join(HOST, "fastx.cpp"), "-lz", "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def records(rng, n):
    recs = []
    for i in range(n):
        L = int(rng.integers(1, 400)) if i % 7 else int(rng.integers(60000, 140000))      # some span the 64 KiB buffer
        seq = bytes(rng.choice(np.frombuffer(b"ACGTN", np.uint8), size=L))
        qual = bytes(rng.integers(33, 127, size=L).astype(np.uint8))
        comment = [b"", b"c1 c2\tc3", b"x"][i % 3]
        recs.append((b"r%d" % i, comment, seq, qual))
    return recs


def write(path, recs, style):
    with open(path, "wb") as f:
        for i, (name, comment, seq, qual) in enumerate(recs):
            hdr = b"@" + name + ((b" " + comment) if comment else b"")
            if style == "simple":
                f.write(hdr + b"\n" + seq + b"\n+\n" + qual + b"\n")
            elif style == "mixed":
                if i % 4 == 1 and len(seq) > 10:          # two-line sequence and quality
                    h = len(seq) // 2
                    f.write(hdr + b"\n" + seq[:h] + b"\n" + seq[h:] + b"\n+" + name + b"\n" + qual[:h] + b"\n" + qual[h:] + b"\n")
                elif i % 4 == 2:                          # CR LF
                    f.write(hdr + b"\r\n" + seq + b"\r\n+\r\n" + qual + b"\r\n")
                elif i % 4 == 3:                          # blank line before the record, '+' line repeats the name
                    f.write(b"\n" + hdr + b"\n" + seq + b"\n+" + name + b" again\n" + qual + b"\n")
                else:
                    f.write(hdr + b"\n" + seq + b"\n+\n" + qual + b"\n")


@pytest.mark.parametrize("style", ["simple", "mixed"])
def test_offsets_point_at_the_parsed_pieces(dumper, style, tmp_path):
    rng = np.random.default_rng(3)
    recs = records(rng, 60)
    path = str(tmp_path / "in.fastq")
    write(path, recs, style)
    data = open(path, "rb").read()
    out = subprocess.run([dumper, path], capture_output=True, text=True)
    assert out.returncode == 0
    lines = out.stdout.splitlines()
    assert lines[-1] == "END -1" and len(lines) == len(recs) + 1
    n_simple = 0
    for (name, comment, seq, qual), line in zip(recs, lines):
        f = line.split("\t")
        assert f[0] == name.decode() and int(f[1]) == len(comment) and int(f[2]) == len(seq) and int(f[3]) == len(qual)
        assert f[8] == "1"
        if f[4] == "1":
            n_simple += 1
            no, co, so, qo = int(f[9]), int(f[5]), int(f[6]), int(f[7])
            assert data[no - 1:no + len(name)] == b"@" + name
            if comment:                                   # pass 2 looks for the comment one byte after the name
                assert co == no + len(name) + 1
            assert data[co:co + len(comment)] == comment
            assert data[so:so + len(seq)] == seq
            assert data[qo:qo + len(qual)] == qual
    if style == "simple":
        assert n_simple == len(recs)
    else:
        assert 0 < n_simple < len(recs)
        for i, line in enumerate(lines[:-1]):
            if i % 4 == 2 or (i % 4 == 1 and len(recs[i][2]) > 10):
                assert line.split("\t")[4] == "0", i        # multi-line and CR LF records are never called simple


def test_fasta_and_gzip(dumper, tmp_path):
    path = str(tmp_path / "a.fasta")
    with open(path, "wb") as f:
        f.write(b">c1 first contig\nACGTACGT\n>c2\nAC\nGT\n>c3\nTTTT\n")
    data = open(path, "rb").read()
    lines = subprocess.run([dumper, path], capture_output=True, text=True).stdout.splitlines()
    f1, f2, f3 = (l.split("\t") for l in lines[:3])
    assert f1[4] == "1" and data[int(f1[6]):int(f1[6]) + 8] == b"ACGTACGT" and data[int(f1[5]):int(f1[5]) + 12] == b"first contig"
    assert data[int(f1[9]):int(f1[9]) + 2] == b"c1" and int(f1[5]) == int(f1[9]) + 3
    assert f2[4] == "0" and int(f2[2]) == 4
    assert f3[4] == "1" and data[int(f3[6]):int(f3[6]) + 4] == b"TTTT" and data[int(f3[9]) - 1:int(f3[9]) + 2] == b">c3"
    gz = str(tmp_path / "r.fastq.gz")
    with gzip.open(gz, "wb") as f:
        f.write(b"@r1\nACGT\n+\nIIII\n")
    lines = subprocess.run([dumper, gz], capture_output=True, text=True).stdout.splitlines()
    assert lines[0].split("\t")[8] == "0"                   # compressed: offsets are not file offsets

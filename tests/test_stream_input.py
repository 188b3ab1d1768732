"""Input reads from a stream (filtlong_b200/csrc/host/streamsrc.cpp), on the CPU: a file fed through a real pipe in uneven
pieces, with pauses, is held in memory byte for byte (inflated, for gzip in every container the file path takes); the
chunks cut while it arrives (plan_next_chunk) are exactly the chunks plan_chunks cuts from the whole buffer, so every cut
is a record start and no chunk is larger than the target; the records read chunk by chunk are the file's records; a
stream larger than the memory budget is declined with a message, and an empty one is an empty input."""
import gzip
import os
import subprocess
import threading
import time

import numpy as np
import pytest

from tests import bgzf_util
from tests.test_textsrc import fastq, fastq_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "filtlong_b200", "csrc", "host")
BIG = 1 << 40                                        # a budget no test input comes near


@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("stream") / "stream_dump")
    srcs = [os.path.join(HOST, s) for s in ("streamsrc.cpp", "textsrc.cpp", "gzmem.cpp", "fastx.cpp")]
    r = subprocess.run(["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "stream_dump.cpp")] + srcs + ["-lz", "-lpthread", "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def feed(exe, data, tmp_path, target=100000, budget=BIG, seed=0, stall_at=None):
    """runs stream_dump with `data` written to its stdin (a pipe) in random pieces of 1 B .. 256 KiB with short pauses;
    stall_at: a fraction of the data after which the writer pauses for 0.3 s. Returns (rc, stdout lines, stderr, held)."""
    rng = np.random.default_rng(seed)
    held = tmp_path / "held.bin"
    if held.exists():
        held.unlink()
    out, err = tmp_path / "out.txt", tmp_path / "err.txt"
    with open(out, "wb") as fo, open(err, "wb") as fe:
        p = subprocess.Popen([exe, str(budget), str(target), str(held)], stdin=subprocess.PIPE, stdout=fo, stderr=fe)
        try:
            pos, stalled = 0, False
            try:
                while pos < len(data):
                    n = int(rng.integers(1, 1 << 18))
                    p.stdin.write(data[pos:pos + n])
                    p.stdin.flush()
                    pos += n
                    if rng.random() < 0.05:
                        time.sleep(float(rng.random()) * 0.02)
                    if stall_at is not None and not stalled and pos >= stall_at * len(data):
                        stalled = True
                        time.sleep(0.3)
            except BrokenPipeError:                  # declined (over the budget): it stopped reading
                pass
            try:
                p.stdin.close()
            except BrokenPipeError:
                pass
            rc = p.wait(timeout=120)
        finally:
            if p.poll() is None:
                p.kill()
                p.wait()
    lines = out.read_bytes().split(b"\n")
    return rc, lines, err.read_bytes().decode(errors="replace"), (held.read_bytes() if held.exists() else None)


def parse(lines):
    chunks = [tuple(int(x) for x in l.split()[1:]) for l in lines if l.startswith(b"CHUNK ")]
    recs = [tuple(l[4:].split(b"\x01")) for l in lines if l.startswith(b"REC ")]
    val = lambda key: [l.split()[1:] for l in lines if l.startswith(key + b" ")][0]
    return dict(chunks=chunks, recs=recs, early=int(val(b"EARLY")[0]), held=[int(x) for x in val(b"HELD")], same=val(b"SAME") == [b"1"],
                end=int(val(b"END")[0]), noplan=b"NOPLAN" in lines)


def record_starts(recs):
    return set(np.cumsum([0] + [len(fastq_bytes([r])) for r in recs]).tolist())


def test_fastq_through_a_pipe_is_cut_while_it_arrives(dumper, tmp_path):
    rng = np.random.default_rng(21)
    recs = fastq(rng, 4000)                          # qualities that start with '@' or hold a '+'
    text = fastq_bytes(recs)
    rc, lines, err, held = feed(dumper, text, tmp_path, seed=1, stall_at=0.6)
    assert rc == 0, err
    d = parse(lines)
    assert held == text and d["held"] == [len(text), 0, len(text)]
    cs = d["chunks"]
    assert len(cs) > 10 and cs[0][0] == 0 and cs[-1][1] == len(text) and not d["noplan"]
    assert all(a[1] == b[0] for a, b in zip(cs, cs[1:]))                # no gap, no overlap
    starts = record_starts(recs)
    assert all(c[0] in starts and 0 < c[1] - c[0] <= 100000 for c in cs)
    assert [c[2] for c in cs] == [0] * (len(cs) - 1) + [1]             # only the chunk cut at the end is the last
    assert d["same"]                                                    # what plan_chunks cuts from the whole buffer
    assert d["early"] >= 1                                              # some chunks were cut before the end
    assert d["end"] == -1 and d["recs"] == recs


@pytest.mark.parametrize("seed", [2, 3, 4])
def test_fastq_chunks_do_not_depend_on_how_the_bytes_arrive(dumper, tmp_path, seed):
    rng = np.random.default_rng(30 + seed)
    recs = fastq(rng, 1500)
    text = fastq_bytes(recs)
    rc, lines, err, held = feed(dumper, text, tmp_path, target=20000 + 7919 * seed, seed=seed)
    assert rc == 0, err
    d = parse(lines)
    assert held == text and d["same"] and d["recs"] == recs and d["end"] == -1


def test_wrapped_fasta_through_a_pipe(dumper, tmp_path):
    rng = np.random.default_rng(22)
    seqs = [bytes(rng.choice(np.frombuffer(b"ACGTNacgt", np.uint8), size=int(L))) for L in rng.integers(1, 30000, size=80)]
    wrap = lambda q: b"".join(q[i:i + 60] + b"\n" for i in range(0, len(q), 60))
    text = b"".join(b">c%d description here\n" % i + wrap(q) for i, q in enumerate(seqs))
    rc, lines, err, held = feed(dumper, text, tmp_path, target=200000, seed=5)
    assert rc == 0, err
    d = parse(lines)
    assert held == text and d["same"] and len(d["chunks"]) >= 4
    assert all(text[c[0]:c[0] + 1] == b">" for c in d["chunks"])
    assert [r[2] for r in d["recs"]] == seqs and d["end"] == -1


def test_a_record_larger_than_the_target_gives_up_like_plan_chunks(dumper, tmp_path):
    text = b">big\n" + b"ACGT" * 50000 + b"\n>small\nACGT\n"
    rc, lines, err, held = feed(dumper, text, tmp_path, target=20000, seed=6)
    assert rc == 0, err
    d = parse(lines)
    assert d["noplan"] and held == text and [r[0] for r in d["recs"]] == [b"big", b"small"]


@pytest.mark.parametrize("kind", ["one", "members", "bgzf", "trailing"])
def test_gzip_streams_are_held_inflated(dumper, tmp_path, kind):
    rng = np.random.default_rng(23)
    a, b = fastq_bytes(fastq(rng, 2000)), fastq_bytes(fastq(rng, 700))
    data, want = {
        "one": (gzip.compress(a + b, 6), a + b),
        "members": (gzip.compress(a, 1) + gzip.compress(b, 9) + gzip.compress(b"", 6), a + b),
        "bgzf": (bgzf_util.zlib_bgzf(a + b) + bgzf_util.EOF_MEMBER, a + b),
        "trailing": (gzip.compress(a + b) + b"\0" * 512, a + b),
    }[kind]
    clean = data[:-512] if kind == "trailing" else data
    assert gzip.decompress(clean) == want
    rc, lines, err, held = feed(dumper, data, tmp_path, seed=7)
    assert rc == 0, err
    d = parse(lines)
    assert held == want and d["held"] == [len(want), 1, len(data)]
    assert d["chunks"] == [] and d["early"] == 0                        # nothing is cut before a gzip stream has ended


def test_a_stream_over_the_budget_is_declined(dumper, tmp_path):
    rng = np.random.default_rng(24)
    text = fastq_bytes(fastq(rng, 3000))
    rc, _, err, held = feed(dumper, text, tmp_path, budget=len(text) // 2, seed=8)
    assert rc == 1 and "standard input did not fit in memory" in err and held is None
    rc, _, err, _ = feed(dumper, text, tmp_path, budget=len(text), seed=8)           # exactly the budget fits
    assert rc == 0, err
    z = gzip.compress(text)                          # compressed and inflated bytes both count
    rc, _, err, held = feed(dumper, z, tmp_path, budget=len(text), seed=9)
    assert rc == 1 and "standard input" in err and "memory" in err and held is None
    rc, _, err, held = feed(dumper, z, tmp_path, budget=len(text) + len(z) + 4096, seed=9)
    assert rc == 0 and held == text, err


def test_an_empty_stream_is_an_empty_input(dumper, tmp_path):
    for data in (b"", gzip.compress(b"")):
        rc, lines, err, held = feed(dumper, data, tmp_path)
        assert rc == 0, err
        d = parse(lines)
        assert held == b"" and d["held"][0] == 0 and d["recs"] == [] and d["end"] == -1

"""The parallel gzip inflater of fl_inflate.h, run serially on the CPU (tests/inflate_dump.cpp) through the same round,
finder, speculative decode, chain / repair, window, resolve and CRC steps the device runs: it must give zlib's bytes or
decline, never different bytes."""
import os
import random

import pytest

from tests import gunzip_corpus as gc

CHUNKS = (4096, 16384, 65536)


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return gc.build_model(str(tmp_path_factory.mktemp("inflate_model")))


@pytest.fixture(scope="module")
def model_asan(tmp_path_factory):
    return gc.build_model(str(tmp_path_factory.mktemp("inflate_model_asan")), sanitize=True)


@pytest.fixture(scope="module")
def cases():
    return gc.corpus()


def _write(tmp_path, name, blob):
    p = str(tmp_path / (name + ".gz"))
    with open(p, "wb") as f:
        f.write(blob)
    return p


@pytest.mark.parametrize("chunk", CHUNKS)
def test_corpus_gives_zlib_bytes_or_declines(model, cases, tmp_path, chunk):
    inflated = declined = 0
    for name, blob in cases:
        want = gc.gzread(blob)
        p = _write(tmp_path, name, blob)
        rc, st, got = gc.run_model(model, p, chunk, 0, len(want) + 4096, str(tmp_path / "out"))
        if rc == 1:
            assert got == want, (name, chunk)
            inflated += 1
            assert st[1] >= 1 and st[3] == 1
        else:
            assert rc == 0, name
            declined += 1
    # everything but Z_FIXED at the smallest chunks (one chunk whose output outgrows its slot) takes the parallel path
    assert inflated >= len(cases) - 1, (inflated, declined)


def test_many_chunks_and_rounds(model, cases, tmp_path):
    """Dozens to hundreds of chunks per file, chunks with less than 32 KiB of output and chunks without a candidate
    start, and a device-memory limit that forces several rounds."""
    name, blob = cases[1]                                          # ont_l6
    want = gc.gzread(blob)
    p = _write(tmp_path, name, blob)
    per_chunk = 4096 * 8 * 3 + (128 << 10) * 3 + 32768 + 4096 * 2
    rc, st, got = gc.run_model(model, p, 4096, len(blob) + 8 * per_chunk, len(want), str(tmp_path / "out"))
    assert rc == 1 and got == want
    members, chunks, redecoded, rounds = st
    assert members == 1 and rounds > 5 and chunks > 20, st
    rc, st1, got = gc.run_model(model, p, 4096, 0, len(want), str(tmp_path / "out"))
    assert rc == 1 and got == want
    assert st1[1] < len(blob) // 4096, "some chunks hold no block start and merge into the one before"


@pytest.mark.parametrize("size", [1 << 20, 4 << 20, 8 << 20])
def test_large_inputs(model, tmp_path, size):
    rnd = random.Random(size)
    data = gc.fastq(rnd, size)
    for level, chunk in ((1, 16384), (6, 65536)):
        blob = gc.deflate_gzip(data, level)
        p = _write(tmp_path, "big", blob)
        rc, st, got = gc.run_model(model, p, chunk, 0, size, str(tmp_path / "out"))
        assert rc == 1 and got == data, (level, chunk, st)
        assert st[1] >= len(blob) // chunk // 3, st


def test_finder_has_no_false_negatives(model, cases, tmp_path):
    """The block-start test accepts every dynamic / stored block start and member header the serial decode meets, over
    the whole stream. False positives are counted over every bit offset of the first 2 Mbit, and only reported: they
    cost a re-decode, never correctness."""
    report = []
    for name, blob in cases:
        if name == "fixed":
            continue
        p = _write(tmp_path, name, blob)
        import subprocess
        limit = min(len(blob) * 8, 2 << 20)
        r = subprocess.run([model, "finder", p, str(limit)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        true_starts, missed, false_pos, fixed = (int(x) for x in r.stdout.split())
        assert missed == 0, (name, r.stdout)
        assert true_starts > 0, name
        report.append("%s: %d starts, %d false positives in %d bits" % (name, true_starts, false_pos, limit))
    print("\n".join(report))


def test_bad_crc_isize_and_truncation_decline(model, tmp_path):
    rnd = random.Random(5)
    data = gc.fastq(rnd, 600000)
    blob = gc.deflate_gzip(data, 6)
    bad_crc = bytearray(blob)
    bad_crc[-8] ^= 1
    bad_isize = bytearray(blob)
    bad_isize[-1] ^= 0x40
    for name, b in (("crc", bad_crc), ("isize", bad_isize), ("trunc", blob[:-3]), ("trunc_mid", blob[:len(blob) // 2]),
                    ("header_only", blob[:10])):
        p = _write(tmp_path, name, bytes(b))
        for chunk in (4096, 65536):
            rc, _, _ = gc.run_model(model, p, chunk, 0, len(data) + 4096, str(tmp_path / "out"))
            assert rc == 0, (name, chunk)
    # over the output capacity
    p = _write(tmp_path, "ok", blob)
    rc, _, _ = gc.run_model(model, p, 16384, 0, len(data) - 1, str(tmp_path / "out"))
    assert rc == 0


def test_mutations_give_zlib_bytes_or_decline_under_sanitizers(model_asan, tmp_path):
    """Bit flips, truncations and inserted bytes: never different bytes, never a read or write out of bounds."""
    rnd = random.Random(99)
    data = gc.fastq(rnd, 200000, 200, 3000)
    bases = [gc.deflate_gzip(data, 6), gc.deflate_gzip(data, 1) + gc.deflate_gzip(data[:5000], 9),
             gc.deflate_gzip(data, 6, flush_every=20000)]
    n_ok = n_declined = 0
    for i in range(36):
        b = bytearray(bases[i % len(bases)])
        kind = i % 3
        if kind == 0:
            for _ in range(rnd.randint(1, 4)):
                b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8)
        elif kind == 1:
            b = b[:rnd.randrange(1, len(b))]
        else:
            at = rnd.randrange(len(b))
            b[at:at] = bytes(rnd.getrandbits(8) for _ in range(rnd.randint(1, 16)))
        b = bytes(b)
        try:
            want = gc.gzread(b)
        except Exception:
            want = None
        p = _write(tmp_path, "m%d" % i, b)
        rc, _, got = gc.run_model(model_asan, p, rnd.choice((4096, 8192)), 0, 400000, str(tmp_path / "out"))
        if rc == 1:
            assert want is not None and got == want, i
            n_ok += 1
        else:
            n_declined += 1
    assert n_declined > 0

"""fl_gzip_inflate on the device: zlib's bytes and the CPU model's statistics (tests/inflate_dump.cpp runs the same
fl_inflate.h steps serially), at small chunks and with device memory limited to force several rounds."""
import zlib

import numpy as np
import pytest

from filtlong_b200 import capi
from tests import gunzip_corpus as gc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    L = capi.lib()
    h = capi.C.c_void_p()
    capi.check(None, L.fl_ctx_create(capi.make_params(), 0, capi.C.byref(h)), "fl_ctx_create")
    yield h
    L.fl_ctx_destroy(h)


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return gc.build_model(str(tmp_path_factory.mktemp("inflate_model_gpu")))


def inflate(ctx, blob, cap, chunk=0, max_dev=0):
    L = capi.lib()
    src = np.frombuffer(blob, dtype=np.uint8)
    out = np.empty(max(cap, 1), dtype=np.uint8)
    n_out, status, st = capi.C.c_uint64(0), capi.C.c_int(-1), capi.GunzipStats()
    rc = L.fl_gzip_inflate(ctx, src.ctypes.data, len(blob), out.ctypes.data, cap, chunk, max_dev, capi.C.byref(n_out),
                           capi.C.byref(status), capi.C.byref(st))
    capi.check(ctx, rc, "fl_gzip_inflate")
    stats = (st.members, st.chunks, st.redecoded, st.rounds)
    if status.value == capi.FL_GUNZIP_OK:
        return status.value, stats, out[:n_out.value].tobytes()
    assert status.value == capi.FL_GUNZIP_DECLINED
    return status.value, stats, None


def per_chunk(chunk):
    return chunk * 8 * 3 + (128 << 10) * 3 + 32768 + 4096 * 2


@pytest.mark.parametrize("chunk", [16384, 65536])
def test_corpus_matches_zlib_and_the_cpu_model(ctx, model, tmp_path, chunk):
    for name, blob in gc.corpus():
        want = gc.gzread(blob)
        p = str(tmp_path / (name + ".gz"))
        open(p, "wb").write(blob)
        for max_dev in (0, len(blob) + 6 * per_chunk(chunk)):
            rc_m, st_m, got_m = gc.run_model(model, p, chunk, max_dev, len(want), str(tmp_path / "out"))
            status, st, got = inflate(ctx, blob, len(want), chunk, max_dev)
            assert (status == capi.FL_GUNZIP_OK) == (rc_m == 1), (name, chunk, max_dev)
            assert st == st_m, (name, chunk, max_dev, st, st_m)
            if status == capi.FL_GUNZIP_OK:
                assert got == want, (name, chunk, max_dev)
            if max_dev and status == capi.FL_GUNZIP_OK and len(blob) > 4 * chunk * 6:
                assert st[3] > 1, (name, st)


def big_fastq(seed, n_bytes, read_len=8000):
    rng = np.random.default_rng(seed)
    rec = []
    total, i = 0, 0
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    while total < n_bytes:
        k = 256
        seq = acgt[rng.integers(0, 4, size=(k, read_len))]
        qual = np.clip(rng.normal(18, 6, size=(k, read_len)), 1, 50).astype(np.uint8) + 33
        for j in range(k):
            r = b"@read%d ch=%d\n" % (i, j) + seq[j].tobytes() + b"\n+\n" + qual[j].tobytes() + b"\n"
            rec.append(r)
            total += len(r)
            i += 1
    return b"".join(rec)


@pytest.fixture(scope="module")
def big():
    return big_fastq(17, 256 << 20)


def test_256mb_single_member_default_settings(ctx, big):
    data = big
    c = zlib.compressobj(1, zlib.DEFLATED, 31)
    blob = c.compress(data) + c.flush()
    status, st, got = inflate(ctx, blob, len(data))
    assert status == capi.FL_GUNZIP_OK and st[1] > 1 and st[0] == 1, st
    assert got == data


def test_large_file_with_a_bad_crc_declines(ctx, big):
    data = big
    c = zlib.compressobj(1, zlib.DEFLATED, 31)
    blob = bytearray(c.compress(data[:64 << 20]) + c.flush())
    blob[-6] ^= 0x10
    status, _, _ = inflate(ctx, bytes(blob), 64 << 20)
    assert status == capi.FL_GUNZIP_DECLINED


def test_too_little_device_memory_declines(ctx):
    blob = gc.deflate_gzip(b"@r\nACGT\n+\nIIII\n" * 1000)
    status, _, _ = inflate(ctx, blob, 1 << 20, 16384, 1000)
    assert status == capi.FL_GUNZIP_DECLINED

"""BGZF compression on the device (fl_bgzf_compress / fl_bgzf_compress_device): what any gzip reader inflates must be the
input byte for byte, the members must be well-formed BGZF, the output deterministic, the ratio close to zlib level 1's on
the same blocks, and a context's scoring results untouched by a compress call."""
import gzip
import os
import zlib

import numpy as np
import pytest

from tests import bgzf_util as bu
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from filtlong_b200 import api
    c = api.Context()
    yield c
    c.close()


def wgsim_fixture():
    return gzip.open(os.path.join(util.REF_FIXTURES, "test_reference_1_first1500.fastq.gz")).read()


def check_round_trip(ctx, data, eof=True):
    out = ctx.bgzf_compress(data, append_eof=eof)
    assert gzip.decompress(out) == data
    body = out[:-28] if eof else out
    if eof:
        assert out[-28:] == bu.EOF_MEMBER
    ms = bu.members(body)
    assert len(ms) == (len(data) + bu.BLOCK - 1) // bu.BLOCK
    for off, size, isize in ms:
        assert size <= 65536 and isize <= bu.BLOCK
        d = zlib.decompressobj(-15)
        assert len(d.decompress(body[off + 18:off + size - 8])) == isize and d.eof
    assert sum(m[2] for m in ms) == len(data)
    return out


@pytest.mark.parametrize("size", [0, 1, 65279, 65280, 65281, 10 * 65280 + 17])
@pytest.mark.parametrize("kind", ["random", "repeat", "fastq", "fasta"])
def test_round_trip_sizes_and_contents(ctx, size, kind):
    rng = np.random.default_rng(size + len(kind))
    if kind == "random":
        data = rng.integers(0, 256, size=size, dtype=np.uint8).tobytes()
    elif kind == "repeat":
        data = b"I" * size
    else:
        data = bu.fastq_corpus(rng, size, lo=300, hi=800, fasta=kind == "fasta")[:size]
    out = check_round_trip(ctx, data)
    assert ctx.bgzf_compress(data) == out                              # deterministic
    if kind == "random" and size:
        assert len(out) <= len(data) + 31 * len(bu.members(out[:-28])) + 28   # stored blocks when nothing compresses


def test_round_trip_reference_fixtures(ctx):
    for name in sorted(os.listdir(util.REF_FIXTURES)):
        p = os.path.join(util.REF_FIXTURES, name)
        data = open(p, "rb").read()
        check_round_trip(ctx, data)
        if name.endswith(".gz"):
            check_round_trip(ctx, gzip.decompress(data))
    out = ctx.bgzf_compress(b"", append_eof=False)
    assert out == b""


def test_round_trip_200mb_and_device_buffers(ctx):
    import torch
    rng = np.random.default_rng(3)
    part = bu.fastq_corpus(rng, 20_000_000, mean_len=10000)
    data = (part * 10)[:200_000_000]
    out = check_round_trip(ctx, data)
    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    cap = len(out)
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = ctx.bgzf_compress_device(d_in, len(data), d_out, cap)
    assert n == len(out) and bytes(d_out[:n].cpu().numpy()) == out
    assert ctx.bgzf_compress_device(d_in, len(data), d_out, cap - 1) is None   # FL_ERANGE when one byte short
    torch.cuda.synchronize()


def test_output_buffer_too_small_is_erange(ctx):
    from filtlong_b200 import capi
    import ctypes as C
    data = bu.fastq_corpus(np.random.default_rng(4), 300_000, lo=300, hi=800)
    full = ctx.bgzf_compress(data)
    src = np.frombuffer(data, np.uint8)
    out = np.zeros(len(full) - 1, np.uint8)
    n = C.c_uint64()
    rc = ctx.L.fl_bgzf_compress(ctx.h, capi.ptr(src), src.size, capi.ptr(out), out.size, 1, C.byref(n))
    assert rc == capi.FL_ERANGE and n.value == len(full)
    assert int(ctx.L.fl_bgzf_bound(0)) == 28 and int(ctx.L.fl_bgzf_bound(65281)) == 2 * 65311 + 28


CORPORA = {
    "long_reads": lambda rng: bu.fastq_corpus(rng, 8_000_000, mean_len=10000),
    "short_reads": lambda rng: bu.fastq_corpus(rng, 8_000_000, lo=300, hi=800),
    "wgsim_fixture": lambda rng: wgsim_fixture(),
    "fasta": lambda rng: bu.fastq_corpus(rng, 8_000_000, lo=300, hi=5000, fasta=True),
}


@pytest.mark.parametrize("corpus", sorted(CORPORA))
def test_ratio_within_5_percent_of_zlib_level_1(ctx, corpus):
    data = CORPORA[corpus](np.random.default_rng(21))
    ours = len(ctx.bgzf_compress(data, append_eof=False))
    theirs = len(bu.zlib_bgzf(data, 1))
    assert ours <= 1.05 * theirs, (corpus, ours / len(data), theirs / len(data))


def test_compress_leaves_scored_reads_alone():
    from filtlong_b200 import api
    rng = np.random.default_rng(9)
    reads = [(util.rand_seq(rng, int(rng.integers(200, 3000))), None) for _ in range(200)]
    reads = [(s, util.rand_qual(rng, len(s))) for s, _ in reads]
    ctx, _ = api.score_and_filter(reads, api.make_params(keep_percent=70.0))
    try:
        before = ctx.row_results()
        data = bu.fastq_corpus(rng, 3_000_000, lo=300, hi=800)
        assert gzip.decompress(ctx.bgzf_compress(data)) == data
        after = ctx.row_results()
        for k in before:
            assert np.array_equal(before[k], after[k]), k
    finally:
        ctx.close()

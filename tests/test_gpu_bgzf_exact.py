"""The BGZF compressor's bytes, member for member, against the exact model of tests/bgzf_model.py: the designed blocks
(together in one call and one per call), the first blocks of natural corpora, device input at every misalignment, and
the blocks around the seam between two launches of 2,048 blocks."""
import zlib

import numpy as np
import pytest

from tests import bgzf_model as bm
from tests import bgzf_util as bu
from tests.test_bgzf import CORPORA

pytestmark = pytest.mark.gpu

CHUNK = 2048                      # blocks per launch of k_bgzf_deflate


@pytest.fixture(scope="module")
def ctx():
    from filtlong_b200 import api
    c = api.Context()
    yield c
    c.close()


def assert_members_equal(got, want, first_block=0):
    """Equal bytes; else the first differing member and its first differing byte."""
    if got == want:
        return
    gm, wm = bu.members(got), bu.members(want)
    for i, (g, w) in enumerate(zip(gm, wm)):
        a, b = got[g[0]:g[0] + g[1]], want[w[0]:w[0] + w[1]]
        if a != b:
            k = next((j for j in range(min(len(a), len(b))) if a[j] != b[j]), min(len(a), len(b)))
            pytest.fail("block %d: member of %d bytes, the model's %d; first difference at byte %d (%s vs %s)"
                        % (first_block + i, len(a), len(b), k, a[k:k + 8].hex(), b[k:k + 8].hex()))
    pytest.fail("%d members, the model gives %d" % (len(gm), len(wm)))


def test_designed_blocks_in_one_call(ctx):
    full = [bm.designed(n)[0] for n in sorted(bm.DESIGNS) if len(bm.designed(n)[0]) == bm.BLOCK]
    data = b"".join(full) + bm.designed("last_130")[0]
    want = b"".join(bm.member(b)[0] for b in full) + bm.member(bm.designed("last_130")[0])[0]
    assert_members_equal(ctx.bgzf_compress(data, append_eof=False), want)


@pytest.mark.parametrize("name", sorted(bm.DESIGNS))
def test_designed_block_alone(ctx, name):
    block = bm.designed(name)[0]
    assert_members_equal(ctx.bgzf_compress(block, append_eof=False), bm.member(block)[0])


@pytest.mark.parametrize("corpus", sorted(CORPORA))
def test_first_blocks_of_corpora(ctx, corpus):
    data = CORPORA[corpus](np.random.default_rng(21))[:10 * bm.BLOCK]
    assert_members_equal(ctx.bgzf_compress(data, append_eof=False), bm.model_bgzf(data))


def test_unaligned_device_input(ctx):
    """The byte-wise load of a block that does not start 16-byte aligned. Each offset compresses other bytes, and on the
    device first, so no block's bytes are left over in shared memory from the call before."""
    import torch
    base = CORPORA["short_reads"](np.random.default_rng(8))[:2 * bm.BLOCK + 777]
    assert_members_equal(ctx.bgzf_compress(base, append_eof=False), bm.model_bgzf(base))
    d = torch.zeros(len(base) + 16, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(int(ctx.L.fl_bgzf_bound(len(base))), dtype=torch.uint8, device="cuda")
    for off in range(1, 16):
        data = base[off * 4099:] + base[:off * 4099]
        d.zero_()
        d[off:off + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        src = d[off:]
        assert src.data_ptr() % 16 == off % 16
        n = ctx.bgzf_compress_device(src, len(data), d_out, d_out.numel(), append_eof=False)
        got = bytes(d_out[:n].cpu().numpy())
        assert got == ctx.bgzf_compress(data, append_eof=False), off
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def long_reads():
    part = bu.fastq_corpus(np.random.default_rng(3), 20_000_000, mean_len=10000)
    n = CHUNK * bm.BLOCK + bm.BLOCK + 1
    return (part * (n // len(part) + 1))[:n]


@pytest.mark.parametrize("extra", [-1, 0, 1, bm.BLOCK + 1])
def test_seam_between_launches(ctx, long_reads, extra):
    n = CHUNK * bm.BLOCK + extra
    data = long_reads[:n]
    out = ctx.bgzf_compress(data, append_eof=False)
    ms = bu.members(out)
    assert len(ms) == (n + bm.BLOCK - 1) // bm.BLOCK
    lo = CHUNK - 3
    assert_members_equal(out[ms[lo][0]:], bm.model_bgzf(data[lo * bm.BLOCK:]), lo)      # blocks 2,045 to 2,049
    for i, (off, size, isize) in enumerate(ms):          # every member inflates to its block
        z = zlib.decompressobj(-15)
        assert z.decompress(out[off + 18:off + size - 8]) == data[i * bm.BLOCK:i * bm.BLOCK + isize] and z.eof, i
    assert sum(m[2] for m in ms) == n

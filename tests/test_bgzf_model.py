"""CPU checks of the exact BGZF model (tests/bgzf_model.py) that tests/test_gpu_bgzf_exact.py holds the kernel to: its
members inflate to their blocks, the designed blocks reach what they are built for, and its parse keeps to the rules."""
import zlib

import numpy as np
import pytest

from tests import bgzf_model as bm
from tests import bgzf_util as bu


def inflate_member(m, block):
    assert m[:16] == bm.HEADER and int.from_bytes(m[16:18], "little") == len(m) - 1
    d = zlib.decompressobj(-15)
    assert d.decompress(m[18:-8]) == block and d.eof and d.unused_data == b""
    assert m[-8:] == (zlib.crc32(block) & 0xffffffff).to_bytes(4, "little") + len(block).to_bytes(4, "little")


@pytest.mark.parametrize("name", sorted(bm.DESIGNS))
def test_designed_block_reaches_its_path_and_inflates(name):
    block, st = bm.designed(name)
    assert bm.DESIGNS[name][1](block, st), name
    m, st2 = bm.member(block)
    inflate_member(m, block)
    assert len(m) == (st["stored_size"] if st["stored"] else st["dyn_size"])
    assert st2["tokens"] == st["tokens"]


def test_coverage_of_the_designs():
    st = {n: bm.designed(n)[1] for n in bm.DESIGNS}
    # each tree reaches its length limit through fl_huff_lengths_sorted's limiting step
    assert any(s["free_depth"][0] > 15 and s["max_len"][0] == 15 for s in st.values())     # literal/length
    assert any(s["free_depth"][1] > 15 and s["max_len"][1] == 15 for s in st.values())     # distance
    assert any(s["free_depth"][2] > 7 and s["max_len"][2] == 7 for s in st.values())       # code lengths
    assert max(s["hlit"] for s in st.values()) == 281 and max(s["hdist"] for s in st.values()) == 30
    assert any(s["dummies"]["dist"] and len(s["dist_used"]) == 1 and s["dist_used"][0] == 0 for s in st.values())
    assert any(s["dummies"]["dist"] and len(s["dist_used"]) == 1 and s["dist_used"][0] > 0 for s in st.values())
    assert any(s["dummies"]["dist"] and not s["dist_used"] for s in st.values())
    diffs = {s["dyn_size"] - s["stored_size"] for s in st.values()}
    assert {-1, 0, 1} <= diffs
    sizes = {len(bm.designed(n)[0]) for n in bm.DESIGNS}
    assert {1, 2, 3, 4, 5, 127, 128, 129, 130, bm.BLOCK} <= sizes
    # a run of four equal non-zero code lengths is coded as the length and a 16 (three repeats)
    assert any(s["clhist"][16] for s in st.values())


@pytest.mark.parametrize("kind", ["fastq", "fasta"])
def test_model_members_inflate_on_corpora(kind):
    rng = np.random.default_rng(71)
    data = bu.fastq_corpus(rng, 1_000_000, mean_len=10000) if kind == "fastq" else \
        bu.fastq_corpus(rng, 1_000_000, lo=300, hi=5000, fasta=True)
    out = bm.model_bgzf(data)
    ms = bu.members(out)
    assert len(ms) == (len(data) + bm.BLOCK - 1) // bm.BLOCK
    for i, (off, size, _) in enumerate(ms):
        inflate_member(out[off:off + size], data[i * bm.BLOCK:(i + 1) * bm.BLOCK])
    # the natural ratio stays near zlib level 1's on the same blocks
    assert len(out) <= 1.05 * len(bu.zlib_bgzf(data, 1))


def test_parse_keeps_to_the_rules():
    rng = np.random.default_rng(5)
    for t in range(300):
        n = int(rng.integers(1, 700))
        alphabet = [2, 3, 4, 16, 256][t % 5]
        block = bytes(rng.integers(0, alphabet, size=n, dtype=np.uint8))
        cand = bm.candidates(block)
        covered = 0
        for p, d, L in bm.parse(block, cand):
            assert p == covered
            covered += L
            if not d:
                assert L == 1
                continue
            seg_end = min((p // bm.SEG + 1) * bm.SEG, n)
            assert 3 <= L <= min(seg_end - p, 258) and d <= min(p, bm.WINDOW)
            assert block[p - d:p - d + L] == block[p:p + L] if d >= L else \
                all(block[i] == block[i - d] for i in range(p, p + L))
            assert p + L == seg_end or block[p + L] != block[p + L - d]     # greedy: as long as the bytes agree
        assert covered == n
        for p, d in enumerate(cand):                                          # a candidate's four bytes agree
            assert not d or (p + 4 <= n and block[p - d:p - d + 4] == block[p:p + 4])

"""The --trim_q model (tests/qtrim_model.py) on the CPU: rows() against the pinned oracle's k-mer mode, where the
same rules run on "in a reference 16-mer", and good_mask() against its definition."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import qtrim_model as qm
from tests import util

FWD = np.zeros(256, dtype=np.uint64)
for ch, code in zip(b"CcGgTt", (1, 1, 2, 2, 3, 3)):
    FWD[ch] = code


def kmer_mask(seq: bytes, kmers) -> np.ndarray:
    """read.cpp:43-58: bases covered by a forward 16-mer of the read that is in the set"""
    L = len(seq)
    mask = np.zeros(L, dtype=bool)
    if L < 16:
        return mask
    codes = FWD[np.frombuffer(seq, dtype=np.uint8)]
    k = np.zeros(L - 15, dtype=np.uint64)
    for j in range(16):
        k = (k << np.uint64(2)) | codes[j:j + L - 15]
    hit = {int(x): (int(x) in kmers) for x in np.unique(k)}
    for s in np.nonzero([hit[int(x)] for x in k])[0]:
        mask[s:s + 16] = True
    return mask


@pytest.fixture(scope="module")
def kmer_case():
    rng = np.random.default_rng(41)
    genome = util.rand_seq(rng, 30000)
    reads = util.long_reads(rng, genome, 60, max_len=4000, junk_frac=0.8)
    k = orc.Kmers()
    k.add_assembly([genome[:12000], genome[15000:27000]])
    masks = [kmer_mask(s, k) for _, s, _ in reads]
    return reads, k, masks


@pytest.mark.parametrize("trim,split", [(True, None)] + [(t, s) for t in (False, True) for s in (1, 16, 31, 32, 33, 500)])
def test_rows_match_the_oracle_in_kmer_mode(kmer_case, trim, split):
    reads, k, masks = kmer_case
    op = orc.make_params(trim=trim, split=split, min_length=1)
    sc = orc.score([(s, q) for _, s, q in reads], op, k)
    n_children = 0
    for i, ((_, seq, _), m) in enumerate(zip(reads, masks)):
        got = qm.rows(m, len(seq), trim, split)
        p = sc.parents[i]
        assert (got["first"], got["last"]) == (p.first, p.last), i
        assert got["bad"] == [tuple(b) for b in sc.bad[i]], i
        assert got["children"] == [(c.start, c.end) for c in sc.children[i]], i
        n_children += len(got["children"])
    assert n_children > 0


def test_good_mask_matches_its_definition_on_random_qualities():
    rng = np.random.default_rng(5)
    for _ in range(400):
        L = int(rng.integers(0, 90))
        Q = int(rng.integers(1, 94))
        # mostly around the threshold, so that runs of every length occur
        q = np.clip(rng.integers(Q + 33 - 3, Q + 33 + 4, size=L), 0, 255).astype(np.uint8).tobytes()
        assert np.array_equal(qm.good_mask(q, Q), qm.good_mask_brute(q, Q)), (Q, q)


@pytest.mark.parametrize("name,qual,Q", qm.crafted(), ids=[c[0] for c in qm.crafted()])
def test_good_mask_on_crafted_reads(name, qual, Q):
    got = qm.good_mask(qual, Q)
    assert np.array_equal(got, qm.good_mask_brute(qual, Q))
    if name == "run of 15" or name.startswith("length 1"):
        assert got.sum() == (16 if name == "length 16" else 0)
    if name == "run of 16":
        assert list(np.nonzero(got)[0]) == list(range(40, 56))


def test_derived_reads_name_the_children_and_keep_the_comment():
    lo, hi = b"#", b"5"
    qual = hi * 20 + lo * 40 + hi * 30 + lo * 5
    seq = b"A" * len(qual)
    out = qm.derived_reads([("r1", b"c=1", seq, qual), ("r2", b"", seq[:10], lo * 10)], 20, True, 30)
    assert [(n, c, len(s)) for n, c, s, _ in out] == [("r1_1-20", b"c=1", 20), ("r1_61-90", b"c=1", 30), ("r2", b"", 10)]
    assert qm.fastq_bytes(out[:1]) == b"@r1_1-20 c=1\n" + b"A" * 20 + b"\n+\n" + hi * 20 + b"\n"

"""The designed contigs of tests/kmer_build_design.py and the one-copy build model of tests/kmer_build_model.py, checked
without a GPU: the model is the oracle's set on every design (the oracle is pinned to the reference) and a brute-force
string build's; the designs tell the model apart from two wrong builds by many 16-mers; and every seam class, offset
and byte class is placed (so that a later edit cannot quietly thin tests/test_gpu_kmer_build.py out)."""
import collections
import functools

import numpy as np

from oracle import oracle as orc
from tests import kmer_build_design as kd
from tests import kmer_build_model as kbm

D = kd.design()


@functools.lru_cache(maxsize=None)
def model():
    return kbm.build(D.contigs)


def test_model_equals_the_oracle():
    ok = orc.Kmers()
    ok.add_assembly(D.contigs)
    members, n, bases = model()
    assert np.array_equal(members, ok.dump())
    assert n == len(D.contigs)
    assert bases == sum(len(s) for s in D.contigs if len(s) >= 16)
    for w in kd.WIDTHS:
        extra, _, _ = kd.wrapped_extra(w)
        ok = orc.Kmers()
        ok.add_assembly(extra)
        assert np.array_equal(kbm.build(extra)[0], ok.dump()), w


def test_model_equals_a_brute_force_build():
    """every contig under 1,100 bases (the short run, the fillers and every copy of the lengths around a step), and the
    wrapped-FASTA contigs of the narrowest widths"""
    sub = [s for s in D.contigs if len(s) < 1100] + kd.wrapped_extra(1)[0] + kd.wrapped_extra(7)[0]
    assert sum(len(s) for s in sub) > 1000000
    assert np.array_equal(kbm.build(sub)[0], kbm.brute_force(sub))
    assert kbm.build([b"ACGTN" * 4])[0].tolist() == kbm.brute_force([b"ACGTN" * 4]).tolist()


# 16-mers by which each wrong build's set differs from the model's on the design (the design gives about 0.6 M each way
# for the first and 1.2 M missing for the second): a GPU build with either bug could not match.
WRONG_DIFFER_AT_LEAST = dict(n_complemented=500000, skipping_other_windows=1000000)


def test_the_designs_tell_the_wrong_builds_apart():
    members = model()[0]
    for name, build in (("n_complemented", kbm.build_n_complemented), ("skipping_other_windows", kbm.build_skipping_other_windows)):
        wrong = build(D.contigs)[0]
        diff = len(np.setxor1d(wrong, members, assume_unique=True))
        print("%s: %d 16-mers differ" % (name, diff))
        assert diff >= WRONG_DIFFER_AT_LEAST[name], name
    # and on the wrapped-FASTA contigs of each width alone
    for w in kd.WIDTHS:
        extra = kd.wrapped_extra(w)[0]
        assert len(np.setxor1d(kbm.build_n_complemented(extra)[0], kbm.build(extra)[0])) >= 100, w


def test_every_seam_offset_and_byte_class_is_placed():
    assert len(kd.OTHER_BYTES) == 25                            # N R Y K M S W B D H V in both cases, . - *
    per = collections.Counter()
    for (cls, d, b), n in D.placements.items():
        assert d in kd.offsets_of(cls)
        per[(cls, d)] += 1
    for cls in kd.SEAM_CLASSES:
        for d in kd.offsets_of(cls):
            assert per[(cls, d)] == len(kd.OTHER_BYTES), (cls, d)
    times = collections.Counter()
    for (cls, d, b), n in D.placements.items():
        times[cls] = min(times.get(cls, n), n)
    # each (class, offset, byte) at least this often (the design gives start 3, end 2, lane 80, step 12, tile 1, pad 1)
    assert all(times[c] >= 1 for c in kd.SEAM_CLASSES)
    assert times["lane"] >= 50 and times["step"] >= 10
    # runs of 15, 16 and 17 non-ACGT bytes at every seam class, lower-case runs across seams
    for cls in kd.SEAM_CLASSES:
        for r in (15, 16, 17):
            assert D.runs.get((cls, r), 0) >= 5, (cls, r)
    assert D.lower_runs >= 1000
    # lengths around every seam, under 16 bases between long ones, and a run of thousands of 1 .. 40 bases
    lens = np.array([len(s) for s in D.contigs])
    for L in kd.LENGTHS:
        assert np.count_nonzero(lens == L) >= 32, L
    assert np.count_nonzero((lens > 0) & (lens < 16)) >= 1000
    assert np.count_nonzero((lens >= 1) & (lens <= 40)) >= 3000
    assert lens.max() > 24 * kd.TILE and D.long_contigs >= 16 and len(D.cuts) >= 30
    # the wrapped-FASTA contigs put non-ACGT bytes on both sides of over a hundred line ends at every width
    for w in kd.WIDTHS:
        _, last, first = kd.wrapped_extra(w)
        assert last >= 120 and first >= 120, w


def test_file_writers():
    c = [b"ACGTACG", b"", b"ACGTAC"]
    assert kd.fasta(c, 3) == b">contig_0\nACG\nTAC\nG\n>contig_1\n>contig_2\nACG\nTAC\n"
    assert kd.fasta(c) == b">contig_0\nACGTACG\n>contig_1\n>contig_2\nACGTAC\n"
    assert kd.fastq(c[:1], 5) == b"@contig_5\nACGTACG\n+\nIIIIIII\n"
    assert kd.chunks(list(range(5)), [1, 3]) == [[0], [1, 2], [3, 4]]

"""BASELINE config 1 and the known answers of the reference's own test suite (test/test_sort.py,
test_trim.py, test_split.py) on the committed fixture bytes, through the C ABI."""
import os

import pytest

from tests import util

FIX = util.REF_FIXTURES


def _fixture_reads(name):
    return [(s, q) for _, s, q in util.read_fastx(os.path.join(FIX, name))]


@pytest.mark.gpu
def test_baseline_config1_on_the_reference_fixture():
    """BASELINE configs[0]: test/test_sort.fastq --min_length 1 --keep_percent 90 -> target 13 500 bp,
    keeping 15 000 bp, all three reads out (SURVEY section 4); raw values are the survey's hex doubles."""
    from filtlong_b200 import api
    reads = _fixture_reads("test_sort.fastq")
    assert [len(s) for s, _ in reads] == [5000, 5000, 5000]
    ctx, summ = api.score_and_filter(reads, api.make_params(min_length=1, keep_percent=90.0))
    assert (summ.status, summ.target, summ.keeping) == (3, 13500, 15000)
    rows = ctx.row_results()
    assert [int(x) for x in rows["passed_final"]] == [1, 1, 1]
    want = [("0x1.6765056776ee5p+6", "0x1.656d069f0b576p+6"), ("0x1.8bebf07f8e0a2p+6", "0x1.8bd0b23c524bfp+6"),
            ("0x1.831476491630dp+6", "0x1.82b0ce9fc8fd7p+6")]
    for i, (m, w) in enumerate(want):
        assert rows["mean_q"][i] == float.fromhex(m) and rows["window_q"][i] == float.fromhex(w), i
    assert [round(float(x), 2) for x in rows["final_score"]] == [0.00, 70.70, 61.54]
    ctx.close()


@pytest.mark.gpu
def test_reference_known_answers_with_the_assembly_fixture():
    """test_sort / test_trim / test_split against test_reference.fasta: 199 964 16-mers, the score order
    1 > 3 > 2, the drifted window qualities 79.999999999999986 / 59.99.. / 19.99.., and the child names
    test_trim.py:74-112 / test_split.py:74-223 pin."""
    from filtlong_b200 import api
    asm = [s for _, s, _ in util.read_fastx(os.path.join(FIX, "test_reference.fasta"))]
    ctx, summ = api.score_and_filter(_fixture_reads("test_sort.fastq"), api.make_params(min_length=1, keep_percent=90.0), assembly=asm)
    assert ctx.kmers_count() == 199964
    rows = ctx.row_results()
    assert [round(float(x), 2) for x in rows["final_score"]] == [70.71, 0.00, 63.23]
    ctx.close()
    ctx, _ = api.score_and_filter(_fixture_reads("test_split.fastq"), api.make_params(min_length=1), assembly=asm)
    assert [repr(float(x)) for x in ctx.read_results()["window_q"][1:]] == ["79.99999999999999", "59.999999999999964", "19.99999999999993"]
    ctx.close()
    ctx, _ = api.score_and_filter(_fixture_reads("test_trim.fastq"), api.make_params(min_length=1, trim=True), assembly=asm)
    rows = ctx.row_results()
    spans = [(int(p), int(s) + 1, int(e)) for p, s, e in zip(rows["parent"], rows["start"], rows["end"])]
    assert spans == [(0, 1, 1300), (1, 21, 701), (2, 1, 970), (3, 13, 1885)]       # test_trim_2_21-701, _3_1-970, _4_13-1885
    ctx.close()
    ctx, _ = api.score_and_filter(_fixture_reads("test_split.fastq"), api.make_params(min_length=1, split=200), assembly=asm)
    rows = ctx.row_results()
    assert len(rows["parent"]) == 5 and int((rows["end"] - rows["start"]).sum()) == 11400   # test_split.py: --split 200 -> 5 reads, 11 400 bp
    ctx.close()

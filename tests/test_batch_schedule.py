"""The batch schedules of tests/test_gpu_batching.py (tests/batch_schedule.py), without a GPU: every schedule covers the
reads in order, each mode's schedules together cross every seam that mode has, and the read set holds what they cut at."""
import numpy as np
import pytest

from tests import batch_schedule as bs


@pytest.fixture(scope="module")
def data():
    return bs.read_set()


@pytest.mark.parametrize("mode", list(bs.MODES))
def test_every_mode_crosses_every_seam(data, mode):
    a = bs.attrs(data, mode)
    paths = bs.paths_of(mode)
    sch = bs.schedules(a, paths)
    got = set()
    for name, steps in sch.items():
        bs.check_cover(steps, len(data["reads"]))
        for st in steps:
            if st[0] == "batch":
                assert st[1] in paths, (name, st)
                assert st[1] == "push" or (a["length"][st[2]:st[3]] > 0).all(), (name, st)   # an empty read: push only
        got |= bs.seams_of(steps, a)
    need = bs.required_seams(a, paths)
    assert need <= got, need - got
    assert ("all_removed" in need) == bool(bs.MODES[mode].get("contam"))
    assert ("childless_next_to_many" in need) == ("split" in bs.MODES[mode]["kw"])
    assert bs.schedules(a, paths) == sch                                              # seeded: the same every time


def test_the_read_set_holds_its_edges(data):
    lengths = np.array([len(r[1]) for r in data["reads"]])
    assert 2_000_000 < lengths.sum() < 3_000_000 and bs.ALLOC_FLOOR < len(lengths) < 2000
    assert all(r[1] == r[1].upper() for r in data["reads"])
    for L in (0, 1, 15, 16, 17):
        assert (lengths == L).any(), L
    assert (lengths > 24576).sum() >= 3 and (lengths == 0).sum() == 1
    assert sum(b"N" in r[1] for r in data["reads"]) >= 3
    assert len({r[0] for r in data["reads"]}) == len(lengths)


@pytest.mark.parametrize("mode", ["trimq10_trim_split500", "trimq20_split1", "kmer_trim_split100"])
def test_reads_have_none_one_and_many_children(data, mode):
    k = bs.attrs(data, mode)["n_child"]
    assert (k == 0).any() and (k == 1).any() and (k > 100).any()


def test_contaminant_reads_on_both_sides_of_max_contam(data):
    for k in (16, 24):
        c = bs.contam_percentages(data, k)
        assert (c > bs.P_CONTAM).sum() > 20 and ((c > 0) & (c <= bs.P_CONTAM)).sum() > 10
    assert (bs.contam_percentages(data, 16) == bs.P_CONTAM).sum() >= 1              # exactly at max_contam: kept


def test_seams_of_names_what_it_sees():
    a = dict(length=np.array([5, 3, 100, 100, 0, 100]), n_child=np.array([0, 0, 0, 1500, 0, 2]),
             removed=np.array([False, False, True, True, False, False]))
    steps = [("batch", "push", 0, 0), ("batch", "push", 0, 2), ("batch", "push", 2, 2), ("observe", "counts"),
             ("batch", "push_bam", 2, 3), ("batch", "push", 3, 4), ("batch", "push", 4, 6)]
    assert bs.seams_of(steps, a) == {"empty:push", "short_only", "empty_push_after_push", "observe:counts",
                                     "after_deferred:push_bam", "all_removed", "childless_next_to_many"}
    n, F = 1200, bs.ALLOC_FLOOR
    flat = dict(length=np.ones(n, int), n_child=np.zeros(n, int), removed=np.zeros(n, bool))
    grow = [("batch", "push", 0, 1), ("batch", "push", 1, 2), ("batch", "push", 2, n)]
    assert {"grow_staging", "grow_arrays"} <= bs.seams_of(grow, flat)
    assert not {"grow_staging", "grow_arrays"} & bs.seams_of([("batch", "push", 0, 1), ("batch", "push", 1, F)], flat)
    assert "grow_arrays" not in bs.seams_of([("batch", "push", 0, F + 1), ("batch", "push", F + 1, n)], flat)
    many = dict(flat, n_child=np.full(n, 2))                 # rows pass the floor in the first batch: nothing grows later
    assert "grow_arrays" not in bs.seams_of([("batch", "push", 0, 600), ("batch", "push", 600, n)], many)

"""k-mer mode on designed hit masks (tests/kmer_masks.py): the reads and the 16-mer set are built so that the painted mask
is known exactly, and the three kernels of the mode meet the masks they are weakest on -- k_kmer_window's flagged-word
path (rows climbing through every binade, first windows on a tie binade, counts hovering at binade edges, window sizes
1 .. 15 and beyond 2^15), k_kmer_scan's seams between its fast, ballot and in-word paths, and k_probe_paint's carries
across lanes, 1024-base steps and 8192-base tiles. The oracle judges every value (test_gpu_parity.run_both / full_check:
per-read and per-row values bit-identical, rescale and selection exact)."""
import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import kmer_masks as km
from tests.test_gpu_parity import full_check, run_both

pytestmark = pytest.mark.gpu


def _run(real, opts, cap=4096):
    ctx, summ, sc, ok = run_both(real.reads, opts, assembly=real.runs, cap=cap)
    assert ctx.kmers_count() == len(ok) == len(real.members)
    full_check(ctx, summ, sc)
    return ctx


@pytest.mark.parametrize("ws", km.WINDOW_SIZES)
def test_window_on_designed_rows(ws):
    """every designed row as a whole read, and as a child row of one read cut by --split (with --trim): rows that start
    and end at every residue mod 32, with lengths ws, ws + 1, ws + 31 .. 33 and ws + 1024 +- 1"""
    whole, read, split, starts, rows = km.window_case(ws)
    real = km.realize(whole + [read], np.random.default_rng(ws))
    ctx = _run(real, dict(window_size=ws, keep_percent=90.0))
    ctx.close()
    ctx = _run(real, dict(window_size=ws, keep_percent=90.0, split=split, trim=True, min_window_q=10.0))
    rr, rw = ctx.read_results(), ctx.row_results()
    r0 = int(rr["row_start"][len(whole)])
    assert int(rr["n_child"][len(whole)]) == len(rows)
    assert list(rw["start"][r0:r0 + len(rows)]) == starts
    assert list(rw["end"][r0:r0 + len(rows)]) == [s + len(r) for s, r in zip(starts, rows)]
    ctx.close()


@pytest.mark.parametrize("trim", [False, True])
@pytest.mark.parametrize("split", km.SPLITS)
def test_scan_on_designed_zero_runs(split, trim):
    """zero runs of split - 1, split and split + 1 bases inside a word, across a word seam, ending in lane 0's word after a
    run open at the end of the previous step, and longer than a step; trim ranges that equal a bad range; hit-less reads
    around `split`; reads of 15 .. 33 bases; at --split 1 one 2 Mbase read with more than 100,000 children"""
    designs = km.scan_designs(split)
    cap = 4096
    if split == 1:
        designs = designs[:2] + [km.many_children(2000000, 1)] + designs[2:]
        cap = 2000000 // 17 + 8
    real = km.realize(designs, np.random.default_rng(100 + split))
    ctx = _run(real, dict(split=split, trim=trim, keep_percent=85.0), cap=cap)
    if split == 1:
        assert ctx.read_results()["n_child"][2] > 100000
    ctx.close()


PAINT_FLAVOURS = [("auto", {}), ("group", {"FL_FILTER_KIND": "22"}), ("pair", {"FL_FILTER_KIND": "26"}),
                  ("single", {"FL_FILTER_KIND": "18"}), ("two_bits", {"FL_FILTER_KIND": "2"}), ("no_filter", {"FL_FILTER": "0"}),
                  ("plain_bitmap", {"FL_ANCHOR": "0"})]


def test_paint_isolated_hits_at_seams(monkeypatch):
    """one 16-base hit at every start within 20 of a lane, step and tile seam and at the last start, pairs of hits
    1 .. 17 apart across each seam, reads of 8192 t + {-17 .. 17} bases: under every probe flavour, bit-identical to
    each other and to the oracle"""
    real = km.realize(km.paint_designs(), np.random.default_rng(5))
    opts = dict(keep_percent=90.0, trim=True, split=20, window_size=50)
    outs = {}
    for tag, env in PAINT_FLAVOURS:
        for k in ("FL_FILTER_KIND", "FL_FILTER", "FL_ANCHOR"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ctx = _run(real, opts)
        outs[tag] = {k: v.tobytes() for k, v in ctx.row_results().items()}
        info = ctx.kmers_probe_info()
        assert info["anchored"] == (tag != "plain_bitmap") and info["pre_filter"] == (tag != "no_filter")
        ctx.close()
    for tag, o in outs.items():
        assert o == outs["auto"], tag


def test_contaminant_percentages_are_the_design_popcount():
    """k_contam_reads counts the same painted mask: with the paint designs' 1-runs as the contaminant set, a read's
    percentage is 100 * popcount / L of its design, bit for bit"""
    real = km.realize(km.paint_designs(), np.random.default_rng(6))
    want = np.array([real.mean(i) for i in range(len(real.reads))])
    with api.Context(api.make_params(max_contam=0.5, keep_percent=90.0)) as ctx:
        ctx.contam_add(real.runs)
        assert ctx.contam_count() == len(real.members)
        ctx.push(api.HostBatch([r[0] for r in real.reads], [r[1] for r in real.reads], want_seq=True))
        pct, removed, counts = ctx.contam_results()
    assert np.array_equal(pct.view(np.uint64), want.view(np.uint64))
    assert np.array_equal(removed, want > 0.5) and counts["reads"] == int((want > 0.5).sum())

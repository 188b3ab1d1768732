"""The designed hit masks of tests/kmer_masks.py, checked without a GPU: every design is realized exactly (the reads
paint back to it under its 16-mer set), the oracle's raw mean, first / last base and bad ranges on the designed reads are
what the design says, and the window kernel's scalar model takes its flagged-word path on the window cases often
enough that tests/test_gpu_kmer_masks.py exercises it (so that a later edit cannot quietly make them event-free)."""
import ctypes as C
import struct

import numpy as np
import pytest

from oracle import oracle as orc
from tests import kmer_masks as km
from tests.test_kmer_window_model import model, pack  # noqa: F401  (the compiled model is a fixture)


def _bits(x):
    return struct.pack("<d", x)


def _realized_exactly(real):
    for d, (seq, _) in zip(real.designs, real.reads):
        assert np.array_equal(km.paint(seq, real.members), d)


def test_every_design_is_realized_exactly():
    rng = np.random.default_rng(1)
    n_designs = n_bases = 0
    cases = [km.paint_designs()] + [km.scan_designs(s) for s in km.SPLITS]
    for ws in (1, 17, 250, 470, 4097):
        whole, read, split, starts, rows = km.window_case(ws)
        cases.append(whole + [read])
    for designs in cases:
        real = km.realize(designs, rng)
        _realized_exactly(real)
        n_designs += len(designs)
        n_bases += sum(len(d) for d in designs)
    # the set is what an assembly of the 1-runs adds, in the oracle's own k-mer code
    ok = orc.Kmers()
    ok.add_assembly(real.runs)
    assert np.array_equal(ok.dump(), real.members)
    print("realized designs: %d reads, %d bases" % (n_designs, n_bases))


def test_design_builders_keep_their_promises():
    for ws in km.WINDOW_SIZES[:13]:
        whole, read, split, starts, rows = km.window_case(ws)
        assert all(km.is_design(d) for d in whole + [read])
        assert sorted({s % 32 for s in starts}) == list(range(32))
        assert sorted({(s + len(r)) % 32 for s, r in zip(starts, rows)}) == list(range(32))
        for s, r in zip(starts, rows):
            assert np.array_equal(read[s:s + len(r)], r) and r[0] and r[-1] and not read[s - 1]
        zs, ze = km.zero_runs_of(read)
        assert set(zip(zs[ze - zs >= split], ze[ze - zs >= split])) == \
            {(0, starts[0])} | {(s + len(r), t) for s, r, t in zip(starts, rows, starts[1:])} | {(starts[-1] + len(rows[-1]), len(read))}
    for c0 in km.tie_levels(250):
        assert 8 <= c0 <= 15
    assert km.tie_levels(250) == list(range(8, 16))
    assert 235 in km.edge_levels(470)
    assert len(km.many_children(2000000, 1).nonzero()[0]) // 16 > 100000


def _expected_bad(d, split, trim):
    """read.cpp:89-117 on a design: zero runs of at least `split`, then the trim ranges [0, first) / [last, L) unless
    they are already there"""
    L = len(d)
    zs, ze = km.zero_runs_of(d)
    bad = [(int(s), int(e)) for s, e in zip(zs, ze) if split is not None and e - s >= split]
    ones = np.nonzero(d)[0]
    first, last = (int(ones[0]), int(ones[-1]) + 1) if len(ones) else (-1, -1)
    if trim:
        if first > 0 and not (bad and bad[0] == (0, first)):
            bad.insert(0, (0, first))
        if last != -1 and last < L and not (bad and bad[-1] == (last, L)):
            bad.append((last, L))
    return first, last, bad


@pytest.mark.parametrize("trim", [False, True])
def test_oracle_values_follow_from_the_design(trim):
    rng = np.random.default_rng(2)
    checked = 0
    for split in km.SPLITS:
        real = km.realize(km.scan_designs(split), rng)
        ok = orc.Kmers()
        ok.insert(real.members)
        p = orc.make_params(split=split, trim=trim)
        sc = orc.score(real.reads, p, ok)
        for i, d in enumerate(real.designs):
            par = sc.parents[i]
            want = real.mean(i)
            assert _bits(par.mean_q) == _bits(want) or (want != want and par.mean_q != par.mean_q), (split, i)
            first, last, bad = _expected_bad(d, split, trim)
            assert (par.first, par.last) == (first, last), (split, i)
            assert sc.bad[i] == bad, (split, i)
            for ch in sc.children[i]:
                assert _bits(ch.mean_q) == _bits(100.0 * float(d[ch.start:ch.end].sum()) / (ch.end - ch.start))
            checked += 1
    print("oracle checked on %d designed reads" % checked)


# Flagged words (words the window kernel walks step by step, one irreversible step done with real double operations)
# that the model takes on the window cases of tests/test_gpu_kmer_masks.py, whole reads and child rows together. The
# cases give 743 in all and 7 .. 102 per window size; a builder edit that drops below these is caught here.
FLAGGED_AT_LEAST = dict(total=600, per_ws=5)


def test_window_cases_take_the_flagged_path(model):   # noqa: F811
    total, per_ws = 0, {}
    for ws in km.WINDOW_SIZES:
        whole, read, split, starts, rows = km.window_case(ws)
        n = 0
        items = [(d, 0, len(d)) for d in whole] + [(read, s, s + len(r)) for s, r in zip(starts, rows)]
        packed = {}
        for d, S, E in items:
            key = id(d)
            if key not in packed:
                packed[key] = pack(d)
            m = packed[key]
            ns = C.c_longlong()
            a = model.kmer_window_model(m.ctypes.data, S, E, ws, None, C.byref(ns))
            b = model.kmer_window_reference(m.ctypes.data, S, E, ws)
            assert a.hex() == b.hex(), (ws, S, E)
            n += ns.value
        per_ws[ws] = n
        total += n
    print("flagged words per window size:", per_ws, "total", total)
    assert total >= FLAGGED_AT_LEAST["total"]
    assert all(v >= FLAGGED_AT_LEAST["per_ws"] for v in per_ws.values()), per_ws

"""The scalar model of k_kmer_window (tests/models/kmer_window_model.c: the device algorithm of
filtlong_b200/csrc/fl_score.cu, word by word) against the reference recurrence itself (read.cpp:216-236 on
{0, 1} qualities) on random and adversarial hit masks: the window quality must come out bit for bit although
the model never walks a row base by base. CPU only."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("kw") / "libkw.so")
    subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "models", "kmer_window_model.c"), "-lm"],
                   check=True)
    L = C.CDLL(so)
    L.kmer_window_model.restype = C.c_double
    L.kmer_window_model.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    L.kmer_window_reference.restype = C.c_double
    L.kmer_window_reference.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    return L


def painted(rng, n, p_hit):
    """a mask as the probe kernel paints it: a hit at position i covers bases i .. i + 15"""
    cov = np.zeros(n + 16, dtype=np.int32)
    idx = np.nonzero(rng.random(n) < p_hit)[0]
    np.add.at(cov, idx, 1)
    np.add.at(cov, idx + 16, -1)
    return np.cumsum(cov)[:n] > 0


def read_like(rng, n, err):
    """errors at rate err; a 16-mer hits if it holds no error; covered = union of the hitting 16-mers"""
    e = (rng.random(n) < err).astype(np.int32)
    ok = np.convolve(e, np.ones(16, dtype=np.int32))[15:n] == 0
    cov = np.zeros(n + 16, dtype=np.int32)
    idx = np.nonzero(ok)[0]
    np.add.at(cov, idx, 1)
    np.add.at(cov, idx + 16, -1)
    return np.cumsum(cov)[:n] > 0


def pack(bits):
    b = np.zeros(((len(bits) + 31) // 32 + 2) * 32, dtype=np.uint8)
    b[:len(bits)] = bits
    return np.ascontiguousarray(np.packbits(b.reshape(-1, 32)[:, ::-1], axis=1).view(">u4").reshape(-1).astype(np.uint32))


def make_mask(rng, kind, n):
    if kind == 0:
        return rng.random(n) < rng.uniform(0.01, 0.99)
    if kind == 1:
        return painted(rng, n, rng.uniform(0.001, 0.3))
    if kind == 2:
        return read_like(rng, n, rng.uniform(0.0, 0.2))
    if kind == 3:                                   # perfect read with a few holes: w sits on the binade edge 1.0
        bits = np.ones(n, dtype=bool)
        bits[rng.integers(0, n, size=rng.integers(0, 20))] = False
        return bits
    if kind == 4:                                   # hovers around half coverage: the edge 0.5, over and over
        blk = int(rng.integers(1, 40))
        return ((np.arange(n) // blk) % 2 == 0) ^ (rng.random(n) < 0.02)
    if kind == 5:                                   # one island in junk: counts pass through every binade
        bits = np.zeros(n, dtype=bool)
        s = int(rng.integers(0, n))
        bits[s:s + int(rng.integers(1, 3000))] = True
        return bits
    bits = read_like(rng, n, rng.uniform(0.02, 0.16))            # a read with a chimeric junk block
    j = int(rng.integers(0, n))
    bits[j:j + int(rng.integers(100, 3000))] = False
    return bits


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_model_equals_reference_recurrence(model, seed):
    rng = np.random.default_rng(seed)
    steps = slow = 0
    for it in range(350):
        n = int(rng.integers(300, 40000))
        ws = [250, 250, 250, 256, 100, 17, 1000][it % 7] if it % 3 else int(rng.integers(16, 600))
        m = pack(make_mask(rng, it % 7, n))
        for S, E in ((0, n), (int(rng.integers(0, n // 2)), int(rng.integers(n // 2, n + 1)))):
            if E <= S:
                continue
            ns = C.c_longlong()
            a = model.kmer_window_model(m.ctypes.data, S, E, ws, None, C.byref(ns))
            b = model.kmer_window_reference(m.ctypes.data, S, E, ws)
            assert struct.pack("<d", a) == struct.pack("<d", b), (it, n, ws, S, E, a.hex(), b.hex())
            steps += max(E - S - ws, 0)
            slow += ns.value
    assert steps > 5 * 10 ** 6


def test_the_case_that_breaks_a_naive_anchor(model):
    """ws = 470, first window exactly half full: w0 = 0.5 sits ON a binade floor; one step up and one down do
    not return to 0.5 (the subtraction falls through the floor onto the finer grid), so the value at that level
    depends on whether the chain has been above it -- the 'record level next to an edge' rule."""
    ws, n = 470, 3000
    bits = np.zeros(n, dtype=bool)
    bits[0:ws:2] = True                                  # 235 of the first 470
    bits[ws] = True                                      # step 0: a one enters (out bit 0 is 1 -> count stays), then play around the level
    bits[ws + 1:ws + 40:3] = True
    m = pack(bits)
    a = model.kmer_window_model(m.ctypes.data, 0, n, ws, None, None)
    b = model.kmer_window_reference(m.ctypes.data, 0, n, ws)
    assert a.hex() == b.hex()


def test_realistic_masks_are_nearly_event_free(model):
    """On read-like masks with ws = 250 the flagged words (walked with true double operations) are a small
    minority: the kernel's cost is the parallel count arithmetic."""
    rng = np.random.default_rng(9)
    for err, bound in ((0.03, 0.002), (0.06, 0.002), (0.09, 0.02), (0.12, 0.08)):
        bits = read_like(rng, 400000, err)
        m = pack(bits)
        ns = C.c_longlong()
        a = model.kmer_window_model(m.ctypes.data, 0, len(bits), 250, None, C.byref(ns))
        assert a.hex() == model.kmer_window_reference(m.ctypes.data, 0, len(bits), 250).hex()
        assert ns.value / (len(bits) / 32) <= bound, (err, ns.value)


def _family(rng, fam, n, ws):
    from tests import kmer_masks as km
    if fam == "opened":                                  # the model kinds made paintable: every 1-run >= 16 bases
        return km.opening(make_mask(rng, int(rng.integers(0, 7)), n))
    if fam == "rising":                                  # sparse or empty first window, then gaps shrinking to full coverage
        return km.rising(rng, n, ws, int(rng.integers(0, 2)))
    return make_mask(rng, int(rng.integers(0, 7)), n)


@pytest.mark.parametrize("ws", list(range(1, 16)) + [32767, 32768, 32769, 65536, 100000])
def test_model_at_tiny_and_huge_window_sizes(model, ws):
    """ws 1..15 (rq = 1, 1/2, 1/3 ...: almost no grid below the count's binade) and ws >= 2^15 (more than 16 binade
    edges, the most a window size below 2^31 needs is 33), on the model's mask kinds, their openings and rising rows."""
    rng = np.random.default_rng(ws)
    slow = 0
    for it in range(45 if ws < 16 else 6):
        fam = ("raw", "opened", "rising")[it % 3]
        n = int(rng.integers(ws + 1, ws * (20 if ws < 16 else 3) + 3000))
        m = pack(_family(rng, fam, n, ws))
        for S, E in ((0, n), (int(rng.integers(0, n // 2)), int(rng.integers(n // 2, n + 1)))):
            if E <= S:
                continue
            ns = C.c_longlong()
            a = model.kmer_window_model(m.ctypes.data, S, E, ws, None, C.byref(ns))
            b = model.kmer_window_reference(m.ctypes.data, S, E, ws)
            assert struct.pack("<d", a) == struct.pack("<d", b), (it, fam, n, ws, S, E, a.hex(), b.hex())
            slow += ns.value
    assert slow > 0


def test_a_row_hovering_at_half_with_more_than_16_edges(model):
    """ws = 100000 has 18 binade edges; a row whose count hovers around ws / 2 after a long climb needs the edge at
    0.5 (the model once kept only 16 edges and came out one ulp off here)."""
    from tests import kmer_masks as km
    rng = np.random.default_rng(3)
    ws = 100000
    for _ in range(4):
        bits = km.hover(rng, 4 * ws, ws, ws // 2, False)
        m = pack(bits)
        a = model.kmer_window_model(m.ctypes.data, 0, len(bits), ws, None, None)
        assert a.hex() == model.kmer_window_reference(m.ctypes.data, 0, len(bits), ws).hex()

"""k_phred_sum's loads run one step ahead of its sums: each lane loads its 16 bytes of step t + 1 while it sums step t, a
lane whose chunk starts at or beyond the read's end loads nothing and keeps the bytes of the step before for the tail mask
to hide, and the crossing replay of a step re-reads its table entries. The cases here aim at the seams of that walk:
  * read lengths one base around 16-byte chunk boundaries of the first step, around 1 to 4 whole steps past the head,
    and around chunk boundaries of later steps: reads of one step, and last steps in which some lanes load and others
    do not;
  * thousands of reads of one length (more than the resident warps, so a warp scores several in a row), alternately of
    high and low quality: bytes of a read or step before, left unmasked, would change the sum;
  * a byte that ties in the running sum's binade, a byte outside the Phred range and a binade crossing, each placed in
    the first steps (the one loaded before the walk and those loaded inside it) and in the last step: the careful and
    serial modes at the walk's edges.
Every read must match the oracle bit for bit. The CPU test checks that the designed reads do reach those modes, on the
lattice model of the kernel (tests/test_phred_lattice_model.py)."""
import numpy as np
import pytest

from tests import util
from tests.test_gpu_parity import full_check, run_both
from tests.test_phred_lattice_model import expo, model_sum, model_window, tables, tie_info

TILE = 512
STEPS = 4                                     # the first steps the designed reads aim at
WINDOWS = [250, 16, 129, 200]
# backgrounds for designed reads, low to high quality; every window of them stays above k_phred_win's 0.5 bound
BACKGROUNDS = [b"$$%", b"$%", b"%", b"%&", b"&", b"'", b"(", b"+", b"5"]


def head(ws):
    return (ws + 15) & ~15


def pipeline_lengths(ws):
    H = head(ws)
    out = []
    for k in range(1, 33):                                        # lanes of the first step that copy, or not
        out += [H + 16 * k + d for d in (-1, 0, 1)]
    for m in (1, 2, 3, 4, 7):
        for k in (0, 1, 7, 31):
            out += [H + TILE * m + 16 * k + d for d in (-1, 0, 1)]
    return sorted({L for L in out if L > ws})


def _qual(rng, L):
    return util.rand_qual(rng, L, mean_q=rng.uniform(5, 30))


@pytest.mark.gpu
@pytest.mark.parametrize("ws", WINDOWS)
def test_lengths_around_pipeline_seams(ws):
    rng = np.random.default_rng(7100 + ws)
    reads = [(b"A" * L, _qual(rng, L)) for L in pipeline_lengths(ws)]
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [1, 5, 17, 100, 511])
def test_stale_bytes_across_reads(tail):
    """6000 reads of one length whose last step holds `tail` bases, alternately Q40 and Q5 (and a few random ones): with
    more reads than resident warps most warps score several, and the lanes past the end of the last step hold bytes of
    the step before, which the tail mask must hide"""
    ws = 250
    L = head(ws) + TILE * 3 + tail
    rng = np.random.default_rng(7200 + tail)
    reads = []
    for i in range(6000):
        if i % 50 == 49:
            q = _qual(rng, L)
        else:
            q = (b"I" if i % 2 else b"&") * L
        reads.append((b"A" * L, q))
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=50.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()


# ---- designed reads: a tie, a byte outside the Phred range, a binade crossing at given steps ----

def _steps(ws, L):
    return -(-(L - head(ws)) // TILE)


def _step_counts(qs, ws, model):
    """per step of k_phred_sum: how many crossing replays and serial walks the lattice model made there"""
    q, tie_any, tie_chars = model
    out, prev = [], (0, 0)
    for t in range(_steps(ws, len(qs))):
        st = {"fast": 0, "cross": 0, "serial": 0}
        model_sum(qs[:min(len(qs), head(ws) + TILE * (t + 1))], ws, q, tie_any, tie_chars, st)
        out.append((st["cross"] - prev[0], st["serial"] - prev[1]))
        prev = (st["cross"], st["serial"])
    return out


def _window_ok(qs, ws, q, a):
    return model_window(qs, ws, q, a) is not None


def _targets(ws, L):
    """the first STEPS steps and the last step of a read of length L, those that exist"""
    n = _steps(ws, L)
    return sorted({t for t in list(range(STEPS)) + [n - 1] if 0 <= t < n})


def LENGTHS(H):
    return [H + TILE * STEPS + 200, H + TILE * (STEPS - 1) + 40, H + TILE + 300]


def designed_reads(ws):
    """[(kind, step, qualities)] for kind in tie / nan / cross"""
    q, a = tables(ws)
    tie_any, tie_chars = tie_info(q)
    model = (q, tie_any, tie_chars)
    H = head(ws)
    out = []
    lengths = LENGTHS(H)
    for L in lengths:
        for t in _targets(ws, L):
            lo, hi = H + TILE * t, min(L, H + TILE * (t + 1))
            # byte outside the Phred range at a lane in the middle of the step's valid part
            qs = list(np.resize(np.frombuffer(b"%&", dtype=np.uint8), L))
            qs[lo + (hi - lo) // 2] = 0x20
            out.append(("nan", t, qs))
            # tie: a background whose running sum is in a binade with exactly one tie byte when the step starts
            for bg in BACKGROUNDS:
                qs = [int(c) for c in np.resize(np.frombuffer(bg, dtype=np.uint8), L)]
                s = 0.0
                for c in qs[:lo]:
                    s += q[c]
                ch = tie_chars.get(expo(s), [])
                if len(ch) != 1 or not 5 <= expo(s) < 52:
                    continue
                qs[lo + 16 * ((hi - lo - 1) // 16 // 2) + 3 if hi - lo > 16 else lo] = ch[0]
                if _window_ok(qs, ws, q, a) and _step_counts(qs, ws, model)[t][1] > 0:
                    out.append(("tie", t, qs))
                    break
            # binade crossing inside the step, replayed on the lattice (not walked serially)
            for bg in BACKGROUNDS:
                qs = [int(c) for c in np.resize(np.frombuffer(bg, dtype=np.uint8), L)]
                if not _window_ok(qs, ws, q, a):
                    continue
                if _step_counts(qs, ws, model)[t][0] > 0:
                    out.append(("cross", t, qs))
                    break
    return out


def test_designed_reads_reach_the_modes():
    """on the lattice model: for window 250, every step target gets a tie read walked serially there and a read whose
    binade crossing is replayed there; every designed read of every window is scored by the kernels, not the fallback,
    unless it holds a byte outside the Phred range"""
    for ws in WINDOWS:
        q, a = tables(ws)
        got = {}
        for kind, t, qs in designed_reads(ws):
            got.setdefault(kind, set()).add(t)
            if kind != "nan":
                assert _window_ok(qs, ws, q, a), (ws, kind, t)
        assert got["nan"] == set(range(STEPS)) | {_steps(ws, L) - 1 for L in LENGTHS(head(ws))}
        if ws == 250:
            assert set(range(STEPS)) <= got["tie"], got["tie"]
            assert set(range(STEPS)) <= got["cross"], got["cross"]


@pytest.mark.gpu
@pytest.mark.parametrize("ws", WINDOWS)
def test_tie_nan_crossing_at_pipeline_steps(ws):
    reads = []
    rng = np.random.default_rng(7300 + ws)
    for i, (_, _, qs) in enumerate(designed_reads(ws)):
        reads.append((b"A" * len(qs), bytes(qs)))
        L = len(qs) - 17 * (i % 3)                                    # and an ordinary read next to it
        reads.append((b"A" * L, _qual(rng, L)))
    ctx, summ, sc, _ = run_both(reads, dict(keep_percent=70.0, window_size=ws))
    full_check(ctx, summ, sc)
    ctx.close()

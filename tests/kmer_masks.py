"""Designed hit masks for k-mer mode (no GPU).

A design is a 0/1 mask over a read whose 1-runs are all at least 16 bases long. `realize` turns designs into reads
and one 16-mer set such that painting the reads (read.cpp:43-58) gives back exactly the designs: the set is the
16-mers of the 1-runs' bases (both strands, as an assembly adds them), and a chance member at a start that touches a
zero of the design is removed by redrawing one base at such a zero (a zero position never belongs to a hit, so no
designed hit changes). Zero positions also carry N, IUPAC letters and lowercase bytes, hit positions lowercase
bytes, so the reads go through the packer's byte mapping too.

The row builders below make the masks the window, scan and paint kernels of k-mer mode are weakest on: rows whose
window count rises through every binade, first windows on a tie binade, counts hovering at binade edges, zero runs
at word and step seams, isolated hits at lane, step and tile seams.
"""
import math

import numpy as np

K = 16
CODE = np.zeros(256, dtype=np.uint8)                      # read.cpp: A/a 0, C/c 1, G/g 2, T/t 3, any other byte 0
for _c, _v in zip(b"ACGTacgt", (0, 1, 2, 3, 0, 1, 2, 3)):
    CODE[_c] = _v
UPPER = np.frombuffer(b"ACGT", dtype=np.uint8)
LOWER = np.frombuffer(b"acgt", dtype=np.uint8)
ZERO_CODE_BYTES = np.frombuffer(b"NnRYKMSWBDHVrykmswbdhv.-aA", dtype=np.uint8)    # all of them map to code 0


# ---- masks --------------------------------------------------------------------------------------------------------------
def runs_of(bits):
    """(starts, ends) of the 1-runs of a bool mask"""
    d = np.diff(np.concatenate([[0], np.asarray(bits, dtype=np.int8), [0]]))
    return np.nonzero(d == 1)[0], np.nonzero(d == -1)[0]


def zero_runs_of(bits):
    return runs_of(~np.asarray(bits, dtype=bool))


def is_design(bits):
    s, e = runs_of(bits)
    return bool(np.all(e - s >= K))


def hit_starts(bits):
    """the starts whose 16 bases all lie in a 1-run: the hits a design asks for"""
    bits = np.asarray(bits, dtype=bool)
    n = len(bits)
    if n < K:
        return np.zeros(0, dtype=bool)
    c = np.concatenate([[0], np.cumsum(bits, dtype=np.int64)])
    return (c[K:] - c[:-K]) == K


def cover(hits, n):
    """bases covered by the hits (a hit at i covers i .. i + 15)"""
    cov = np.zeros(n + 1, dtype=np.int64)
    idx = np.nonzero(hits)[0]
    np.add.at(cov, idx, 1)
    np.add.at(cov, idx + K, -1)
    return np.cumsum(cov)[:n] > 0


def opening(bits):
    """the largest design inside a mask: every 1-run shorter than 16 removed"""
    bits = np.asarray(bits, dtype=bool)
    return cover(hit_starts(bits), len(bits))


# ---- 16-mers --------------------------------------------------------------------------------------------------------------
def kmers_of_codes(codes):
    """forward 16-mer (2 bits per base, first base highest) at every start of a code array"""
    codes = np.asarray(codes, dtype=np.uint32)
    n = len(codes) - K + 1
    if n <= 0:
        return np.zeros(0, dtype=np.uint32)
    k = np.zeros(n, dtype=np.uint32)
    for j in range(K):
        k = (k << np.uint32(2)) | codes[j:j + n]
    return k


def kmer_set_of(run_codes):
    """the 16-mers an assembly made of these sequences adds: every 16-mer of each, and its reverse complement"""
    parts = []
    for c in run_codes:
        parts.append(kmers_of_codes(c))
        parts.append(kmers_of_codes((3 - np.asarray(c, dtype=np.int64))[::-1]))
    return np.unique(np.concatenate(parts)) if parts else np.zeros(0, dtype=np.uint32)


def paint(seq, members):
    """read.cpp:43-58 restated: the bases of `seq` (bytes) covered by a forward 16-mer in `members` (sorted uint32)"""
    codes = CODE[np.frombuffer(seq, dtype=np.uint8)]
    k = kmers_of_codes(codes)
    if len(k) == 0 or len(members) == 0:
        return np.zeros(len(seq), dtype=bool)
    i = np.minimum(np.searchsorted(members, k), len(members) - 1)
    return cover(members[i] == k, len(seq))


class Realized:
    """reads (seq, qual) realizing `designs` under the 16-mer set `members`; `runs` are the 1-runs' bases (upper case),
    the sequences that add exactly `members` as an assembly"""

    def __init__(self, designs, reads, runs, members):
        self.designs, self.reads, self.runs, self.members = designs, reads, runs, members

    def mean(self, i):
        """what the design says the read's raw mean is: 100 * popcount / L (0/0 is NaN, as in read.cpp)"""
        d = self.designs[i]
        with np.errstate(invalid="ignore", divide="ignore"):
            return 100.0 * float(np.count_nonzero(d)) / float(len(d)) if len(d) else float("nan")


def realize(designs, rng, fancy=True):
    designs = [np.asarray(d, dtype=bool) for d in designs]
    for d in designs:
        assert is_design(d), "a 1-run shorter than 16"
    codes = [rng.integers(0, 4, size=len(d)).astype(np.uint8) for d in designs]
    run_codes = []
    for d, c in zip(designs, codes):
        for s, e in zip(*runs_of(d)):
            run_codes.append(c[s:e])
    members = kmer_set_of(run_codes)
    for d, c in zip(designs, codes):
        want = hit_starts(d)
        zeros = np.nonzero(~d)[0]
        for _ in range(64):
            k = kmers_of_codes(c)
            if len(k) == 0 or len(members) == 0:
                break
            i = np.minimum(np.searchsorted(members, k), len(members) - 1)
            bad = np.nonzero((members[i] == k) & ~want)[0]
            if len(bad) == 0:
                break
            # a colliding start touches at least one zero of the design: redraw one of them
            lo, hi = np.searchsorted(zeros, bad), np.searchsorted(zeros, bad + K)
            pos = np.unique(zeros[lo + (rng.random(len(bad)) * (hi - lo)).astype(np.int64)])
            c[pos] = (c[pos] + rng.integers(1, 4, size=len(pos))) % 4
        else:
            raise AssertionError("chance members could not be removed")
    reads = []
    for d, c in zip(designs, codes):
        seq = UPPER[c].copy()
        if fancy and len(d):
            low = rng.random(len(d)) < 0.05
            seq[low] = LOWER[c[low]]
            z = np.nonzero(~d & (c == 0))[0]
            z = z[rng.random(len(z)) < 0.3]
            seq[z] = ZERO_CODE_BYTES[rng.integers(0, len(ZERO_CODE_BYTES), size=len(z))]
        reads.append((seq.tobytes(), b"I" * len(d)))
    runs = [UPPER[c].tobytes() for c in run_codes]
    return Realized(designs, reads, runs, members)


# ---- the window kernel's rows ----------------------------------------------------------------------------------------------
def tie_levels(ws):
    """counts c in 0..ws whose c / ws lies in a tie binade (rq = 1 / ws is n + 1/2 units of the binade's grid)"""
    rq = 1.0 / ws
    m, e_rq = math.frexp(rq)                    # rq = m * 2^e_rq, m in [0.5, 1)
    mant = int(m * 2.0 ** 53)
    e_rq -= 1
    out = []
    for e in range(e_rq + 1, 1):
        s = e - e_rq
        if s > 52:
            break
        if mant & ((1 << s) - 1) == 1 << (s - 1):
            lo, hi = int(np.ceil(2.0 ** e * ws)), int(np.ceil(2.0 ** (e + 1) * ws)) - 1
            out.extend(range(max(lo, 1), min(hi, ws) + 1))
    return out


def edge_levels(ws):
    """the counts next to the binade edges 2^e * ws that a count 0..ws can reach"""
    out = set()
    e = 0
    while 2.0 ** e * ws >= 1.0:
        x = 2.0 ** e * ws
        out.update(c for c in (int(np.floor(x)) - 1, int(np.floor(x)), int(np.ceil(x)), int(np.ceil(x)) + 1) if 0 < c <= ws)
        e -= 1
    return sorted(out)


def rising(rng, n, ws, lead):
    """zeros (lead = 0) or one 16-run (lead = 1) in the first window, then 16-runs with gaps that shrink block by block
    until the row is fully covered: the count climbs through every binade, each new record level next to an edge"""
    out = np.zeros(n, dtype=bool)
    if lead:
        out[:K] = True
    p = max(ws, K + 1)
    for gap in sorted(rng.integers(0, 64, size=6))[::-1]:
        end = min(n, p + max(3 * ws, 200))
        while p < end:
            out[p:p + K] = True
            p += K + int(gap)
    out[p:] = True
    return opening(out)


def first_window(rng, n, ws, c0, child):
    """a first window holding exactly c0 ones (a child row must begin with a covered base), then a sparse tail"""
    out = np.zeros(n, dtype=bool)
    if child:
        if c0 < K + 1 or c0 > ws:
            return None
        a = K + int(rng.integers(0, max(1, c0 - 2 * K))) if c0 >= 2 * K + 1 else c0
        out[:a] = True
        b = c0 - a
        if b:
            if ws - b <= a:                             # no room for a gap: one run of c0 then the tail
                return None
            out[ws - b:ws + K] = True
    else:
        out[ws - c0:ws + (K if c0 < K else 0)] = True
    p = ws + K + 1
    while p < n:
        p += int(rng.integers(1, 40))
        out[p:p + int(rng.integers(K, 40))] = True
        p += K
    out = opening(out)
    return out if out[:ws].sum() == c0 else None          # (too short a row cannot hold the straddling run)


def hover(rng, n, ws, c0, lead_one):
    """a pattern of ws bases holding c0 ones in runs >= 16, repeated, each copy with a few runs moved or stretched by one
    or two bases: the count hovers within +-2 of c0 (two edge crossings within a 32-step word when c0 is on an edge)"""
    if c0 < K or ws - c0 < 2:
        return None
    n_runs = max(1, min(c0 // K, (ws - c0) // 2))
    while n_runs > 1 and ws - c0 < 2 * (n_runs + (0 if lead_one else 1)):
        n_runs -= 1
    lens = np.full(n_runs, c0 // n_runs)
    lens[:c0 % n_runs] += 1
    if lens.min() < K:
        return None
    gaps_n = n_runs + (0 if lead_one else 1)
    z = ws - c0
    if z < gaps_n:
        return None
    gaps = np.ones(gaps_n, dtype=np.int64)
    extra = rng.multinomial(z - gaps_n, np.ones(gaps_n) / gaps_n)
    gaps += extra
    starts, p, g = [], 0, 0
    if not lead_one:
        p += int(gaps[0])
        g = 1
    for i in range(n_runs):
        starts.append(p)
        p += int(lens[i])
        if g < gaps_n:
            p += int(gaps[g])
            g += 1
    out = np.zeros(n, dtype=bool)
    base = 0
    while base < n:
        for s, L in zip(starts, lens):
            ds, de = 0, 0
            if base > 0 and rng.random() < 0.3:
                ds, de = int(rng.integers(-1, 2)), int(rng.integers(-2, 3))
            a, b = base + s + ds, base + s + int(L) + de
            if b - a >= K:
                out[max(a, 0):min(b, n)] = True
        base += ws
    out = opening(out)
    return out


def model_kind(rng, kind, n):
    """the opening of one of tests/test_kmer_window_model.py's mask kinds"""
    from tests.test_kmer_window_model import make_mask
    return opening(make_mask(rng, kind, n))


def window_rows(rng, ws, n_rows, lengths, child):
    """n_rows designs for window size ws, the kinds taking turns: rising, tie-binade first window, hovering at half
    and at binade edges, openings of the model's mask kinds; lengths cycle through `lengths`"""
    rows = []
    ties = tie_levels(ws)
    edges = edge_levels(ws)
    i = 0
    while len(rows) < n_rows:
        n = int(lengths[len(rows) % len(lengths)])
        kind = i % 6
        i += 1
        r = None
        if kind == 0:
            r = rising(rng, n, ws, 1 if child else int(rng.integers(0, 2)))
        elif kind == 1 and ties:
            r = first_window(rng, n, ws, int(ties[int(rng.integers(0, len(ties)))]), child)
        elif kind == 2:
            r = hover(rng, n, ws, ws // 2 + int(rng.integers(0, 2)) * (ws % 2), child)
        elif kind == 3 and edges:
            r = hover(rng, n, ws, int(edges[int(rng.integers(0, len(edges)))]), child)
        elif kind >= 4:
            r = model_kind(rng, int(rng.integers(0, 7)), n)
        if r is None or len(r) != n:
            continue
        if child:
            r[:K] = True                                # a child begins and ends with a covered base
            r[-K:] = True
            r = opening(r)
        rows.append(r)
    return rows


def join_as_children(rows, split, rng, start_residues):
    """one read holding `rows` as children under --split `split`: each row follows a zero run of at least `split`
    bases, long enough that the row starts at the wanted residue mod 32; a zero run after the last"""
    parts, pos, starts = [], 0, []
    for r, res in zip(rows, start_residues):
        g = split + ((res - (pos + split)) % 32)
        parts.append(np.zeros(g, dtype=bool))
        pos += g
        starts.append(pos)
        parts.append(r)
        pos += len(r)
    parts.append(np.zeros(split + int(rng.integers(0, 40)), dtype=bool))
    return np.concatenate(parts), starts


def max_zero_run(bits):
    s, e = zero_runs_of(bits)
    return int((e - s).max()) if len(s) else 0


# ---- the cases of tests/test_gpu_kmer_masks.py (also checked on the CPU by tests/test_kmer_mask_design.py) -------------
WINDOW_SIZES = [1, 2, 3, 7, 15, 16, 17, 33, 100, 250, 256, 470, 1000, 4097, 32768, 32769, 65536, 100000]
SPLITS = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025]
LANE, STEP, TILE = 32, 1024, 8192


def window_case(ws):
    """(whole-read designs, one read holding child rows, the --split that cuts it into exactly those rows, the rows'
    starts). Child rows start at every residue mod 32 and end at every residue mod 32, with lengths ws, ws + 1,
    ws + 31 .. 33 and ws + 1024 +- 1."""
    rng = np.random.default_rng(7000 + ws)
    big = ws >= 4096
    whole_len = [ws + 1 + x for x in ((1, 40, 1100, 2 * ws) if big else (1, 33, 1025, 3000, 12000, 20 * ws + 500))]
    whole = window_rows(rng, ws, 8 if big else 18, whole_len, child=False)
    lengths = [max(ws + d, K) for d in (0, 1, 31, 32, 33, 1023, 1025)]
    n_child = 32 if big else 64
    rows = window_rows(rng, ws, n_child, lengths, child=True)
    # the first 32 rows start at residue j, the rest end at residue j
    res = [j % 32 if j < 32 else (j - len(rows[j])) % 32 for j in range(n_child)]
    split = max(max_zero_run(r) for r in rows) + 1
    read, starts = join_as_children(rows, split, rng, res)
    return whole, read, split, starts, rows


def _carve(L, zruns):
    bits = np.ones(L, dtype=bool)
    for p, z in zruns:
        bits[p:p + z] = False
    return bits


def scan_designs(split):
    """designs for --split `split`: zero runs of split - 1, split and split + 1 bases inside one word, across a word seam,
    ending in lane 0's word of a step after a run open at the end of the previous step, and longer than a whole step;
    leading and trailing zero runs (the trim ranges); hit-less reads around `split`; reads of 15 .. 33 bases"""
    rng = np.random.default_rng(9000 + split)
    out = []
    for rep in range(3):
        zr, pos = [], K + int(rng.integers(0, 64))
        for z in (split - 1, split, split + 1, 1024 + int(rng.integers(1, 700))):
            if z < 1:
                continue
            for where in ("word", "seam", "lane0", "step"):
                q = pos + K
                if where == "word":
                    if z > 30:
                        continue
                    q = (q + 31) // 32 * 32
                    p = q + 1 + int(rng.integers(0, 31 - z))
                elif where == "seam":
                    if z < 2:
                        continue
                    q = (q + z + 31) // 32 * 32
                    p = q - int(rng.integers(1, z))
                elif where == "lane0":
                    if z < 2:
                        continue
                    q = (q + z + STEP - 1) // STEP * STEP
                    p = q + int(rng.integers(0, min(31, z - 1) + 1)) - z
                else:
                    if z < STEP:
                        continue
                    q = (q + STEP - 1) // STEP * STEP
                    p = q - int(rng.integers(0, z - STEP + 1))
                if p < pos + K:
                    continue
                zr.append((p, z))
                pos = p + z
        L = pos + K + int(rng.integers(0, 100))
        lead = (split + rep - 1) if rep else 0                    # leading / trailing zero runs: the trim ranges
        trail = (split + 1 - rep) if rep < 2 else 0
        bits = np.concatenate([np.zeros(lead, bool), _carve(L, zr), np.zeros(trail, bool)])
        out.append(bits)
    for L in (split - 1, split, split + 1):                       # no hit at all
        if L > 0:
            out.append(np.zeros(L, dtype=bool))
    for L in (15, 16, 17, 31, 32, 33):
        out.append(np.zeros(L, dtype=bool) if L < K else np.ones(L, dtype=bool))
        if L > K:
            b = np.zeros(L, dtype=bool)
            b[L - K:] = True
            out.append(b)
            b = np.zeros(L, dtype=bool)
            b[:K] = True
            out.append(b)
    return [opening(b) for b in out]


def many_children(n, gap):
    """about n bases of 16-runs separated by `gap` zeros: one child per run under --split gap"""
    period = K + gap
    bits = (np.arange(n) % period) < K
    bits[n - (n % period):] = False
    return opening(bits)


def paint_designs():
    """isolated hits (exactly 16 bases) at every start within 20 of a lane, step and tile seam and at the last start,
    pairs of hits with a gap of 1 .. 17 across each seam, read lengths 8192 t + {-17, -16, -1, 0, 1, 15, 16, 17}"""
    out = []
    seams = [LANE * m for m in (5, 41, 70)] + [STEP * m for m in (3, 6, 9, 13)] + [TILE, 2 * TILE]
    L = 2 * TILE + 200
    for d in range(-20, 21):
        b = np.zeros(L, dtype=bool)
        for s in seams:
            b[s + d:s + d + K] = True
        out.append(b)
    for gap in range(1, 18):
        b = np.zeros(L, dtype=bool)
        for i, s in enumerate(seams):
            a = s - K - int((gap + i) % (gap + 2))                  # the gap starts before, at or after the seam
            b[a:a + K] = True
            b[a + K + gap:a + 2 * K + gap] = True
        out.append(b)
    for t in (1, 2):
        for dl in (-17, -16, -1, 0, 1, 15, 16, 17):
            n = TILE * t + dl
            b = np.zeros(n, dtype=bool)
            b[n - K:] = True                                        # a hit at the last start, L - 16
            b[TILE * t - K - 3:TILE * t - 3] |= dl >= 0
            out.append(b)
            b = np.zeros(n, dtype=bool)
            b[n - 2 * K - 1:n - K - 1] = True
            out.append(b)
    return [opening(b) for b in out]

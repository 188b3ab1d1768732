"""Designed contigs for the one-copy 16-mer build, `k_kmers_add<false>` (no GPU).

The build kernel does position-dependent work at its seams: a warp takes a tile of 8,192 bases of one sequence in
steps of 1,024, 32 bases per lane; a lane's 16-mers need the next lane's words (the next step's for lane 31); the
reverse 16-mer clears its non-ACGT fields from a 64-bit window of the mask, whose second word is bounded by the
sequence's padded (64-base) length; sequences under 16 bases take a tile and are skipped. The five packers in front of
it (host batches, FASTQ / FASTA text, wrapped FASTA, device 2-bit + mask, device ASCII) each compute that mask their way.

So the contigs below put non-ACGT bytes at every offset S - 16 .. S + 15 of every seam S: the contig's start and end,
the lane boundaries of a step (32 k, in the first and in the last step of a tile), the step and tile boundaries
(1,024 k and 8,192 k) and the end of the 64-base padding. Copy c of a contig carries its byte at S + (c mod 32) - 16 of
every seam at once, drawn in turn from every byte class that packs to code 0; further copies carry runs of 15, 16 and
17 such bytes straddling every seam, and lower-case runs across them. Contig lengths sit on and around every seam, a
contig of about 200 kbases spans two dozen tiles, contigs under 16 bases sit between the long ones, and a run of a few
thousand contigs of 1 to 40 bases fills warps with many sequences. The genome is random, so the true 16-mer set is
sparse in 4^16 and one wrong 16-mer shows.

`wrapped_extra(w)` adds, for a FASTA file wrapped at w bases a line, contigs with a non-ACGT byte on the last base of a
line, on the first base of the next, on both, and lower case across the line end.
"""
import functools
from dataclasses import dataclass, field

import numpy as np

from tests import kmer_masks as km
from tests.kmer_build_model import ACGT, K

LANE, STEP, TILE, ALIGN = 32, 1024, 8192, 64
OTHER_BYTES = bytes(b for b in km.ZERO_CODE_BYTES.tobytes() if not ACGT[b]) + b"*"   # every byte class that packs to 0
SEAM_CLASSES = ("start", "end", "lane", "step", "tile", "pad")
LENGTHS = ([0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 192, 256, 512, 2048, 4095]
           + [STEP + d for d in (-1, 0, 1, 15, 16, 17)]
           + [TILE + d for d in (-1, 0, 1, 15, 16, 17)]
           + [2 * TILE + d for d in (-1, 0, 1, 16)]
           + [24 * TILE + 1000])
WIDTHS = [1, 7, 31, 32, 33, 60, 64, 1000]
UPPER = np.frombuffer(b"ACGT", dtype=np.uint8)


def padded(L):
    return (L + ALIGN - 1) // ALIGN * ALIGN


def seams(L):
    """{position: classes} of the seams of a contig of L bases that have an offset -16 .. 15 inside it"""
    out = {}

    def add(cls, S):
        if S - K < L and S + K > 0:
            out.setdefault(S, []).append(cls)

    add("start", 0)
    add("end", L)
    add("pad", padded(L))
    for base in (0, 7 * STEP):                                     # the lane boundaries of a tile's first and last step
        for k in range(1, STEP // LANE):
            add("lane", base + LANE * k)
    for k in range(1, L // STEP + 1):
        add("tile" if k % (TILE // STEP) == 0 else "step", STEP * k)
    return out


def offsets_of(cls):
    """the offsets from a seam of class `cls` that can lie inside a contig"""
    return range(0, K) if cls == "start" else range(-K, 0) if cls in ("end", "pad") else range(-K, K)


@dataclass
class Design:
    contigs: list                                         # bytes, in file order
    placements: dict = field(default_factory=dict)        # (class, offset, byte) -> single non-ACGT bytes placed there
    runs: dict = field(default_factory=dict)              # (class, run length) -> runs at or across such a seam
    lower_runs: int = 0                                   # lower-case runs across a seam
    cuts: list = field(default_factory=list)              # record-aligned chunk cuts: before and after the long contigs
    long_contigs: int = 0


def _template(rng, L):
    return UPPER[rng.integers(0, 4, size=L)].copy()


def _placed_copies(t, rounds, counter, d_out):
    """32 * rounds copies of template t: copy c has a byte at S + (c mod 32) - 16 of every seam S. The byte goes round
    the byte classes, first to those not yet placed at that offset of the seam's classes (a seam can be of several: the
    end of a contig of 8,192 bases is also a tile boundary and the end of its padding)"""
    L = len(t)
    sm = seams(L)
    out = []
    for c in range(32 * rounds):
        d = c % 32 - 16
        s = t.copy()
        for S, classes in sm.items():
            p = S + d
            if not 0 <= p < L:
                continue
            key = (tuple(classes), d)
            rot = counter.get(key, 0)
            counter[key] = rot + 1
            order = [OTHER_BYTES[(rot + i) % len(OTHER_BYTES)] for i in range(len(OTHER_BYTES))]
            b = max(order, key=lambda b: sum((cls, d, b) not in d_out.placements for cls in classes))
            s[p] = b
            for cls in classes:
                d_out.placements[(cls, d, b)] = d_out.placements.get((cls, d, b), 0) + 1
        out.append(s.tobytes())
    return out


def _run_copies(t, rng, d_out):
    """copies with runs of 15, 16 and 17 non-ACGT bytes at every seam (ending at it, straddling it from r - 1, r / 2 and
    1 bases before it, starting at it), one with lower case across every seam, and one all in lower case"""
    L = len(t)
    sm = seams(L)
    other = np.frombuffer(OTHER_BYTES, dtype=np.uint8)
    out = []
    for r in (15, 16, 17):
        for lead in (r, r - 1, r // 2, 1, 0):
            s = t.copy()
            for S, classes in sm.items():
                a, b = max(S - lead, 0), min(S - lead + r, L)
                if b <= a:
                    continue
                s[a:b] = other[rng.integers(0, len(other), size=b - a)]
                if b - a == r:
                    for cls in classes:
                        d_out.runs[(cls, r)] = d_out.runs.get((cls, r), 0) + 1
            out.append(s.tobytes())
    s = t.copy()
    for S in sm:
        a, b = max(S - 20, 0), min(S + 20, L)
        if b > a:
            s[a:b] = s[a:b] | 0x20
            d_out.lower_runs += 1
    out.append(s.tobytes())
    out.append((t | 0x20).tobytes())
    return out


def _short(rng, genome, n_max):
    """a contig of 1 .. n_max bases, sometimes with a non-ACGT byte or lower case"""
    n = int(rng.integers(1, n_max + 1))
    p = int(rng.integers(0, len(genome) - n))
    s = genome[p:p + n].copy()
    if rng.random() < 0.4:
        s[int(rng.integers(0, n))] = OTHER_BYTES[int(rng.integers(0, len(OTHER_BYTES)))]
    if rng.random() < 0.2:
        s |= 0x20
    return s.tobytes()


@functools.lru_cache(maxsize=None)
def design(seed=1600):
    rng = np.random.default_rng(seed)
    d = Design([])
    counter = {}
    genome = _template(rng, 100000)
    for L in LENGTHS:
        t = _template(rng, L)
        copies = _placed_copies(t, 4 if L < TILE else 1, counter, d) + _run_copies(t, rng, d)
        for i, s in enumerate(copies):
            if L >= TILE and i < 2:
                d.cuts += [len(d.contigs), len(d.contigs) + 1]
                d.long_contigs += 1
            d.contigs.append(s)
            if rng.random() < 0.25:                                 # a contig under 16 bases between the long ones
                d.contigs.append(_short(rng, genome, 15))
        if L == 4095:                                               # a run of thousands of contigs of 1 .. 40 bases
            d.contigs += [_short(rng, genome, 40) for _ in range(3000)]
    d.cuts = sorted(set(c for c in d.cuts if 0 < c < len(d.contigs)))
    return d


@functools.lru_cache(maxsize=None)
def wrapped_extra(w, seed=1700):
    """contigs for a FASTA file wrapped at w bases a line: (contigs, bytes placed on the last base of a line, bytes
    placed on the first base of a line). Line ends at least 40 bases apart carry a non-ACGT byte on the line's last
    base, on the next line's first base, or on both; a fourth contig has lower case across them."""
    rng = np.random.default_rng(seed + w)
    L = min(max(64 * w, 4096), 70000)
    t = _template(rng, L)
    ends = np.arange(w, L, w * max(1, -(-40 // w)))                # positions of a line's first base
    other = np.frombuffer(OTHER_BYTES, dtype=np.uint8)
    out, last, first = [], 0, 0
    for where in ("last", "first", "both"):
        s = t.copy()
        if where in ("last", "both"):
            s[ends - 1] = other[rng.integers(0, len(other), size=len(ends))]
            last += len(ends)
        if where in ("first", "both"):
            s[ends] = other[rng.integers(0, len(other), size=len(ends))]
            first += len(ends)
        out.append(s.tobytes())
    s = t.copy()
    for e in ends:
        s[max(e - 3, 0):e + 3] |= 0x20
    out.append(s.tobytes())
    return out, last, first


# ---- the files the text paths read ----------------------------------------------------------------------------------
def _wrap(s, w):
    n = len(s) // w
    lines = np.frombuffer(s, dtype=np.uint8)[:n * w].reshape(n, w)
    body = np.hstack([lines, np.full((n, 1), ord("\n"), dtype=np.uint8)]).tobytes()
    return body + (s[n * w:] + b"\n" if len(s) % w else b"")


def fasta(contigs, width=None, first=0):
    """FASTA text, one line per sequence (width None) or wrapped at `width` bases a line (an empty sequence: no line)"""
    parts = []
    for i, s in enumerate(contigs):
        parts.append(b">contig_%d\n" % (first + i))
        if s:
            parts.append(s + b"\n" if width is None or len(s) <= width else _wrap(s, width))
    return b"".join(parts)


def fastq(contigs, first=0):
    return b"".join(b"@contig_%d\n%s\n+\n%s\n" % (first + i, s, b"I" * len(s)) for i, s in enumerate(contigs))


def chunks(contigs, cuts):
    """the contigs cut into record-aligned pieces at `cuts` (indices)"""
    b = [0] + list(cuts) + [len(contigs)]
    return [contigs[b[i]:b[i + 1]] for i in range(len(b) - 1) if b[i + 1] > b[i]]

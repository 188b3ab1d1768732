"""An exact model of the BGZF members `k_bgzf_deflate` (filtlong_b200/csrc/fl_bgzf.cu) writes, from the rules of DESIGN
§4.7, and blocks designed to reach the compressor's rare paths.

`member(block)` gives the bytes of one member and what the coverage checks need; `model_bgzf(data)` the members of every
65,280-byte block of data, back to back. The Huffman code lengths come from fl_huff_lengths_sorted itself (fl_bgzf.h,
built for the host by tests/bgzf_codes_dump.cpp and pinned by tests/test_bgzf_codes.py); everything else is plain Python.

The rules, one block of n bytes at a time:
  * candidates: positions p with p + 4 <= n are hashed, h = (little-endian 4 bytes at p * 0x9E3779B1 mod 2^32) >> 19,
    in steps of 512 positions split into warps of 32. p's candidate is the latest earlier position of its warp with the
    same h, if its four bytes agree (only that one is tried); else the latest hashed position with that h in an earlier
    step, if it is at most 32,768 back and its four bytes agree; else none;
  * parse: segment t is [128 t, 128 t + 128) cut to the block, parsed greedily. A candidate gives a match when at least 3
    bytes are left in the segment; its length is the number of agreeing bytes, at most min(bytes left, 258), and at least 3;
  * codes: histograms with the end-of-block symbol, dummy symbols (the lowest unused ones) up to two used symbols per
    tree, lengths limited to 15 bits, HLIT / HDIST trimmed, the code lengths run-length coded (18 for 11+ zeros, 17 for
    3-10 zeros, 16 for 3-6 repeats of the previous length), their code with dummies, limited to 7 bits, HCLEN trimmed
    to at least 4;
  * member: the dynamic block, or the stored one when the dynamic member is not smaller.
"""
import atexit
import bisect
import heapq
import shutil
import struct
import tempfile
import zlib

import numpy as np

from tests import bgzf_util as bu

BLOCK = bu.BLOCK
STEP, WARP, SEG = 512, 32, 128
HASH_BITS, WINDOW, MAX_MATCH = 13, 32768, 258
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
# RFC 1951 3.2.5
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
HEADER = b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0"

_dumper = None


def _huff_lengths(freqs, maxbits):
    global _dumper
    if _dumper is None:
        d = tempfile.mkdtemp(prefix="bgzf_model_")
        atexit.register(shutil.rmtree, d, True)
        _dumper = bu.build_codes_dumper(d)
    return bu.huff_codes(_dumper, freqs, maxbits)[0]


def hashes(a):
    """4-byte words and their 13-bit hashes at every position p with p + 4 <= len(a)."""
    a = np.frombuffer(bytes(a), np.uint8).astype(np.uint64)
    m = max(len(a) - 3, 0)
    x = a[:m] | a[1:m + 1] << 8 | a[2:m + 2] << 16 | a[3:m + 3] << 24
    return x, ((x * 0x9E3779B1) & 0xffffffff) >> (32 - HASH_BITS)


def candidates(block):
    """Candidate distance of every position (0: none)."""
    n = len(block)
    x, h = (v.tolist() for v in hashes(block))
    m = len(x)
    cand = [0] * n
    table = {}                                      # hash -> latest position of an earlier step
    for base in range(0, m, STEP):
        top = min(base + STEP, m)
        for w in range(base, top, WARP):
            lanes = {}                              # hash -> latest earlier position of this warp
            for p in range(w, min(w + WARP, top)):
                hp, d = h[p], 0
                q = lanes.get(hp)
                if q is not None and x[q] == x[p]:
                    d = p - q
                if not d:
                    t = table.get(hp)
                    if t is not None and p - t <= WINDOW and x[t] == x[p]:
                        d = p - t
                cand[p] = d
                lanes[hp] = p
        for p in range(base, top):
            table[h[p]] = p
    return cand


def parse(block, cand):
    """Greedy parse of every segment: (position, distance, length) per token, distance 0 for a literal."""
    n, tokens = len(block), []
    for s in range(0, n, SEG):
        e, p = min(s + SEG, n), s
        while p < e:
            d, L = cand[p], 0
            if d and e - p >= 3:
                lim = min(e - p, MAX_MATCH)
                while L < lim and block[p - d + L] == block[p + L]:
                    L += 1
            if L >= 3:
                tokens.append((p, d, L))
                p += L
            else:
                tokens.append((p, 0, 1))
                p += 1
    return tokens


def len_code(L):
    c = bisect.bisect_right(LEN_BASE, L) - 1
    return c, LEN_EXTRA[c], L - LEN_BASE[c]


def dist_code(d):
    c = bisect.bisect_right(DIST_BASE, d) - 1
    return c, DIST_EXTRA[c], d - DIST_BASE[c]


def add_dummies(hist):
    """The lowest unused symbols get count 1 until two are used; whether any was added."""
    used, added = sum(1 for f in hist if f), False
    for i in range(len(hist)):
        if used >= 2:
            break
        if not hist[i]:
            hist[i], used, added = 1, used + 1, True
    return added


def free_depth(hist):
    """Longest length of an unrestricted Huffman code over the used symbols."""
    heap = [(f, i, 0) for i, f in enumerate(hist) if f]
    if len(heap) < 2:
        return 1 if heap else 0
    heapq.heapify(heap)
    k = len(hist)
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        heapq.heappush(heap, (a[0] + b[0], k, max(a[2], b[2]) + 1))
        k += 1
    return heap[0][2]


def canonical(lengths):
    """RFC 1951 3.2.2 codes, most significant bit first."""
    count = [0] * 17
    for L in lengths:
        count[L] += 1
    count[0] = 0
    nxt, c = [0] * 17, 0
    for b in range(1, 17):
        c = (c + count[b - 1]) << 1
        nxt[b] = c
    codes = [0] * len(lengths)
    for i, L in enumerate(lengths):
        if L:
            codes[i] = nxt[L]
            nxt[L] += 1
    return codes


def rle(lengths):
    """Code-length symbols of the header: (symbol, extra bits value)."""
    out, i = [], 0
    while i < len(lengths):
        v, run = lengths[i], 1
        while i + run < len(lengths) and lengths[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while run >= 11:
                k = min(run, 138)
                out.append((18, k - 11))
                run -= k
            if run >= 3:
                out.append((17, run - 3))
                run = 0
            out += [(0, 0)] * run
        else:
            out.append((v, 0))
            run -= 1
            while run >= 3:
                k = min(run, 6)
                out.append((16, k - 3))
                run -= k
            out += [(v, 0)] * run
    return out


class Bits:
    """LSB-first bit writer."""

    def __init__(self):
        self.out, self.acc, self.nb = bytearray(), 0, 0

    def put(self, v, n):
        self.acc |= v << self.nb
        self.nb += n
        while self.nb >= 8:
            self.out.append(self.acc & 0xff)
            self.acc >>= 8
            self.nb -= 8

    def huff(self, code, n):                      # Huffman codes go most significant bit first
        self.put(int(format(code, "0%db" % n)[::-1], 2), n)

    def bytes(self):
        return bytes(self.out) + (bytes([self.acc]) if self.nb else b"")


def member(block):
    """(bytes of the member, stats) for one block of 1 to 65,280 bytes."""
    block = bytes(block)
    n = len(block)
    assert 1 <= n <= BLOCK
    cand = candidates(block)
    tokens = parse(block, cand)
    lhist, dhist = [0] * 286, [0] * 30
    lhist[256] = 1
    for p, d, L in tokens:
        if d:
            lhist[257 + len_code(L)[0]] += 1
            dhist[dist_code(d)[0]] += 1
        else:
            lhist[block[p]] += 1
    lused, dused = [i for i, f in enumerate(lhist) if f], [i for i, f in enumerate(dhist) if f]
    ldummy, ddummy = add_dummies(lhist), add_dummies(dhist)
    llen, dlen = _huff_lengths(lhist, 15), _huff_lengths(dhist, 15)
    hlit, hdist = 286, 30
    while hlit > 257 and not llen[hlit - 1]:
        hlit -= 1
    while hdist > 1 and not dlen[hdist - 1]:
        hdist -= 1
    syms = rle(llen[:hlit] + dlen[:hdist])
    clhist = [0] * 19
    for s, _ in syms:
        clhist[s] += 1
    cldummy = add_dummies(clhist)
    cllen = _huff_lengths(clhist, 7)
    hclen = 19
    while hclen > 4 and not cllen[CL_ORDER[hclen - 1]]:
        hclen -= 1
    lcode, dcode, clcode = canonical(llen), canonical(dlen), canonical(cllen)

    bits = Bits()
    bits.put(1 | 2 << 1, 3)
    bits.put(hlit - 257, 5)
    bits.put(hdist - 1, 5)
    bits.put(hclen - 4, 4)
    for s in CL_ORDER[:hclen]:
        bits.put(cllen[s], 3)
    for s, x in syms:
        bits.huff(clcode[s], cllen[s])
        if s >= 16:
            bits.put(x, {16: 2, 17: 3, 18: 7}[s])
    for p, d, L in tokens:
        if not d:
            bits.huff(lcode[block[p]], llen[block[p]])
            continue
        c, eb, ev = len_code(L)
        bits.huff(lcode[257 + c], llen[257 + c])
        bits.put(ev, eb)
        c, eb, ev = dist_code(d)
        bits.huff(dcode[c], dlen[c])
        bits.put(ev, eb)
    bits.huff(lcode[256], llen[256])
    body = bits.bytes()
    dyn_size, stored_size = len(HEADER) + 2 + len(body) + 8, len(HEADER) + 2 + 5 + n + 8
    stored = dyn_size >= stored_size
    if stored:
        body = b"\x01" + struct.pack("<HH", n, n ^ 0xffff) + block
    size = len(HEADER) + 2 + len(body) + 8
    out = HEADER + struct.pack("<H", size - 1) + body + struct.pack("<II", zlib.crc32(block) & 0xffffffff, n)
    stats = dict(tokens=tokens, cand=cand, lhist=lhist, dhist=dhist, clhist=clhist,
                 llen=llen, dlen=dlen, cllen=cllen,
                 max_len=(max(llen), max(dlen), max(cllen)),
                 free_depth=(free_depth(lhist), free_depth(dhist), free_depth(clhist)),
                 hlit=hlit, hdist=hdist, hclen=hclen, lit_used=lused, dist_used=dused,
                 dummies=dict(lit=ldummy, dist=ddummy, cl=cldummy),
                 stored=stored, dyn_size=dyn_size, stored_size=stored_size)
    return out, stats


def model_bgzf(data):
    """The members of every 65,280-byte block of data, back to back (no EOF member)."""
    return b"".join(member(data[lo:lo + BLOCK])[0] for lo in range(0, len(data), BLOCK))


# ---- designed blocks ------------------------------------------------------------------------------------------------
# A block is random bytes with copies written into it. A copy (q, p, k, L) puts bytes [q, q + k) at [p, p + k), one byte
# at a time, so p - q < k gives a periodic run; the byte after it is made to differ from the one after the source. The
# greedy parse is meant to give the token (p, p - q, L) for L > 0; for L == 0 a literal at p whose candidate is p - q,
# and for L == -1 a literal without a candidate, the source's hash being on no position in between. Where the model
# does not give that (a 13-bit hash of some other position hides the source), the source is drawn again. `_settle`
# returns the block and the model's stats.

def _random(rng, n, k=256):
    """n random bytes below k: 64 keeps a block dynamic (6 bits a literal) and its chance 4-byte repeats few."""
    return bytearray(rng.integers(0, k, size=n, dtype=np.uint8).tobytes())


def _write(buf, copies):
    for q, p, k, _ in sorted(copies, key=lambda c: c[1]):
        if not k:
            continue
        for i in range(k):
            buf[p + i] = buf[q + i]
        if p + k < len(buf) and buf[p + k] == buf[q + k]:
            buf[p + k] ^= 0x5a


def _hidden(h, q, p):
    """Whether a position after q, where p looks (its warp, else the earlier steps), has q's hash."""
    end = p if p // WARP == q // WARP else p - p % STEP
    return bool((h[q + 1:end] == h[q]).any())


def _expected(c, tok, cand):
    q, p, _, L = c
    if L > 0:
        return tok.get(p) == (p, p - q, L)
    return tok.get(p) == (p, 0, 1) and cand[p] == (p - q if L == 0 else 0)


def _settle(buf, copies, rng, rounds=400):
    """Draws sources again until every copy gives what it is meant to; returns (bytes, stats)."""
    copies = list(copies)
    dest = {}
    for c in copies:
        for i in range(c[1], c[1] + c[2] + 1):
            dest[i] = c

    def root(c):                                   # a source that is itself a copy is drawn at its own source
        while c[0] in dest and dest[c[0]] is not c:
            c = dest[c[0]]
        return c

    for _ in range(rounds):
        _write(buf, copies)
        h = hashes(buf)[1]
        bad = [c for c in copies if _hidden(h, c[0], c[1])]
        if not bad:
            block = bytes(buf)
            cand = candidates(block)
            tok = {t[0]: t for t in parse(block, cand)}
            bad = [c for c in copies if not _expected(c, tok, cand)]
            if not bad:
                return block, member(block)[1]
        for c in {root(c) for c in bad}:            # with the byte before it, which may have started the match early
            q, p, k, _ = c
            lo, hi = max(q - 1, 0), q + max(min(k, p - q), 4)
            buf[lo:hi] = _random(rng, hi - lo)
    raise AssertionError("designed copies do not settle: %s" % bad[:5])


def _seg_ok(p, k):
    return p % SEG + k <= SEG


def fifteen_bit_block():
    """The distance tree's counts are 1, 1, 2, ..., 1597 over 17 codes (an unrestricted Huffman code 16 deep), from
    4-byte copies followed by a byte that breaks them. Distances below 32 reach back inside a warp; the others reach
    an earlier step."""
    rng = np.random.default_rng(1501)
    fib = [1, 1]
    while len(fib) < 17:
        fib.append(fib[-1] + fib[-2])
    # (distance, count): the rarest codes reach back across a step, the commonest inside a warp
    dists = [1024, 768, 512, 384, 256, 192, 128, 96, 64, 48, 25, 17, 13, 9, 7, 5, 4]
    buf = _random(rng, BLOCK)
    used = bytearray(BLOCK + 8)
    copies = []
    for d, cnt in zip(dists, fib):
        p = d
        while cnt:
            q = p - d
            fits = (_seg_ok(p, 4) and p + 5 <= BLOCK and not any(used[q:q + 4]) and not any(used[p:p + 5])
                    and (p // WARP == q // WARP if d < WARP else p // STEP > q // STEP))
            if fits:
                used[q:q + 4] = b"\1" * 4
                used[p:p + 5] = b"\1" * 5
                copies.append((q, p, 4, 4))
                cnt -= 1
                p += 5
            else:
                p += 1
            assert p + 5 <= BLOCK, "the copies do not fit one block"
    return _settle(buf, copies, rng)


def _top(c):
    """The largest distance of distance code c."""
    return DIST_BASE[c + 1] - 1 if c < 29 else WINDOW


def all_symbols_block():
    """Every match length 3..128, each cut by the end of its segment, and every distance code: HLIT 281, HDIST 30.
    Codes 0-9 reach back inside a warp (periodic runs when the distance is below the length), the others to an
    earlier step."""
    rng = np.random.default_rng(281)
    buf = _random(rng, BLOCK)
    used = bytearray(BLOCK + 8)
    lengths = list(range(3, 129))
    # the in-warp codes need (128 - L) % 32 >= d; the first length that allows it takes each
    plan = {}
    for c in range(10):
        L = next(L for L in lengths if L not in plan and (-L) % WARP >= DIST_BASE[c])
        plan[L] = DIST_BASE[c]
    # the others (distance d >= 33) need an earlier step: p % 512 = 128 - L < d in a step's first segment
    far = [_top(c) for c in range(10, 30)]
    for i, L in enumerate(L for L in lengths if L not in plan):
        plan[L] = next(d for j in range(len(far)) for d in [far[(i + j) % len(far)]] if d >= SEG or SEG - L < d)
    copies = []
    for L in sorted(plan, key=lambda L: -plan[L]):
        d, k = plan[L], max(L, 4)
        for s in range(0, BLOCK - SEG, SEG):
            p = s + SEG - L
            q = p - d
            ok = q >= 0 and not any(used[p:p + k + 1]) and not any(used[q:q + min(k, d)])
            ok = ok and (p // WARP == q // WARP if d < WARP else p // STEP > q // STEP)
            if ok:
                used[q:q + min(k, d)] = b"\1" * min(k, d)
                used[p:p + k + 1] = b"\1" * (k + 1)
                copies.append((q, p, k, L))
                break
        else:
            raise AssertionError("no room for length %d at distance %d" % (L, d))
    return _settle(buf, copies, rng)


def window_block():
    """A 4-byte string again 32,768 bytes later (a match) and another 32,769 bytes later (literals; nothing in between
    has its hash), and a third string at three places, the last matched to the middle one."""
    rng = np.random.default_rng(32768)
    copies = [(1000, 1000 + WINDOW, 4, 4), (3000, 3000 + WINDOW + 1, 4, -1), (20000, 21000, 4, 4), (21000, 30000, 4, 4)]
    return _settle(_random(rng, BLOCK, 64), copies, rng)


WINDOW_BLOCK_MISS = 3000 + WINDOW + 1            # where window_block's string 32,769 bytes back must stay literal


def collision_pair(seed=6):
    """Two different 4-byte strings with the same 13-bit hash."""
    rng = np.random.default_rng(seed)
    seen = {}
    while True:
        g = bytes(rng.integers(0, 256, size=4, dtype=np.uint8))
        h = int(hashes(g + b"\0")[1][0])
        if h in seen and seen[h] != g:
            return seen[h], g
        seen[h] = g


def warp_collision_block():
    """At p, the latest earlier lane of the warp has p's hash but other bytes; p's string is in the table from an earlier
    step, so p still matches."""
    rng = np.random.default_rng(66)
    ga, gb = collision_pair()
    buf = _random(rng, BLOCK, 64)
    q, r, p = 700, 5 * STEP + 3, 5 * STEP + 20
    for _ in range(200):
        buf[q:q + 4], buf[r:r + 4], buf[p:p + 4] = gb, ga, gb
        block = bytes(buf)
        x, h = hashes(block)
        cand = candidates(block)
        ok = (h[r] == h[p] and not (h[r + 1:p] == h[p]).any() and not (h[q + 1:p - p % STEP] == h[p]).any()
              and cand[p] == p - q and not (h[p - p % WARP:r] == h[p]).any())
        if ok and (p, p - q, 4) in parse(block, cand):
            return block, member(block)[1]
        buf = _random(rng, BLOCK, 64)
    raise AssertionError("no warp collision block")


WARP_COLLISION = (700, 5 * STEP + 3, 5 * STEP + 20)  # (table source, colliding lane, matched position)


def seam_block():
    """A copy across two segment seams, copies with 1 and 2 bytes left in their segment (literals, then a match from
    the next segment's first byte), and runs of period 1, 2 and 3 inside one segment."""
    rng = np.random.default_rng(128)
    buf = _random(rng, BLOCK, 64)
    copies = [(300, 4 * SEG + 100, 28, 28), (328, 5 * SEG, 128, 128), (456, 6 * SEG, 44, 44)]   # 200 bytes at 612
    for left in (1, 2):                            # 12 bytes from 3,000 back, starting `left` bytes before a seam
        s = (40 + 4 * left) * SEG
        copies += [(s - left - 3000, s - left, 12, 0), (s - 3000, s, 0, 12 - left)]
    for i, d in enumerate((1, 2, 3)):              # runs of 60 bytes at the start of segments 80, 84, 88
        s = (80 + 4 * i) * SEG
        copies.append((s, s + d, 60 - d, 60 - d))
    return _settle(buf, copies, rng)




def histogram_block(seed):
    """Every byte value 1 to 300 times (counts drawn from seed), shuffled: no 4-byte string repeats, so the block is all
    literals and its literal code follows the drawn counts, whose spread makes long literal and code-length codes."""
    rng = np.random.default_rng(seed)
    b = np.repeat(np.arange(256, dtype=np.uint8), rng.integers(1, 301, 256))
    rng.shuffle(b)
    return b[:BLOCK].tobytes()


def searched_histogram_block(reached):
    """The first histogram_block, by seed, whose model stats meet `reached`."""
    for seed in range(64):
        block = histogram_block(seed)
        st = member(block)[1]
        if reached(block, st):
            return block, st
    raise AssertionError("no seed below 64 reaches it")


def _literal_limited(b, st):
    return st["max_len"][0] == 15 and st["free_depth"][0] > 15 and not st["dist_used"] and not st["stored"]


def _code_lengths_limited(b, st):
    return st["max_len"][2] == 7 and st["free_depth"][2] > 7 and not st["stored"]


def stored_edge_block(repeat, dist=900):
    """Random bytes whose last `repeat` bytes copy those `dist` before them: the dynamic member's size minus the stored
    one's falls about a byte per repeated byte."""
    rng = np.random.default_rng(65311)
    buf = _random(rng, BLOCK)
    _write(buf, [(BLOCK - repeat - dist, BLOCK - repeat, repeat, None)])
    return bytes(buf)


def _has(st, *tokens):
    return set(tokens) <= set(st["tokens"])


def _literal_after_candidate(st, p, d):
    return (p, 0, 1) in st["tokens"] and st["cand"][p] == d


def _stored_edge(R, diff):
    return lambda: (stored_edge_block(R), None), \
        lambda b, st: st["dyn_size"] - st["stored_size"] == diff and st["stored"] == (diff >= 0)


def _plain(data):
    return lambda: (data, None)


def _seam_ok(b, st):
    runs = all(_has(st, ((80 + 4 * i) * SEG + d, d, 60 - d)) for i, d in enumerate((1, 2, 3)))
    cut = all(_literal_after_candidate(st, (40 + 4 * k) * SEG - k, 3000) and _has(st, ((40 + 4 * k) * SEG, 3000, 12 - k))
              for k in (1, 2))
    return runs and cut and _has(st, (612, 312, 28), (640, 312, 128), (768, 312, 44))


def _warp_collision_ok(b, st):
    q, r, p = WARP_COLLISION
    x, h = hashes(b)
    return h[r] == h[p] and x[r] != x[p] and st["cand"][p] == p - q and _has(st, (p, p - q, 4))


_GATTACA = b"GATTACA" * 10000

# name -> (build: () -> (block, stats or None), reached: (block, stats) -> bool). What each design is built to reach:
DESIGNS = {
    # a distance code of 15 bits, the unrestricted code being 16 deep (fl_huff_lengths_sorted's limiting step)
    "fifteen_bit_distance": (fifteen_bit_block, lambda b, st: st["max_len"][1] == 15 and st["free_depth"][1] == 16),
    # a literal code of 15 bits in an all-literal block, the unrestricted code being 16 deep
    "fifteen_bit_literal": (lambda: searched_histogram_block(_literal_limited), _literal_limited),
    # a code-length code of 7 bits, the unrestricted one being 8 deep (the limit FL_BGZF_MAX_CL_BITS at work)
    "seven_bit_code_lengths": (lambda: searched_histogram_block(_code_lengths_limited), _code_lengths_limited),
    # match lengths 3..128 and distance codes 0..29: the largest HLIT (281) and HDIST (30)
    "all_symbols": (all_symbols_block, lambda b, st: st["hlit"] == 281 and st["hdist"] == 30
                    and {t[2] for t in st["tokens"] if t[1]} >= set(range(3, 129)) and len(st["dist_used"]) == 30),
    # one used distance symbol, 0 (the dummy is 1) or 2 (the dummy is 0); a block without matches (two dummies)
    "one_distance_code_0": (_plain(b"A" * 512), lambda b, st: st["dist_used"] == [0] and st["dhist"][:2] == [st["dhist"][0], 1]),
    "one_distance_code_2": (_plain(b"ABC" * 170), lambda b, st: st["dist_used"] == [2] and st["dhist"][0] == 1),
    "no_match": (_plain(bytes(np.random.default_rng(100).integers(0, 256, 100, dtype=np.uint8))),
                 lambda b, st: st["dist_used"] == [] and st["dhist"][:2] == [1, 1] and st["hdist"] == 2),
    # a match at distance 32,768, literals at 32,769, and the table keeping the latest of three
    "window": (window_block, lambda b, st: _has(st, (1000 + WINDOW, WINDOW, 4), (30000, 9000, 4), (21000, 1000, 4))
               and (WINDOW_BLOCK_MISS, 0, 1) in st["tokens"] and st["cand"][WINDOW_BLOCK_MISS] == 0 and not st["stored"]),
    # an in-warp candidate that fails the byte check, the position falling back to the table
    "warp_collision": (warp_collision_block, lambda b, st: _warp_collision_ok(b, st) and not st["stored"]),
    # copies across segment seams, with 1 or 2 bytes left in a segment, and runs with d < L
    "seams": (seam_block, lambda b, st: _seam_ok(b, st) and not st["stored"]),
    # the stored / dynamic choice: dynamic minus stored size +1 and 0 (stored), -1 (dynamic)
    "stored_edge_plus_1": _stored_edge(56, 1),
    "stored_edge_tie": _stored_edge(57, 0),
    "stored_edge_minus_1": _stored_edge(58, -1),
}
# short last blocks (1 to 3 bytes have no hashed position), and a full one
for _n in (1, 2, 3, 4, 5, 127, 128, 129, 130, BLOCK):
    DESIGNS["last_%d" % _n] = (_plain(_GATTACA[:_n]),
                              lambda b, st, n=_n: len(b) == n and (any(st["cand"]) if n > 7 else not any(st["cand"])))

_built = {}


def designed(name):
    """(block, stats) of a designed block."""
    if name not in _built:
        block, st = DESIGNS[name][0]()
        _built[name] = (block, st if st is not None else member(block)[1])
    return _built[name]

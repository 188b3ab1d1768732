"""Exact models of the short-read 16-mer build (`-1` / `-2`), and designed inputs that reach each of its paths.

The reference builds its set from short reads with an order-dependent state machine (kmers.cpp:142-166): a 16-mer
enters the set at its 4th sighting, or at its 3rd if its FIRST sighting was a false positive of the Bloom filter (13
salted hashes into 1,917,295,480 bits). fl_kmers.cu computes a closed, order-free form of that machine instead:
every add has an index t in the add stream (file, record, position, forward before reverse), and

    FP(X)     <=>  every Bloom bit of X was set by the first sighting of some 16-mer before t_first(X)
    X in set  <=>  cnt(X) >= 4  or  (cnt(X) == 3 and FP(X))

Here both are written down plainly over an explicit add stream (`sequential_set`, `closed_form_set`), with the add
stream built from reads exactly as k_kmers_add orders it (`add_stream`). The Bloom hash inverts in closed form
(`cover`), so a 16-mer that sets any chosen bit can be written down, and reads placed before, between or after the
sightings of a 16-mer X decide whether X reaches the set through the false-positive clause. `designs()` builds those
inputs; each names its 16-mers with the membership they must have and the path that gives it.
"""
import numpy as np

K = 16
TABLE_BITS = 1917295480                     # bloom_filter.h as configured by kmers.cpp:29-36
SALTS = (0x1B5793D2, 0x81BDFA38, 0xEB8E30D5, 0x45B52496, 0x85C1FE3C, 0x3DACB627, 0x78776869,
         0x94A40D1E, 0x5F9BB638, 0x40FB59D5, 0x8174BDB2, 0x0B466EAA, 0x209D29A7)
M32 = 0xFFFFFFFF

FWD = {ord(c): v for c, v in zip("ACGTacgt", (0, 1, 2, 3, 0, 1, 2, 3))}   # kmers.cpp:176-196, anything else 0
REV = {ord(c): v for c, v in zip("TGCAtgca", (0, 1, 2, 3, 0, 1, 2, 3))}   # kmers.cpp:199-219 (<< 30), anything else 0


# ---- the Bloom hash and its inverse ---------------------------------------------------------------------------------
def bloom_hash(kmer, salt):
    """bloom_filter.h's hash_ap for a 4-byte key: s ^ ~((s << 11) + (k ^ (s >> 5)))"""
    return (salt ^ ~((((salt << 11) & M32) + (kmer ^ (salt >> 5))) & M32)) & M32


def bloom_bits(kmer, table_bits=TABLE_BITS, salts=SALTS):
    return [bloom_hash(kmer, s) % table_bits for s in salts]


def bloom_bits_np(kmers, table_bits=TABLE_BITS, salts=SALTS):
    """[n, len(salts)] bit indices of many 16-mers at once"""
    k = np.asarray(kmers, dtype=np.uint64)[:, None]
    s = np.asarray(salts, dtype=np.uint64)[None, :]
    m = np.uint64(M32)
    h = (s ^ (~((((s << np.uint64(11)) & m) + (k ^ (s >> np.uint64(5)))) & m) & m)) & m
    return h % np.uint64(table_bits)


def cover(bit, j, wrap=0, table_bits=TABLE_BITS, salts=SALTS):
    """The 16-mer whose hash under salt j is bit + wrap * table_bits (so it sets `bit`), or None past 2^32."""
    h = bit + wrap * table_bits
    if h > M32:
        return None
    s = salts[j]
    return (((~(h ^ s) & M32) - ((s << 11) & M32)) & M32) ^ (s >> 5)


# ---- 16-mers and reads ----------------------------------------------------------------------------------------------
def kmer_seq(kmer):
    """the 16 bases of a forward 16-mer code (first base in the top bits)"""
    return bytes(b"ACGT"[(kmer >> (30 - 2 * i)) & 3] for i in range(K))


def seq_kmer(seq):
    k = 0
    for c in seq[:K]:
        k = (k << 2) | FWD.get(c, 0)
    return k


def rc(kmer):
    """the reverse complement of a 16-mer code"""
    x = ~kmer & M32
    r = 0
    for _ in range(K):
        r = (r << 2) | (x & 3)
        x >>= 2
    return r


def rc_np(kmers):
    x = ~np.asarray(kmers, dtype=np.uint32)
    r = np.zeros_like(x)
    for _ in range(K):
        r = (r << np.uint32(2)) | (x & np.uint32(3))
        x = x >> np.uint32(2)
    return r


def read_adds(seq):
    """[(forward, reverse) per position] of one read (kmers.cpp:99-121); a read shorter than 16 adds nothing"""
    out = []
    if len(seq) < K:
        return out
    fwd = rev = 0
    for i, c in enumerate(seq):
        fwd = ((fwd << 2) & M32) | FWD.get(c, 0)
        rev = (rev >> 2) | (REV.get(c, 0) << 30)
        if i >= K - 1:
            out.append((fwd, rev))
    return out


def add_stream(files):
    """The add stream of k_kmers_add: files in order, records in order, per position the forward 16-mer (t = 2p) before
    the reverse one (t = 2p + 1), t counted across records and files. Returns a list of 16-mers (index = t)."""
    stream = []
    for reads in files:
        for seq in reads:
            for f, r in read_adds(seq):
                stream.append(f)
                stream.append(r)
    return stream


def assembly_set(seqs):
    """kmers.cpp:137-139: every forward and reverse 16-mer of the assembly"""
    s = set()
    for seq in seqs:
        for f, r in read_adds(seq):
            s.add(f)
            s.add(r)
    return s


# ---- the two models -------------------------------------------------------------------------------------------------
def sequential_set(stream, members=(), table_bits=TABLE_BITS, salts=SALTS, trace=None):
    """kmers.cpp:142-166 add by add. `members`: the set before the first add (an assembly's 16-mers). `trace`, a dict,
    receives per 16-mer whether its first sighting hit a false positive of the filter."""
    kmers = set(members)
    bloom = set()
    counts = {}
    for x in stream:
        if x in kmers:
            continue
        bits = bloom_bits(x, table_bits, salts)
        if not all(b in bloom for b in bits):
            bloom.update(bits)
            if trace is not None:
                trace.setdefault(x, False)
        elif x not in counts:
            counts[x] = 2
            if trace is not None:
                trace.setdefault(x, True)
        else:
            counts[x] += 1
            if counts[x] >= 4:
                kmers.add(x)
                del counts[x]
    return kmers


def closed_form_set(stream, members=(), table_bits=TABLE_BITS, salts=SALTS, detail=None):
    """fl_kmers.cu's closed form: cnt (saturating at 4) and t_first per 16-mer not in `members`, bit_time per Bloom bit
    = min t_first over the 16-mers touching it, then cnt >= 4, or cnt == 3 and bit_time < t_first on all 13 bits.
    `detail`, a dict, receives per 16-mer (cnt, t_first, fp, number of its bits with bit_time < t_first)."""
    members = set(members)
    cnt, t_first = {}, {}
    for t, x in enumerate(stream):
        if x in members:                    # has_bit: an assembly 16-mer never counts, nor sets a Bloom time
            continue
        if x not in t_first:
            t_first[x] = t
        cnt[x] = min(cnt.get(x, 0) + 1, 4)
    bit_time = {}
    for x, t in t_first.items():
        for b in bloom_bits(x, table_bits, salts):
            if t < bit_time.get(b, 1 << 64):
                bit_time[b] = t
    out = set(members)
    for x, c in cnt.items():
        covered = sum(bit_time[b] < t_first[x] for b in bloom_bits(x, table_bits, salts))
        fp = covered == len(salts)
        if detail is not None:
            detail[x] = (c, t_first[x], fp, covered)
        if c >= 4 or (c == 3 and fp):
            out.add(x)
    return out


# ---- designs --------------------------------------------------------------------------------------------------------
# 16-mers found by a search over random X (numpy: `search_self_cover` / `search_neighbour_cover` with the seeds named),
# frozen here; tests/test_bloom_model.py checks the property each was chosen for.
#   SELF_COVER: (X, j, j') with bit j of X == bit j' of rc(X): a read of rc(X) sets one of X's bits with its forward
#       16-mer just before it adds X as its reverse one (about 1 X in 10^7). Seeds 3 and 5.
#   NEIGHBOUR_COVER: (X, c, j) with bit j of X set by rc(c + X[:15]): in the read c + X, the reverse 16-mer at position
#       0 sets it just before X is added as the forward one at position 1. Seeds 4 and 6.
SELF_COVER = ((1369130566, 10, 9), (60486580, 1, 12))
NEIGHBOUR_COVER = ((1906612580, 1, 4), (519751898, 2, 3))


def search_self_cover(seed, batch=1 << 20, max_batches=64):
    """X such that one of rc(X)'s Bloom bits is one of X's: returns (X, j, j')"""
    rng = np.random.default_rng(seed)
    for _ in range(max_batches):
        x = rng.integers(0, 1 << 32, size=batch, dtype=np.uint64).astype(np.uint32)
        x = x[x != rc_np(x)]                     # a palindrome shares all its bits with itself
        bx, br = bloom_bits_np(x), bloom_bits_np(rc_np(x))
        eq = bx[:, :, None] == br[:, None, :]
        hit = np.nonzero(eq.any(axis=(1, 2)))[0]
        if hit.size:
            i = int(hit[0])
            j, jj = map(int, np.argwhere(eq[i])[0])
            return int(x[i]), j, jj
    return None


def search_neighbour_cover(seed, batch=1 << 20, max_batches=64):
    """X and a base c such that rc(c + X[:15]) -- the reverse 16-mer at p when X is the forward one at p + 1 -- sets one
    of X's Bloom bits: returns (X, c, j)"""
    rng = np.random.default_rng(seed)
    for _ in range(max_batches):
        x = rng.integers(0, 1 << 32, size=batch, dtype=np.uint64).astype(np.uint32)
        bx = bloom_bits_np(x)
        for c in range(4):
            w = rc_np((np.uint32(c) << np.uint32(30)) | (x >> np.uint32(2)))
            br = bloom_bits_np(w)
            eq = (bx[:, :, None] == br[:, None, :]) & (w != x)[:, None, None]
            hit = np.nonzero(eq.any(axis=(1, 2)))[0]
            if hit.size:
                i = int(hit[0])
                return int(x[i]), c, int(np.argwhere(eq[i])[0][0])
    return None


def palindrome(rng):
    half = rng.integers(0, 1 << 16)
    return int(half) << 16 | rc(int(half)) >> 16       # 8 bases, then their reverse complement


class Design:
    """One input of the short-read build: `files` (the -1 file's reads, the -2 file's), `assembly` (-a, may be empty) and
    the named 16-mers it was built for. expect[name] = (16-mer, member, path); path is (sightings, Bloom bits set before
    the first sighting) with sightings saturating at 4, or None where only the membership is written down (a reverse
    complement, a palindrome's single sighting pair)."""

    def __init__(self, name, seed):
        self.name = name
        self.rng = np.random.default_rng(seed)
        self.files = [[], []]
        self.assembly = []
        self.expect = {}

    def x(self):
        while True:
            k = int(self.rng.integers(0, 1 << 32))
            if k != rc(k):
                return k

    def covers(self, x, which=range(13), shift=1):
        """one 16-base read per chosen bit of x: the 16-mer whose hash under another salt lands on that bit"""
        bits = bloom_bits(x)
        return [kmer_seq(cover(bits[j], (j + shift) % 13)) for j in which]

    def want(self, label, kmer, member, sightings=None, covered=None, rc_member=None):
        self.expect[label] = (kmer, member, None if sightings is None else (sightings, covered))
        if rc_member is not None:
            self.expect["rc(%s)" % label] = (rc(kmer), rc_member, None)

    def fillers(self, n_bytes):
        """records shorter than 16 bases (they add nothing to the stream) making more than n_bytes of FASTQ"""
        n = n_bytes // 20                         # a record takes at least 10 bytes besides its bases
        lens = self.rng.integers(1, 16, size=n)
        bases = np.frombuffer(b"ACGT", np.uint8)[self.rng.integers(0, 4, size=int(lens.sum()))].tobytes()
        ends = np.cumsum(lens)
        return [bases[e - L:e] for e, L in zip(ends.tolist(), lens.tolist())]


def _d1_covered_before():
    d = Design("covered_before_first_sighting", 101)
    S1 = d.files[0]
    x = d.x(); S1 += d.covers(x) + [kmer_seq(x)] * 3; d.want("covered", x, True, 3, 13, rc_member=False)
    x = d.x(); S1 += [kmer_seq(x)] * 3; d.want("not_covered", x, False, 3, 0, rc_member=False)
    x = d.x(); S1 += d.covers(x) + [kmer_seq(x)] * 2; d.want("covered_twice", x, False, 2, 13, rc_member=False)
    x = d.x(); S1 += [kmer_seq(x)] * 4; d.want("four", x, True, 4, 0, rc_member=True)
    x = d.x(); S1 += d.covers(x, range(12)) + [kmer_seq(x)] * 3; d.want("12_of_13", x, False, 3, 12, rc_member=False)
    return d


def _d2_last_cover():
    d = Design("last_cover_around_first_sighting", 102)
    S1 = d.files[0]
    x = d.x(); c = d.covers(x)
    S1 += c[:12] + [kmer_seq(x), c[12]] + [kmer_seq(x)] * 2; d.want("next_record", x, False, 3, 12, rc_member=False)
    x = d.x(); c = d.covers(x)
    S1 += c[:12] + [kmer_seq(x) + c[12]] + [kmer_seq(x)] * 2; d.want("later_position", x, False, 3, 12, rc_member=False)
    x = d.x(); c = d.covers(x)                # a 1-base record between: it adds nothing, so X stays after the cover
    S1 += c[:12] + [c[12], b"G"] + [kmer_seq(x)] * 3; d.want("record_before", x, True, 3, 13, rc_member=False)
    x = d.x(); c = d.covers(x)
    S1 += c[:12] + [c[12] + kmer_seq(x)] + [kmer_seq(x)] * 2; d.want("position_before", x, True, 3, 13, rc_member=False)
    return d


def _d3_strand_order(i, first_as_reverse):
    """X's first sighting and the 16-mer setting its last bit are the two strands of one position"""
    x, j, _ = SELF_COVER[i]
    d = Design("strand_order_%s" % ("cover_forward" if first_as_reverse else "cover_reverse"), 103 + i)
    others = [jj for jj in range(13) if jj != j]
    if first_as_reverse:      # read rc(X): rc(X) forward at t = 2p sets bit j, X reverse at 2p + 1
        d.files[0] += d.covers(x, others) + [kmer_seq(rc(x))] + [kmer_seq(x)] * 2
        d.want("x", x, True, 3, 13, rc_member=False)
    else:                     # read X: X forward at 2p, rc(X) reverse at 2p + 1 sets bit j too late
        d.files[0] += d.covers(x, others) + [kmer_seq(x)] * 3
        d.want("x", x, False, 3, 12, rc_member=False)
    return d


def _d4_position_order(i, cover_first):
    """the reverse 16-mer at p against X's first sighting at p + 1 (cover_first), or X reverse at p against the
    forward 16-mer at p + 1"""
    x, c, j = NEIGHBOUR_COVER[i]
    d = Design("position_order_%s" % ("cover_first" if cover_first else "x_first"), 105 + i)
    others = [jj for jj in range(13) if jj != j]
    read = b"ACGT"[c:c + 1] + kmer_seq(x)       # reverse at p = 0 sets bit j (t = 1), X forward at p = 1 (t = 2)
    if cover_first:
        d.files[0] += d.covers(x, others) + [read] + [kmer_seq(x)] * 2
        d.want("x", x, True, 3, 13, rc_member=False)
    else:                     # the read backwards: X reverse at p = 0 (t = 1), the cover forward at p = 1 (t = 2)
        d.files[0] += d.covers(x, others) + [_revcomp(read)] + [kmer_seq(x)] * 2
        d.want("x", x, False, 3, 12, rc_member=False)
    return d


def _d5_across_files():
    d = Design("across_files", 107)
    S1, S2 = d.files
    xa, xb = d.x(), d.x()
    cb = d.covers(xb)
    S1 += d.covers(xa) + cb[:12] + [kmer_seq(xb)]
    S2 += [cb[12]] + [kmer_seq(xb)] * 2 + [kmer_seq(xa)] * 3
    d.want("covers_in_1_x_in_2", xa, True, 3, 13, rc_member=False)
    d.want("x_in_1_last_cover_in_2", xb, False, 3, 12, rc_member=False)
    return d


def _d6_assembly_covers():
    d = Design("assembly_covers", 108)
    xa, xb = d.x(), d.x()
    d.assembly = d.covers(xa)                # in the set before the short reads: skipped, their Bloom bits never set
    d.files[0] += d.covers(xa) + [kmer_seq(xa)] * 3 + d.covers(xb) + [kmer_seq(xb)] * 3
    d.want("assembly_covers", xa, False, 3, 0, rc_member=False)
    d.want("read_covers", xb, True, 3, 13, rc_member=False)
    return d


def _d7_n_mask_cover():
    """the last bit's cover exists only as the reverse 16-mer of a window with an N (reverse strand: N -> 0, kmers.cpp:
    199-219), not as the reverse complement of the window's forward 16-mer (N -> A there, so T on the other strand)"""
    d = Design("n_mask_cover", 109)
    x = d.x()
    bit = bloom_bits(x)[12]
    for salt in range(13):
        k = cover(bit, salt)
        zero = [q for q in range(K) if (k >> (2 * q)) & 3 == 0]
        if salt != 12 and zero:
            break
    w = bytearray(b"TGCA"[(k >> (2 * q)) & 3] for q in range(K))   # reverse code of base q at bits 2q
    w[zero[0]] = ord("N")
    d.files[0] += d.covers(x, range(12)) + [bytes(w)] + [kmer_seq(x)] * 3
    d.want("x", x, True, 3, 13, rc_member=False)
    d.n_cover = k
    return d


def _d8_palindromes():
    d = Design("palindromes", 110)
    S1 = d.files[0]
    p1, p2, p3 = (palindrome(d.rng) for _ in range(3))
    S1 += d.covers(p1) + [kmer_seq(p1)]; d.want("one_read_covered", p1, False, 2, 13)
    S1 += [kmer_seq(p2)]; d.want("one_read", p2, False, 2, 0)
    S1 += [kmer_seq(p3)] * 2; d.want("two_reads", p3, True, 4, 0)
    return d


def _d9_chunk_seams():
    """more than 1 MiB of records between the covers and X, so that text chunks of 1 MiB put seams there"""
    d = Design("chunk_seams", 111)
    xa, xb = d.x(), d.x()
    cb = d.covers(xb)
    d.files[0] += d.covers(xa) + cb[:12] + [kmer_seq(xb)] + d.fillers(1100 << 10) + [cb[12], kmer_seq(xa)]
    d.seam_filler = len(d.files[0]) - 3      # a filler record past the first MiB (the CR LF variant's)
    d.files[0] += d.fillers(1100 << 10) + [kmer_seq(xa)] * 2 + [kmer_seq(xb)] * 2
    d.want("covered_across_seams", xa, True, 3, 13, rc_member=False)
    d.want("last_cover_across_seams", xb, False, 3, 12, rc_member=False)
    return d


def _revcomp(seq):
    comp = bytes.maketrans(b"ACGTNacgtn", b"TGCANtgcan")
    return seq.translate(comp)[::-1]


def designs():
    return [_d1_covered_before(), _d2_last_cover(), _d3_strand_order(0, True), _d3_strand_order(1, False),
            _d4_position_order(0, True), _d4_position_order(1, False), _d5_across_files(), _d6_assembly_covers(),
            _d7_n_mask_cover(), _d8_palindromes(), _d9_chunk_seams()]


def model_set(files, assembly=(), **kw):
    """the set of a design's input by the closed form (the sequential model gives the same: tests/test_bloom_model.py)"""
    return closed_form_set(add_stream(files), assembly_set(assembly), **kw)


def combined(ds):
    """all designs in one input: the -1 files one after another, the -2 files likewise, the assemblies together"""
    files = [[r for d in ds for r in d.files[0]], [r for d in ds for r in d.files[1]]]
    return files, [a for d in ds for a in d.assembly]


# ---- the combined designs as files ----------------------------------------------------------------------------------
def long_reads(ds, seed=112):
    """one FASTQ read per named 16-mer of the designs: random bases around it, so that under k-mer scoring a read's mean
    quality is > 0 exactly when its 16-mer is in the set (and `--min_mean_q 1` keeps exactly those reads)"""
    rng = np.random.default_rng(seed)
    lut = np.frombuffer(b"ACGT", np.uint8)
    out = []
    for d in ds:
        for label, (k, _, _) in d.expect.items():
            a, b = (int(v) for v in rng.integers(40, 400, size=2))
            seq = lut[rng.integers(0, 4, size=a)].tobytes() + kmer_seq(k) + lut[rng.integers(0, 4, size=b)].tobytes()
            qual = (rng.integers(5, 40, size=len(seq)).astype(np.uint8) + 33).tobytes()
            out.append(("%s:%s" % (d.name, label), seq, qual))
    return out


def write_combined(directory, ds, gz=False, crlf=False):
    """the designs' combined -1 / -2 files, assembly and long reads under `directory`. crlf: one record of the chunk-seam
    design's filler past its first MiB ends its lines with CR LF (the CLI hands the rest of the file to its host reader
    from that chunk on). Returns {"S1", "S2", "A", "FQ"}: paths."""
    import gzip
    import os
    files, asm = combined(ds)
    seam = None
    if crlf:
        base = 0
        for d in ds:
            if hasattr(d, "seam_filler"):
                seam = base + d.seam_filler
            base += len(d.files[0])
    out = {}
    for tag, reads in (("S1", files[0]), ("S2", files[1])):
        parts = []
        for i, seq in enumerate(reads):
            nl = b"\r\n" if i == seam else b"\n"
            parts.append(b"@%s_%d" % (tag.encode(), i) + nl + seq + nl + b"+" + nl + b"I" * len(seq) + nl)
        path = os.path.join(directory, "%s.fastq%s" % (tag.lower(), ".gz" if gz else ""))
        with (gzip.open(path, "wb", compresslevel=1) if gz else open(path, "wb")) as f:
            f.write(b"".join(parts))
        out[tag] = path
    out["A"] = os.path.join(directory, "asm.fasta")
    with open(out["A"], "wb") as f:
        f.write(b"".join(b">c%d\n%s\n" % (i, s) for i, s in enumerate(asm)))
    out["FQ"] = os.path.join(directory, "reads.fastq")
    with open(out["FQ"], "wb") as f:
        f.write(b"".join(b"@%s\n%s\n+\n%s\n" % (n.encode(), s, q) for n, s, q in long_reads(ds)))
    return out


def cli_args(paths, with_assembly=True):
    return (["-a", paths["A"]] if with_assembly else []) + ["-1", paths["S1"], "-2", paths["S2"], "--min_mean_q", "1", paths["FQ"]]


def count_line(stderr):
    """the "N reads, M 16-mers" line of the short-read build (kmers.cpp:56-57), without its progress redraws"""
    lines = [l.split("\r")[-1].strip() for l in stderr.split("\n")]
    i = lines.index("Hashing 16-mers from short reads")
    return next(l for l in lines[i + 1:] if l.endswith("16-mers"))

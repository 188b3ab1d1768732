"""The test model of unaligned BAM input (filtlong_b200/csrc/host/bam.h): a small BAM writer with arbitrary aux fields, a
reader, the FASTQ equivalent of a BAM file, and the BAM the CLI is expected to write for given scoring results."""
import gzip
import struct

import numpy as np

from tests import bgzf_util

SEQ_CODES = b"=ACMGRSVTWYHKDBN"
_CODE_OF = {c: i for i, c in enumerate(SEQ_CODES)}
FIXED = struct.Struct("<iiBBHHHiiii")          # refID pos l_read_name mapq bin n_cigar_op flag l_seq next_refID next_pos tlen


# ---- aux fields ----
def aux_z(tag, value):
    return tag + b"Z" + value + b"\0"


def aux_f(tag, value):
    return tag + b"f" + struct.pack("<f", value)


def aux_i(tag, value):
    return tag + b"i" + struct.pack("<i", value)


def aux_b(tag, sub, values):
    fmt = {b"c": "b", b"C": "B", b"s": "h", b"S": "H", b"i": "i", b"I": "I", b"f": "f"}[sub]
    return tag + b"B" + sub + struct.pack("<I", len(values)) + struct.pack("<%d%s" % (len(values), fmt), *values)


# ---- writer ----
def pack_seq(seq):
    codes = [_CODE_OF[c] for c in seq]
    if len(codes) % 2:
        codes.append(0)
    return bytes((codes[i] << 4) | codes[i + 1] for i in range(0, len(codes), 2))


def record(name, seq, qual=None, aux=b"", flag=4, cigar=(), mapq=255, bin_=4680, ref_id=-1, pos=-1, next_ref_id=-1, next_pos=-1,
           tlen=0, l_read_name=None, l_seq=None):
    """One BAM record (block_size included). qual: Phred values (bytes) or None for none (0xFF). l_read_name / l_seq
    override the fields for malformed records."""
    q = bytes(qual) if qual is not None else b"\xff" * len(seq)
    cig = b"".join(struct.pack("<I", c) for c in cigar)
    body = FIXED.pack(ref_id, pos, len(name) + 1 if l_read_name is None else l_read_name, mapq, bin_, len(cigar), flag,
                      len(seq) if l_seq is None else l_seq, next_ref_id, next_pos, tlen)
    body += name + b"\0" + cig + pack_seq(seq) + q + aux
    return struct.pack("<I", len(body)) + body


def header(text=b"@HD\tVN:1.6\tSO:unknown\n@RG\tID:rg1\tSM:s\n", refs=()):
    h = b"BAM\1" + struct.pack("<I", len(text)) + text + struct.pack("<I", len(refs))
    for name, length in refs:
        h += struct.pack("<I", len(name) + 1) + name + b"\0" + struct.pack("<I", length)
    return h


def bgzf(raw):
    """BGZF of the uncompressed stream, ending with the EOF member: a BAM file."""
    return bgzf_util.zlib_bgzf(raw) + bgzf_util.EOF_MEMBER


# ---- reader ----
def header_end(raw):
    assert raw[:4] == b"BAM\1"
    p = 8 + struct.unpack_from("<I", raw, 4)[0]
    n_ref = struct.unpack_from("<I", raw, p)[0]
    p += 4
    for _ in range(n_ref):
        p += 4 + struct.unpack_from("<I", raw, p)[0] + 4
    return p


def records(raw):
    """The records of an uncompressed BAM stream: dicts with their offsets in it and their decoded fields."""
    out, p = [], header_end(raw)
    while p < len(raw):
        bs = struct.unpack_from("<I", raw, p)[0]
        ref_id, pos, l_name, mapq, bin_, n_cigar, flag, l_seq, nref, npos, tlen = FIXED.unpack_from(raw, p + 4)
        name_off = p + 36
        seq_off = name_off + l_name + 4 * n_cigar
        qual_off = seq_off + (l_seq + 1) // 2
        aux_off = qual_off + l_seq
        nib = np.frombuffer(raw[seq_off:qual_off], np.uint8)
        codes = np.stack([nib >> 4, nib & 15], 1).reshape(-1)[:l_seq]
        q = raw[qual_off:aux_off]
        out.append(dict(start=p, size=4 + bs, name=raw[name_off:name_off + l_name - 1], name_off=name_off, name_len=l_name - 1,
                        seq_off=seq_off, qual_off=qual_off, len=l_seq, flag=flag,
                        seq=np.frombuffer(SEQ_CODES, np.uint8)[codes].tobytes(),
                        qual=None if l_seq and q[0] == 0xFF else q, aux=raw[aux_off:p + 4 + bs], fixed=raw[p + 4:p + 36]))
        p += 4 + bs
    return out


def inflate(path_or_bytes):
    data = path_or_bytes if isinstance(path_or_bytes, bytes) else open(path_or_bytes, "rb").read()
    return gzip.decompress(data)


def aux_fields(aux):
    """[(tag, raw bytes of the whole field)]"""
    out, p = [], 0
    sizes = {b"A": 1, b"c": 1, b"C": 1, b"s": 2, b"S": 2, b"i": 4, b"I": 4, b"f": 4}
    while p < len(aux):
        t = aux[p + 2:p + 3]
        if t in (b"Z", b"H"):
            e = aux.index(b"\0", p + 3) + 1
        elif t == b"B":
            e = p + 8 + struct.unpack_from("<I", aux, p + 4)[0] * sizes[aux[p + 3:p + 4]]
        else:
            e = p + 3 + sizes[t]
        out.append((aux[p:p + 2], aux[p:e]))
        p = e
    return out


# ---- the FASTQ equivalent and the expected output ----
def to_fastq(raw):
    """The FASTQ equivalent of a BAM stream: name = read_name, no comment; SEQ decoded; QUAL + 33, or a FASTA record
    when QUAL starts with 0xFF."""
    out = []
    for r in records(raw):
        if r["qual"] is None:
            out.append(b">" + r["name"] + b"\n" + r["seq"] + b"\n")
        else:
            out.append(b"@" + r["name"] + b"\n" + r["seq"] + b"\n+\n" + bytes((x + 33) & 255 for x in r["qual"]) + b"\n")
    return b"".join(out)


def child_record(raw, r, s, e):
    """The record of the child [s, e) of record r: the parent's fixed fields, name_<s+1>-<e>, the slice, RG only."""
    name = r["name"] + b"_%d-%d" % (s + 1, e)
    fixed = bytearray(r["fixed"])
    fixed[8] = len(name) + 1
    struct.pack_into("<i", fixed, 16, e - s)
    qual = b"\xff" * (e - s) if r["qual"] is None else r["qual"][s:e]
    rg = b"".join(f for tag, f in aux_fields(r["aux"]) if tag == b"RG")
    body = bytes(fixed) + name + b"\0" + pack_seq(r["seq"][s:e]) + qual + rg
    return struct.pack("<I", len(body)) + body


def expected_output(raw, results):
    """The uncompressed BAM pass 2 writes. results[i] = (n_child, [(start, end, passed), ...]) as the survivor tests
    give them (a read without children has one row)."""
    out = bytearray(raw[:header_end(raw)])
    for r, (n_child, rows) in zip(records(raw), results):
        if n_child == 0:
            if rows[0][2]:
                out += raw[r["start"]:r["start"] + r["size"]]
            continue
        for s, e, passed in rows:
            if passed and e - s > 0:
                out += child_record(raw, r, s, e)
    return bytes(out)


def name_hash(name):
    """fl_name_hash.h, restated"""
    m = (1 << 64) - 1
    h = 0xCBF29CE484222325
    for c in name:
        h = ((h ^ c) * 0x100000001B3) & m
    h ^= h >> 29
    h = (h * 0xBF58476D1CE4E5B9) & m
    h ^= h >> 32
    return h


def random_reads(rng, n, lo=1, hi=3000, no_qual_every=0, n_frac=0.02):
    """(name, seq, qual or None, aux) reads with IUPAC codes, names of odd and even lengths, the usual aux fields."""
    acgt = np.frombuffer(b"ACGT", np.uint8)
    out = []
    for i in range(n):
        L = int(rng.integers(lo, hi + 1))
        seq = bytearray(acgt[rng.integers(0, 4, size=L)].tobytes())
        for p in rng.integers(0, L, size=max(1, int(L * n_frac))) if rng.random() < 0.5 else []:
            seq[p] = SEQ_CODES[int(rng.integers(0, 16))]
        name = b"read_%d" % i + b"x" * int(rng.integers(0, 3))
        qual = None if no_qual_every and i % no_qual_every == 3 else np.clip(rng.normal(14, 5, L), 1, 60).astype(np.uint8).tobytes()
        aux = b""
        if i % 3 != 2:
            aux += aux_z(b"RG", b"rg1")
        aux += aux_f(b"qs", float(rng.uniform(5, 30)))
        if i % 2 == 0:
            aux += aux_z(b"MM", b"C+m?,1,0,3;") + aux_b(b"ML", b"C", [int(x) for x in rng.integers(0, 256, size=3)])
        if i % 5 == 1:
            aux += aux_b(b"fi", b"S", [int(x) for x in rng.integers(0, 65536, size=L)])
        out.append((name, bytes(seq), qual, aux))
    return out


def bam_of(reads, hdr=None):
    """uncompressed BAM stream of (name, seq, qual, aux) reads"""
    return (hdr if hdr is not None else header()) + b"".join(record(n, s, q, a) for n, s, q, a in reads)

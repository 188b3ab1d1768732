"""The test model of aligned BAM input (--aligned, filtlong_b200/csrc/host/bam.h): aligned records built with
bam_util.record, a seeded coordinate-sorted file of reads with supplementary and secondary records, the FASTQ equivalent
(what `samtools fastq` writes: read records only, reverse-complemented where flag 0x10 is set), the walker's index and
the BAM that pass 2 writes for given pass flags."""
import numpy as np

from tests import bam_util as bu

OPS = {c: i for i, c in enumerate("MIDNSHP=X")}
# samtools' complement of the 16 SEQ codes "=ACMGRSVTWYHKDBN"
_COMP = dict(zip(b"=ACMGRSVTWYHKDBN", b"=TGKCYSBAWRDMHVN"))
READ_MASK, REVERSE = 0x900, 0x10


def cigar(text):
    """'5S10M2I' -> the packed operations"""
    out, num = [], ""
    for ch in text:
        if ch.isdigit():
            num += ch
        else:
            out.append(int(num) << 4 | OPS[ch])
            num = ""
    return tuple(out)


def revcomp(seq):
    return bytes(_COMP[c] for c in reversed(seq))


def is_read(r):
    return r["flag"] & READ_MASK == 0


def primary_cigar(rng, L):
    """a CIGAR whose query length is L: soft clips, matches, an insertion and a deletion"""
    if L < 12:
        return "%dM" % L
    s0, s1, ins = int(rng.integers(0, L // 4)), int(rng.integers(0, L // 4)), int(rng.integers(1, 4))
    m = L - s0 - s1 - ins
    a = m // 2
    return ("%dS" % s0 if s0 else "") + "%dM%dI2D%dM" % (a, ins, m - a) + ("%dS" % s1 if s1 else "")


def aligned_reads(rng, reads, n_refs=2, ref_len=10 ** 6, sup_max=3, secondary_every=5, unmapped_every=9):
    """(ref_id, pos, record bytes) of the reads (name, seq, qual or None, aux) and their followers, unsorted. A read is
    forward, reverse or unmapped (some unmapped ones with 0x10 too); it has 0 to sup_max hard-clipped supplementary
    records and, every secondary_every-th, a secondary record with SEQ '*'."""
    out = []
    for i, (name, seq, qual, ax) in enumerate(reads):
        L = len(seq)
        unmapped = i % unmapped_every == 4
        rev = bool(i % 2) if unmapped else bool(rng.random() < 0.5)
        stored = revcomp(seq) if rev else seq
        squal = None if qual is None else (qual[::-1] if rev else qual)
        ref, pos = int(rng.integers(0, n_refs)), int(rng.integers(0, ref_len))
        if unmapped:
            out.append((-1, -1, bu.record(name, stored, squal, ax, flag=4 | (REVERSE if rev else 0))))
            continue
        out.append((ref, pos, bu.record(name, stored, squal, ax, flag=REVERSE if rev else 0, cigar=cigar(primary_cigar(rng, L)),
                                        ref_id=ref, pos=pos, mapq=60)))
        for _ in range(int(rng.integers(0, sup_max + 1))):
            a = int(rng.integers(0, L))
            b = int(rng.integers(a + 1, L + 1))
            srev = bool(rng.random() < 0.5)
            piece = stored[a:b] if not srev else revcomp(stored[a:b])
            pq = None if squal is None else (squal[a:b] if not srev else squal[a:b][::-1])
            cg = ("%dH" % a if a else "") + "%dM" % (b - a) + ("%dH" % (L - b) if L - b else "")
            sref, spos = int(rng.integers(0, n_refs)), int(rng.integers(0, ref_len))
            out.append((sref, spos, bu.record(name, piece, pq, bu.aux_z(b"SA", b"chr1,1,+,5M,60,0;"), flag=0x800 | (REVERSE if srev else 0),
                                              cigar=cigar(cg), ref_id=sref, pos=spos, mapq=20)))
        if i % secondary_every == 1:
            sref, spos = int(rng.integers(0, n_refs)), int(rng.integers(0, ref_len))
            out.append((sref, spos, bu.record(name, b"", b"", b"", flag=0x100, cigar=cigar("%dM" % L), ref_id=sref, pos=spos, mapq=0)))
    return out


def sorted_bam(recs, n_refs=2, ref_len=10 ** 6):
    """the uncompressed BAM of (ref_id, pos, record) records, coordinate-sorted (unmapped last, stable)"""
    hdr = bu.header(text=b"@HD\tVN:1.6\tSO:coordinate\n@RG\tID:rg1\tSM:s\n",
                    refs=[(b"chr%d" % (k + 1), ref_len) for k in range(n_refs)])
    order = sorted(range(len(recs)), key=lambda k: (recs[k][0] < 0, recs[k][0], recs[k][1], k))
    return hdr + b"".join(recs[k][2] for k in order)


def to_fastq(raw):
    """the FASTQ equivalent: the read records only, each in its original orientation"""
    out = []
    for r in bu.records(raw):
        if not is_read(r):
            continue
        seq, qual = r["seq"], r["qual"]
        if r["flag"] & REVERSE:
            seq = revcomp(seq)
            qual = None if qual is None else qual[::-1]
        if qual is None:
            out.append(b">" + r["name"] + b"\n" + seq + b"\n")
        else:
            out.append(b"@" + r["name"] + b"\n" + seq + b"\n+\n" + bytes((x + 33) & 255 for x in qual) + b"\n")
    return b"".join(out)


def model_index(raw):
    """(reads, followers) as the walker indexes them: reads (name_off, name_len, seq_off, qual_off, len, name_hash,
    reverse); followers (offset, reads before it, name_hash, index of the read of its name or -1)"""
    reads, followers, by_name = [], [], {}
    for r in bu.records(raw):
        if is_read(r):
            by_name[r["name"]] = len(reads)
            reads.append((r["name_off"], r["name_len"], r["seq_off"], r["qual_off"], r["len"], bu.name_hash(r["name"]),
                          1 if r["flag"] & REVERSE else 0))
        else:
            followers.append([r["start"], len(reads), bu.name_hash(r["name"]), r["name"]])
    return reads, [(s, b, h, by_name.get(n, -1)) for s, b, h, n in followers]


def expected_output(raw, passed, want):
    """the uncompressed BAM pass 2 writes: the header, then every record whose read's pass flag (passed: by read name)
    is `want`, in input order; an orphan only when want is false"""
    out = bytearray(raw[:bu.header_end(raw)])
    for r in bu.records(raw):
        if bool(passed.get(r["name"], False)) == want:
            out += raw[r["start"]:r["start"] + r["size"]]
    return bytes(out)

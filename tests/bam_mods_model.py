"""The test model of `--keep_mods` (filtlong_b200/csrc/fl_bam_mods.h): the base-modification tags of an unaligned BAM
record (SAMtags 1.7: MM:Z, ML:B:C, MN) parsed and checked, re-based to a child [s, e), and -- written apart from both,
sharing no code with them -- a decoder from tags to the calls they make, which the tests hold every child to."""
import re
import struct

from tests import bam_util as bu

KEPT, INVALID = 1, 2
_COUNTED = {"A": "A", "C": "C", "G": "G", "T": "T", "U": "T"}


# ---- parse / validate ----
def tags_of(aux):
    """(fields, error): fields maps RG / MM / ML / MN to the raw fields (RG: a list, in order), plus 'order', the
    MM / ML tags in the parent's order; error is None when no tag appears twice and the types are right."""
    f = {"RG": [], "order": []}
    err = None
    for tag, raw in bu.aux_fields(aux):
        t = tag.decode()
        if t == "RG":
            f["RG"].append(raw)
        elif t in ("MM", "ML", "MN"):
            if t in f:
                err = "duplicate " + t
            f[t] = raw
            if t != "MN":
                f["order"].append(t)
    if "MM" in f and f["MM"][2:3] != b"Z":
        err = err or "MM is not Z"
    if "ML" in f and f["ML"][2:4] != b"BC":
        err = err or "ML is not B:C"
    return f, err


_GROUP = re.compile(rb"([ACGTUN])([+-])([a-z]+|[0-9]+)([.?]?)((?:,[0-9]+)*);")


def parse_mm(mm):
    """[(base, strand, codes, flag, [delta texts])] or None when MM:Z does not parse or a delta is 2^32 or more"""
    groups, p = [], 0
    while p < len(mm):
        m = _GROUP.match(mm, p)
        if not m:
            return None
        deltas = m.group(5).split(b",")[1:]
        if any(int(d) >= 1 << 32 for d in deltas):
            return None
        groups.append((m.group(1).decode(), m.group(2).decode(), m.group(3).decode(), m.group(4).decode(), deltas))
        p = m.end()
    return groups


def n_codes(codes):
    return 1 if codes.isdigit() else len(codes)


def base_positions(seq, base):
    """the SEQ positions a group of this base counts"""
    if base == "N":
        return list(range(len(seq)))
    want = _COUNTED[base]
    return [i for i, c in enumerate(seq.decode()) if c == want]


def valid_tags(seq, aux):
    """(groups, ml values or None) when the record's tags are valid, else None"""
    f, err = tags_of(aux)
    if err or "MM" not in f:
        return None
    groups = parse_mm(f["MM"][3:-1])
    if groups is None:
        return None
    total = 0
    for base, _, codes, _, deltas in groups:
        if deltas:
            last = sum(int(d) + 1 for d in deltas) - 1
            if last >= len(base_positions(seq, base)):
                return None
        total += len(deltas) * n_codes(codes)
    ml = None
    if "ML" in f:
        ml = list(f["ML"][8:])
        if len(ml) != total:
            return None
    if "MN" in f:
        t = f["MN"][2:3]
        fmt = {b"c": "<b", b"C": "<B", b"s": "<h", b"S": "<H", b"i": "<i", b"I": "<I"}.get(t)
        if fmt is None or struct.unpack(fmt, f["MN"][3:])[0] != len(seq):
            return None
    return groups, ml


# ---- re-base ----
def rebase(seq, aux, s, e):
    """(aux bytes of the child [s, e) after its RG fields, status): the re-based MM / ML in the parent's order and MN:I,
    or b"" when the tags are missing or invalid."""
    f, _ = tags_of(aux)
    v = valid_tags(seq, aux)
    if v is None:
        return b"", (INVALID if "MM" in f else 0)
    groups, ml = v
    mm_out, ml_out, ml_at = b"", b"", 0
    for base, strand, codes, flag, deltas in groups:
        nc = n_codes(codes)
        before_s = sum(1 for p in base_positions(seq, base) if p < s)
        before_e = sum(1 for p in base_positions(seq, base) if p < e)
        idx, kept = -1, []
        for k, d in enumerate(deltas):
            idx += int(d) + 1
            if before_s <= idx < before_e:
                kept.append((k, idx, d))
        text = b"".join(b"," + (str(idx - before_s).encode() if j == 0 else d) for j, (k, idx, d) in enumerate(kept))
        mm_out += (base + strand + codes + flag).encode() + text + b";"
        if ml is not None:
            ml_out += bytes(ml[ml_at + k * nc + c] for k, _, _ in kept for c in range(nc))
        ml_at += len(deltas) * nc
    fields = {"MM": b"MMZ" + mm_out + b"\0"}
    if ml is not None:
        fields["ML"] = b"MLBC" + struct.pack("<I", len(ml_out)) + ml_out
    return b"".join(fields[t] for t in f["order"]) + b"MNI" + struct.pack("<I", e - s), KEPT


def child_record(raw, r, s, e, keep_mods):
    """bam_util.child_record plus, with keep_mods, the re-based tags; and the child's status"""
    rec = bu.child_record(raw, r, s, e)
    if not keep_mods:
        return rec, 0
    extra, status = rebase(r["seq"], r["aux"], s, e)
    body = rec[4:] + extra
    return struct.pack("<I", len(body)) + body, status


def expected_output(raw, results, keep_mods):
    """bam_util.expected_output with keep_mods; returns (stream, [kept, invalid])"""
    out = bytearray(raw[:bu.header_end(raw)])
    counts = [0, 0]
    for r, (n_child, rows) in zip(bu.records(raw), results):
        if n_child == 0:
            if rows[0][2]:
                out += raw[r["start"]:r["start"] + r["size"]]
            continue
        for s, e, passed in rows:
            if passed and e - s > 0:
                rec, st = child_record(raw, r, s, e, keep_mods)
                out += rec
                if st:
                    counts[st - 1] += 1
    return bytes(out), counts


# ---- decode, written apart from the two above ----
def decode(seq, aux):
    """the calls of a record's tags: sorted [(SEQ position, strand, code, probability)] (probability None without ML)"""
    fields = dict(bu.aux_fields(aux))
    mm = fields[b"MM"][3:-1].decode()
    ml = fields[b"ML"][8:] if b"ML" in fields else None
    calls, v = [], 0
    for group in mm.split(";")[:-1]:
        parts = group.split(",")
        head = parts[0]
        base, strand, rest = head[0], head[1], head[2:].rstrip(".?")
        codes = [rest] if rest.isdigit() else list(rest)
        counted = base if base in "ACGTN" else "T"
        where = [i for i, c in enumerate(seq.decode()) if counted == "N" or c == counted]
        pos = -1
        for d in parts[1:]:
            pos += int(d) + 1
            for code in codes:
                calls.append((where[pos], strand, code, None if ml is None else ml[v]))
                v += 1
    return sorted(calls)

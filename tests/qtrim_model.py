"""The model of `--trim_q Q` in numpy / Python.

A base is good iff it lies in a run of 16 consecutive bases whose quality bytes are all >= 33 + Q. Good plays the role
that "in a reference 16-mer" plays in k-mer mode, so the rows follow the reference's read.cpp:75-143 and main.cpp:139-147
with "base i is good" for "qualities[i] != 0". A child's mean / window quality is the Phred score of its own substring,
and a read without child ranges is its own row, whole."""
import numpy as np

from oracle import oracle as orc

K = 16


def good_mask(qual: bytes, Q: int) -> np.ndarray:
    """bool per base: inside a run of K bases whose quality bytes (unsigned) are all >= 33 + Q"""
    q = np.frombuffer(qual, dtype=np.uint8)
    L = q.size
    if L < K:
        return np.zeros(L, dtype=bool)
    c = np.concatenate(([0], np.cumsum(q >= 33 + Q)))
    starts = np.nonzero(c[K:] - c[:-K] == K)[0]
    d = np.zeros(L + 1, dtype=np.int64)
    np.add.at(d, starts, 1)
    np.add.at(d, starts + K, -1)
    return np.cumsum(d[:L]) > 0


def good_mask_brute(qual: bytes, Q: int) -> np.ndarray:
    """the definition, base by base"""
    q = list(qual)
    L = len(q)
    return np.array([any(all(x >= 33 + Q for x in q[s:s + K]) for s in range(max(0, i - K + 1), i + 1) if s + K <= L)
                     for i in range(L)], dtype=bool)


def rows(mask, L, trim, split):
    """read.cpp:75-143 on a good-base mask: dict(first, last, bad, children); split None = not set"""
    mask = np.asarray(mask, dtype=bool)
    idx = np.nonzero(mask)[0]
    first = int(idx[0]) if idx.size else -1
    last = int(idx[-1]) + 1 if idx.size else -1
    bad, children = [], []
    if trim or split is not None:
        if split is not None:
            i = 0
            while i < L:
                if not mask[i]:
                    s = i
                    while i < L and not mask[i]:
                        i += 1
                    if i - s >= split:
                        bad.append((s, i))
                else:
                    i += 1
        if trim:
            if first > 0 and (not bad or bad[0] != (0, first)):
                bad.insert(0, (0, first))
            if last != -1 and last < L and (not bad or bad[-1] != (last, L)):
                bad.append((last, L))
        if bad:
            rs = 0
            for s, e in bad:
                if s - rs > 0:
                    children.append((rs, s))
                rs = e
            if L - rs > 0:
                children.append((rs, L))
    return dict(first=first, last=last, bad=bad, children=children)


def crafted():
    """(name, qualities, Q): the edges of the definition and of the device's word layout"""
    lo, hi = b"#", b"5"                                  # Phred 2 and 20
    cases = [
        ("run of 15", lo * 40 + hi * 15 + lo * 40, 20),
        ("run of 16", lo * 40 + hi * 16 + lo * 40, 20),
        ("runs at both ends", hi * 16 + lo * 100 + hi * 20, 20),
        ("all good", hi * 300, 20),
        ("length 1", hi, 20),
        ("length 15", hi * 15, 20),
        ("length 16", hi * 16, 20),
        ("bytes >= 128", bytes([200]) * 20 + lo * 10 + bytes([128]) * 16 + bytes([127]) * 16, 93),
        ("Q = 1", b"\"" * 16 + b"!" * 5 + b"\"" * 15, 1),
        ("Q = 93", b"~" * 16 + b"}" * 16, 93),
    ]
    for edge in (32, 64, 1024):
        for off in range(-16, 1):                      # runs crossing base edge-1 / edge
            q = bytearray(lo * (edge + 100))
            q[edge + off:edge + off + 16] = hi * 16
            cases.append(("run at %d%+d" % (edge, off), bytes(q), 20))
    return cases


def read_rows(reads, Q, trim, split):
    """per read (seq, qual, ...): rows() of its good mask"""
    return [rows(good_mask(r[1], Q), len(r[0]), trim, split) for r in reads]


def score_rows(reads, Q, params_kw):
    """oracle.Scored of a --trim_q run, finalised. reads: (seq, qual); params_kw: oracle.make_params keywords (trim and
    split included). Parents and children are scored by the oracle in plain Phred mode, children on their substrings."""
    plain = {k: v for k, v in params_kw.items() if k not in ("trim", "split")}
    op = orc.make_params(**plain)
    parents, bads, kids = [], [], []
    total = 0
    model = read_rows(reads, Q, params_kw.get("trim", False), params_kw.get("split"))
    for i, ((seq, qual), m) in enumerate(zip(reads, model)):
        p = orc.score([(seq, qual)], op).parents[0]
        p.parent, p.start, p.end = i, 0, len(seq)
        p.first, p.last, p.n_bad, p.n_child = m["first"], m["last"], len(m["bad"]), len(m["children"])
        ch = []
        for s, e in m["children"]:
            c = orc.score([(seq[s:e], qual[s:e])], op).parents[0]
            c.parent, c.start, c.end = i, s, e
            ch.append(c)
        parents.append(p)
        bads.append(m["bad"])
        kids.append(ch)
        total += len(seq)
    sc = orc.Scored(parents, bads, kids, total_bases=total)
    return orc.finalize(sc, orc.make_params(**params_kw))


def derived_reads(reads, Q, trim, split):
    """one record per row: (name, comment, seq, qual) with the child name name_<s+1>-<e> and the parent's comment.
    reads: (name, comment, seq, qual)"""
    out = []
    for (name, comment, seq, qual), m in zip(reads, read_rows([(r[2], r[3]) for r in reads], Q, trim, split)):
        if not m["children"]:
            out.append((name, comment, seq, qual))
        for s, e in m["children"]:
            out.append(("%s_%d-%d" % (name, s + 1, e), comment, seq[s:e], qual[s:e]))
    return out


def fastq_bytes(records):
    """FASTQ text of (name, comment, seq, qual) records"""
    return b"".join(b"@" + name.encode() + ((b" " + comment) if comment else b"") + b"\n" + seq + b"\n+\n" + qual + b"\n"
                    for name, comment, seq, qual in records)


def derived_target(target_bases, keep_percent, input_bases):
    """-t T for the derived run: main.cpp:229-237 on the INPUT's bases"""
    t = target_bases if target_bases is not None else (1 << 63) - 1
    if keep_percent is not None:
        t = min(t, int((keep_percent / 100.0) * input_bases))
    return t

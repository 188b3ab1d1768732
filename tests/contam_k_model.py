"""A numpy model of the contaminant set of k-mers longer than 16 (`--contam_k K`, DESIGN.md §4.12) and of a read's
contaminant percentage c against it, plus a brute-force string version of both that the model is checked against.

The set: every window of K bases of a record that holds only ACGTacgt adds min(forward, reverse complement), as 2-bit codes
(A 0, C 1, G 2, T 3) with the first base in the high bits; case does not matter. The log's count M is the number of forward
and reverse k-mers: 2 x canonical - palindromes. A read's bases are its 2-bit codes, a non-ACGT base being A. A base is
covered when a k-mer that contains it is in the set on either strand; c = 100.0 * covered / L (NaN for an empty read)."""
import numpy as np

_CODE = np.zeros(256, dtype=np.uint64)
for _c, _v in zip(b"ACGTacgt", [0, 1, 2, 3, 0, 1, 2, 3]):
    _CODE[_c] = _v
_VALID = np.zeros(256, dtype=bool)
_VALID[np.frombuffer(b"ACGTacgt", np.uint8)] = True


def _windows(codes, k):
    """forward and reverse-complement k-mers of every window start (len(codes) - k + 1 of them)"""
    n = len(codes) - k + 1
    fwd = np.zeros(n, dtype=np.uint64)
    rc = np.zeros(n, dtype=np.uint64)
    for j in range(k):
        c = codes[j:j + n]
        fwd = (fwd << np.uint64(2)) | c
        rc |= (np.uint64(3) - c) << np.uint64(2 * j)
    return fwd, rc


def canonical(fwd, k):
    """min(forward, reverse complement) of forward k-mers (uint64 array)"""
    fwd = np.asarray(fwd, dtype=np.uint64)
    rc = revcomp(fwd, k)
    return np.minimum(fwd, rc)


def revcomp(fwd, k):
    fwd = np.asarray(fwd, dtype=np.uint64)
    rc = np.zeros_like(fwd)
    x = fwd.copy()
    for _ in range(k):
        rc = (rc << np.uint64(2)) | (np.uint64(3) - (x & np.uint64(3)))
        x >>= np.uint64(2)
    return rc


def record_kmers(seq, k):
    """canonical k-mers of one contaminant record's ACGT-only windows, and which of them are palindromes"""
    a = np.frombuffer(seq, dtype=np.uint8)
    if len(a) < k:
        return np.zeros(0, np.uint64), np.zeros(0, bool)
    fwd, rc = _windows(_CODE[a], k)
    bad = np.concatenate([[0], np.cumsum(~_VALID[a])])
    ok = bad[k:] - bad[:-k] == 0
    return np.minimum(fwd, rc)[ok], (fwd == rc)[ok]


def kmer_set(records, k):
    """(sorted unique canonical k-mers, M = forward and reverse members)"""
    parts = [record_kmers(s, k) for s in records]
    keys = np.concatenate([p[0] for p in parts] + [np.zeros(0, np.uint64)])
    pal = np.concatenate([p[0][p[1]] for p in parts] + [np.zeros(0, np.uint64)])
    u = np.unique(keys)
    return u, 2 * len(u) - len(np.unique(pal))


def read_codes(seq):
    return _CODE[np.frombuffer(seq, dtype=np.uint8)]


def percent(seq, members, k):
    """c of one read against the sorted canonical members"""
    L = len(seq)
    if L == 0:
        return np.float64(np.nan)
    if L < k or len(members) == 0:
        return np.float64(100.0) * np.float64(0) / np.float64(L)
    fwd, rc = _windows(read_codes(seq), k)
    key = np.minimum(fwd, rc)
    i = np.searchsorted(members, key)
    hit = (i < len(members)) & (members[np.minimum(i, len(members) - 1)] == key)
    d = np.zeros(L + 1, dtype=np.int64)
    s = np.nonzero(hit)[0]
    np.add.at(d, s, 1)
    np.add.at(d, s + k, -1)
    covered = int((np.cumsum(d)[:L] > 0).sum())
    return np.float64(100.0) * np.float64(covered) / np.float64(L)


def percents(reads, members, k):
    return np.array([percent(s, members, k) for s in reads], dtype=np.float64)


# ---- brute force: strings, slices and a Python set ---------------------------------------------------------------------
_RC = bytes.maketrans(b"ACGT", b"TGCA")


def _bf_code(w):
    v = 0
    for ch in w:
        v = (v << 2) | b"ACGT".index(ch)
    return v


def brute_set(records, k):
    canon, pal = set(), set()
    for s in records:
        u = s.upper()
        for i in range(len(u) - k + 1):
            w = u[i:i + k]
            if w.strip(b"ACGT"):
                continue
            r = w.translate(_RC)[::-1]
            m = min(w, r)                      # A < C < G < T in ASCII as in 2-bit codes
            canon.add(_bf_code(m))
            if w == r:
                pal.add(_bf_code(m))
    return canon, 2 * len(canon) - len(pal)


def brute_percent(seq, canon, k):
    L = len(seq)
    if L == 0:
        return float("nan")
    u = bytes(ch if ch in b"ACGT" else ord("A") for ch in seq.upper())
    covered = [False] * L
    for i in range(L - k + 1):
        w = u[i:i + k]
        if min(_bf_code(w), _bf_code(w.translate(_RC)[::-1])) in canon:
            for j in range(i, i + k):
                covered[j] = True
    return 100.0 * sum(covered) / L

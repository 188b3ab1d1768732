"""The one-copy 16-mer build (kmers.cpp:75-134, 137-139, 176-225) restated in numpy, without the C oracle (no GPU).

Every sequence of 16 or more bases adds, at each start s, its forward 16-mer (A/a 0, C/c 1, G/g 2, T/t 3, any other
byte 0; first base in the high bits) and its reverse 16-mer (the complement, newest base on top, where a non-ACGT byte
is 0 again rather than the complement of 0). A sequence under 16 bases adds nothing but is counted. `build` returns the
sorted members, the number of sequences and the bases of the sequences that take part: what fl_kmers_add_text reports.

Two wrong builds sit beside it, so that a test can show its designs tell them apart from the right one: a non-ACGT byte
complemented on the reverse strand like A, and a window holding a non-ACGT byte adding nothing.
"""
import numpy as np

K = 16
CODE = np.zeros(256, dtype=np.uint32)
ACGT = np.zeros(256, dtype=bool)
for _c, _v in zip(b"ACGTacgt", (0, 1, 2, 3, 0, 1, 2, 3)):
    CODE[_c] = _v
    ACGT[_c] = True


def _windows(seqs):
    """the concatenated bytes and, per 16-mer start, its index there (the starts of every sequence of >= 16 bases)"""
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    a = np.frombuffer(b"".join(seqs), dtype=np.uint8)
    first = np.cumsum(lens) - lens                              # where each sequence begins in `a`
    n_win = np.maximum(lens - (K - 1), 0)
    first_win = np.cumsum(n_win) - n_win                        # where each sequence's starts begin in the output
    starts = np.repeat(first - first_win, n_win) + np.arange(int(n_win.sum()))
    return a, starts, lens


def _kmers(starts, fwd_code, rev_code):
    """forward and reverse 16-mers at `starts` of the code arrays (computed at every index, then picked)"""
    n = max(len(fwd_code) - (K - 1), 0)
    fwd = np.zeros(n, dtype=np.uint32)
    rev = np.zeros(n, dtype=np.uint32)
    for j in range(K):
        fwd = (fwd << np.uint32(2)) | fwd_code[j:j + n]
        rev |= rev_code[j:j + n] << np.uint32(2 * j)            # base j of the window: bits 2j+1:2j of the reverse
    return fwd[starts], rev[starts]


def _build(seqs, rev_of_other, drop_other_windows):
    seqs = [bytes(s) for s in seqs]
    a, starts, lens = _windows(seqs)
    c = CODE[a]
    ok = ACGT[a]
    rc = np.where(ok, np.uint32(3) - c, np.uint32(rev_of_other)).astype(np.uint32)
    fwd, rev = _kmers(starts, c, rc)
    if drop_other_windows and len(starts):
        bad = np.concatenate([[0], np.cumsum(~ok, dtype=np.int64)])
        keep = bad[starts + K] == bad[starts]
        fwd, rev = fwd[keep], rev[keep]
    members = np.unique(np.concatenate([fwd, rev]))
    return members, len(seqs), int(lens[lens >= K].sum())


def build(seqs):
    """(sorted members, sequences, bases of the sequences of >= 16 bases) of an assembly made of `seqs` (bytes)"""
    return _build(seqs, 0, False)


def build_n_complemented(seqs):
    """wrong: a non-ACGT byte is complemented on the reverse strand like A (to T, 3)"""
    return _build(seqs, 3, False)


def build_skipping_other_windows(seqs):
    """wrong: a window that holds any non-ACGT byte adds nothing"""
    return _build(seqs, 0, True)


_FWD_DIGITS = bytes.maketrans(b"ACGTacgt", b"01230123")
_REV_DIGITS = bytes.maketrans(b"ACGTacgt", b"32103210")
_OTHER_TO_ZERO = bytes(b if b in b"ACGTacgt" else ord("0") for b in range(256))


def brute_force(seqs):
    """the same set one 16-mer at a time with Python strings: slice, translate to base-4 digits, int(..., 4)"""
    out = set()
    for s in seqs:
        s = bytes(s)
        for i in range(len(s) - K + 1):
            w = s[i:i + K]
            out.add(int(w.translate(_OTHER_TO_ZERO).translate(_FWD_DIGITS), 4))
            out.add(int(w[::-1].translate(_OTHER_TO_ZERO).translate(_REV_DIGITS), 4))
    return np.array(sorted(out), dtype=np.uint32)

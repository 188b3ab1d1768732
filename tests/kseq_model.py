"""The reference's input semantics in plain Python: klib's kseq_read (reference src/kseq.h:98-151, 182-224) byte by byte,
and the two loops that consume it, the reads loop (src/main.cpp:76-125) and the reference-file loop
(src/kmers.cpp:88-134). The device parser (fl_text.cu) and the host reader (csrc/host/fastx.cpp) are both held to it.

kseq_read's rules, as followed here:
  * with no header character pending, skip bytes up to the next '>' or '@', wherever it is (kseq.h:187-191); -1 at EOF;
  * the name runs up to the first C-locale isspace byte, which is consumed (kseq.h:193, ks_getuntil KS_SEP_SPACE); -1
    when the stream ends right after the header character;
  * unless that byte was '\\n', the rest of the line is the comment (kseq.h:194);
  * sequence lines follow until a line starts with '>', '+' or '@'; an empty line is skipped; the first byte of each line
    is taken as it is, the rest of the line is appended (kseq.h:199-203); '>' or '@' is kept as the next header character
    (kseq.h:204); anything but '+' (EOF included) ends a FASTA record (kseq.h:211-212);
  * FASTQ: the rest of the '+' line is skipped, -2 if the stream ends inside it (kseq.h:217-218); quality lines are
    appended until the quality is at least as long as the sequence or the stream ends (kseq.h:219); -2 when the lengths
    differ (kseq.h:222); the next call skips to a header character again (kseq.h:221);
  * every line read through ks_getuntil(KS_SEP_LINE) loses one trailing '\\r' when the string it was appended to is
    then longer than one byte (kseq.h:146) -- and only when the call read anything (kseq.h:142): the first byte of a
    sequence line is appended by ks_getc, so a line that is that one byte at the very end of the stream keeps its '\\r'.

A record's byte extents (`name_off`, `seq_off`, `qual_off`) are reported where the record is one slice of the input: one
sequence line, one quality line, nothing stripped (`plain`). -3 (a stream error) cannot happen on bytes in memory.
"""
import dataclasses

SPACE = frozenset(b" \t\n\v\f\r")          # isspace() in the C locale


@dataclasses.dataclass
class Record:
    ret: int                      # kseq_read's return: the sequence length, or -2
    name: bytes
    comment: bytes
    seq: bytes
    qual: bytes
    is_fastq: bool
    start: int                    # offset of the header character
    end: int                      # offset one past the last byte the record consumed
    name_off: int
    seq_off: int = -1             # first byte of the first sequence line (-1: none)
    qual_off: int = -1
    seq_lines: int = 0
    qual_lines: int = 0
    stripped_cr: bool = False

    @property
    def cname(self):
        """the name as the reference uses it: a C string (main.cpp:81,90,99,114)"""
        return cstr(self.name)

    @property
    def plain(self):
        """the record is one slice of the input: name, comment, sequence and quality lie there as they are"""
        return self.ret >= 0 and not self.stripped_cr and self.seq_lines == 1 and (not self.is_fastq or self.qual_lines == 1)


def cstr(b):
    z = b.find(b"\0")
    return b if z < 0 else b[:z]


class KSeq:
    def __init__(self, data):
        self.d = bytes(data)
        self.pos = 0
        self.last_char = 0

    def _getc(self):
        if self.pos >= len(self.d):
            return -1
        c = self.d[self.pos]
        self.pos += 1
        return c

    def _getuntil(self, s, space):
        """ks_getuntil2 into bytearray s (appending): -1 when nothing was read at EOF, else (length, delimiter or 0)"""
        d, n = self.d, len(self.d)
        if self.pos >= n:
            return -1, 0
        i = self.pos
        if space:
            while i < n and d[i] not in SPACE:
                i += 1
        else:
            i = d.find(b"\n", i)
            i = n if i < 0 else i
        s += d[self.pos:i]
        dret = d[i] if i < n else 0
        self.pos = i + 1 if i < n else n
        stripped = False
        if not space and len(s) > 1 and s[-1] == 13:
            del s[-1]
            stripped = True
        return len(s), dret, stripped

    def read(self):
        """One kseq_read: -1 at the end, else a Record (ret >= 0, or -2)."""
        if self.last_char == 0:
            c = self._getc()
            while c >= 0 and c not in (62, 64):
                c = self._getc()
            if c < 0:
                return -1
            self.last_char = c
        start = self.pos - 1                  # the header character, read by this call or by the one before
        name = bytearray()
        r = self._getuntil(name, True)
        if r[0] < 0:
            return -1
        c = r[1]
        rec = Record(0, b"", b"", b"", b"", False, start, 0, start + 1)
        comment = bytearray()
        if c != 10:
            r = self._getuntil(comment, False)
            if r[0] >= 0 and r[2]:
                rec.stripped_cr = True
        seq = bytearray()
        while True:
            c = self._getc()
            if c < 0 or c in (62, 43, 64):
                break
            if c == 10:
                continue
            if rec.seq_lines == 0:
                rec.seq_off = self.pos - 1
            rec.seq_lines += 1
            seq.append(c)
            r = self._getuntil(seq, False)
            if r[0] >= 0 and r[2]:
                rec.stripped_cr = True
        if c in (62, 64):
            self.last_char = c
        rec.name, rec.comment, rec.seq = bytes(name), bytes(comment), bytes(seq)
        rec.is_fastq = c == 43
        if not rec.is_fastq:
            rec.ret = len(seq)
            rec.end = self.pos - 1 if c in (62, 64) else self.pos
            return rec
        c = self._getc()
        while c >= 0 and c != 10:
            c = self._getc()
        if c == -1:
            rec.ret, rec.end = -2, self.pos
            return rec
        rec.qual_off = self.pos
        qual = bytearray()
        while True:
            r = self._getuntil(qual, False)
            if r[0] < 0:
                break
            rec.qual_lines += 1
            if r[2]:
                rec.stripped_cr = True
            if len(qual) >= len(seq):
                break
        self.last_char = 0
        rec.qual = bytes(qual)
        rec.end = self.pos
        rec.ret = len(seq) if len(seq) == len(qual) else -2
        return rec


def kseq_all(data):
    """Every kseq_read of `data` up to and including the first negative return: a list of Records, then -1 when the
    stream ended normally (a -2 Record is the list's last element otherwise)."""
    k, out = KSeq(data), []
    while True:
        r = k.read()
        if r == -1:
            return out + [-1]
        out.append(r)
        if r.ret < 0:
            return out


@dataclasses.dataclass
class ReadsResult:
    records: list                 # the Records read, in order
    total_bases: int
    error: list                   # the reference's error lines (stderr, without blank lines), [] when it goes on
    fasta: bool = False           # the output format (main.cpp:133-134)
    fastq: bool = False

    @property
    def log_line(self):
        """what the reads loop's last progress line says (misc.cpp:47-49, without the thousands separators)"""
        return "%d reads (%d bp)" % (len(self.records), self.total_bases)


def reads_loop(data, have_kmers):
    """main.cpp:76-125 over `data`: the records the reference scores, or the error it stops with."""
    recs, total, any_fasta, any_fastq, names = [], 0, False, False, set()
    for r in kseq_all(data):
        if r == -1:
            break
        if r.ret == -2:
            return ReadsResult(recs, total, ["Error: incorrect FASTQ format for read " + r.cname.decode("latin-1")])
        total += len(r.seq)
        fasta_format = len(r.qual) == 0 and len(r.seq) > 0
        fastq_format = len(r.qual) > 0 and len(r.seq) > 0 and len(r.qual) == len(r.seq)
        any_fasta, any_fastq = any_fasta or fasta_format, any_fastq or fastq_format
        if any_fasta and any_fastq:
            return ReadsResult(recs, total, ["Error: could not parse input reads",
                                             "  problem occurred at read " + r.cname.decode("latin-1")])
        if fasta_format and not have_kmers:
            return ReadsResult(recs, total, ["Error: FASTA input not supported without an external reference"])
        recs.append(r)
        if r.cname in names:
            return ReadsResult(recs, total, ["Error: duplicate read name: " + r.cname.decode("latin-1")])
        names.add(r.cname)
    return ReadsResult(recs, total, [], any_fasta, any_fastq)


def reference_loop(data):
    """kmers.cpp:88-134 over `data`: (records counted, bases hashed, the records). Hashing stops silently at the first
    negative return; every record is counted, but only those of 16 bases or more are hashed and add to the bases."""
    recs = [r for r in kseq_all(data) if r != -1 and r.ret >= 0]
    return len(recs), sum(len(r.seq) for r in recs if len(r.seq) >= 16), recs


def pass2_output(data, keep=None):
    """main.cpp:263-311 without children: the records of `data` the reads loop accepted, printed as the reference prints
    them -- lead character by the output format, the C-string name, " " and the comment as a C string when the comment
    has any byte, the sequence and (FASTQ) the quality as C strings. `keep`: a predicate on the record index."""
    res = reads_loop(data, True)
    assert not res.error
    out = bytearray()
    for i, r in enumerate(res.records):
        if keep is not None and not keep(i):
            continue
        out += (b">" if res.fasta else b"@") + r.cname
        if r.comment:
            out += b" " + cstr(r.comment)
        out += b"\n" + cstr(r.seq) + b"\n"
        if res.fastq:
            out += b"+\n" + cstr(r.qual) + b"\n"
    return bytes(out)


def record_starts_at(b, p, fastq):
    """csrc/host/textsrc.cpp's cut rule: may a chunk start at byte p (the start of a line)?"""
    if p >= len(b):
        return False
    if not fastq:
        return b[p] == 62
    if b[p] != 64:
        return False
    eol = lambda i: (lambda j: len(b) if j < 0 else j)(b.find(b"\n", i)) if i < len(b) else len(b)
    e0 = eol(p)
    s1 = e0 + 1
    e1 = eol(s1)
    s2 = e1 + 1
    if e1 <= s1 or b[s1] in b"@>+":
        return False
    if s2 >= len(b) or b[s2] != 43:
        return False
    e2 = eol(s2)
    s3 = e2 + 1
    e3 = eol(s3)
    return s3 <= len(b) and e3 - s3 == e1 - s1


def plan_cuts(b, fastq, target):
    """Chunk starts as textsrc.cpp's plan_chunks() places them: the last record start at or before every `target`
    bytes; None when no such start exists (the host reader then parses the whole file)."""
    cuts, pos = [0], 0
    while len(b) - pos > target:
        p = pos + target
        found = False
        while p > pos:
            q = b.rfind(b"\n", pos, p)
            if q < 0:
                break
            cand = q + 1
            if cand > pos and record_starts_at(b, cand, fastq):
                found = True
                break
            p = cand - 1
        if not found:
            return None
        cuts.append(cand)
        pos = cand
    return cuts + [len(b)]

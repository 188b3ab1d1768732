"""The device FASTQ / FASTA parser (fl_text.cu) against the reference's input semantics (tests/kseq_model.py).

A seeded generator starts from clean FASTQ, 2-line FASTA and wrapped FASTA and applies mutations of the kinds where a
line-based parser and kseq part ways. The device may hand any chunk back (FALLBACK: the host reader, which follows kseq,
parses it); what it accepts must be exactly what the reference reads. On the CPU the model is pinned to the host reader
and to recorded runs of the reference CLI; on the GPU every fuzz input goes through fl_reads_push_text (Phred and k-mer
mode) and fl_kmers_add_text (FASTQ, 2-line FASTA, wrapped FASTA), whole and cut into chunks the way textsrc.cpp cuts
them, and a set of them through the CLI on every input path."""
import collections
import gzip
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from tests import kseq_model as km

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "filtlong_b200", "csrc", "host")
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")

CLASSES = ["seq_lead", "empty_fasta", "blank", "cr", "nul", "header_space", "plus_qual_lead", "qual_len", "fasta_head_in_fastq",
           "truncated", "nul_dup_names"]


# ---------------------------------------------------------------------------------------------
# The generator
# ---------------------------------------------------------------------------------------------
def _seq(rng, n):
    s = bytearray(rng.choice(np.frombuffer(b"ACGT", np.uint8), size=n).tobytes())
    if n > 4 and rng.random() < 0.2:
        s[rng.integers(0, n)] = ord("N")
    return bytes(s)


def clean_lines(rng, kind):
    """A clean input as (lines, roles): roles are (record, 'h' header / 's' sequence / 'p' plus / 'q' quality)."""
    lines, roles = [], []
    width = int(rng.integers(1, 25))
    for r in range(int(rng.integers(1, 7))):
        name = b"r%d" % r + (b"_x" * int(rng.integers(0, 3)))
        comment = [b"", b" c%d" % r, b" a b\tc"][int(rng.integers(0, 3))]
        s = _seq(rng, int(rng.integers(1, 60)))
        if kind == "fastq":
            q = bytes(rng.integers(35, 74, size=len(s)).astype(np.uint8))
            for line, role in ((b"@" + name + comment, "h"), (s, "s"), (b"+" if r % 2 else b"+" + name, "p"), (q, "q")):
                lines.append(line)
                roles.append((r, role))
        else:
            lines.append(b">" + name + comment)
            roles.append((r, "h"))
            chunks = [s] if kind == "fasta2" else [s[i:i + width] for i in range(0, len(s), width)]
            for c in chunks:
                lines.append(c)
                roles.append((r, "s"))
    return lines, roles


def _pick(rng, roles, want):
    idx = [i for i, (_, r) in enumerate(roles) if r in want]
    return int(rng.choice(idx)) if idx else None


def mutate(rng, lines, roles, cls):
    """Applies one mutation of class `cls` in place; returns False when it does not apply to this input."""
    ins = lambda b, i, x: b[:i] + x + b[i:]
    if cls == "seq_lead":
        i = _pick(rng, roles, "s")
        if i is None:
            return False
        lead = bytes([b"@>+"[int(rng.integers(0, 3))]])
        lines[i] = lead + (lines[i][1:] if rng.random() < 0.5 else lines[i])
    elif cls == "empty_fasta":
        i = _pick(rng, roles, "h")
        for k in range(int(rng.integers(1, 4))):
            lines.insert(i, b">e%d" % k)
            roles.insert(i, (-1, "h"))
    elif cls == "blank":
        i = int(rng.integers(0, len(lines) + 1))
        lines.insert(i, b"")
        roles.insert(i, (-1, "b"))
    elif cls == "cr":
        i = int(rng.integers(0, len(lines)))
        lines[i] = lines[i] + b"\r" if rng.random() < 0.6 else ins(lines[i], int(rng.integers(0, len(lines[i]) + 1)), b"\r")
    elif cls == "nul":
        i = _pick(rng, roles, "hsq")
        if i is None:
            return False
        lines[i] = ins(lines[i], int(rng.integers(1 if roles[i][1] == "h" else 0, len(lines[i]) + 1)), b"\0")
    elif cls == "header_space":
        i = _pick(rng, roles, "h")
        h = lines[i]
        how = int(rng.integers(0, 4))
        if how == 0 and b" " in h:
            sp = bytes([b"\t\v\f\r"[int(rng.integers(0, 4))]])
            lines[i] = h.replace(b" ", sp, 1)
        elif how == 1:
            lines[i] = h + b" " * int(rng.integers(1, 3))
        elif how == 2:
            lines[i] = h[:1] + b" " + h[1:]                      # "@ name": the name is empty
        else:
            lines[i] = h[:1]                                     # "@" alone
    elif cls == "plus_qual_lead":
        i = _pick(rng, roles, "pq")
        if i is None:
            return False
        if roles[i][1] == "p":
            lines[i] = b"+name again"
        else:
            lines[i] = bytes([b"@+"[int(rng.integers(0, 2))]]) + lines[i][1:]
    elif cls == "qual_len":
        i = _pick(rng, roles, "q")
        if i is None:
            return False
        lines[i] = lines[i] + b"I" if rng.random() < 0.5 or len(lines[i]) < 2 else lines[i][:-1]
    elif cls == "fasta_head_in_fastq":
        i = _pick(rng, roles, "h")
        if lines[i][:1] != b"@":
            return False
        lines[i] = b">" + lines[i][1:]
    elif cls == "nul_dup_names":
        hs = [i for i, (_, r) in enumerate(roles) if r == "h"]
        if len(hs) < 2:
            return False
        a, b = (int(x) for x in rng.choice(hs, size=2, replace=False))
        lines[a] = lines[a][:1] + b"dup\0a"
        lines[b] = lines[b][:1] + b"dup\0b" + (b" tail" if rng.random() < 0.5 else b"")
    else:
        raise ValueError(cls)
    return True


def make_case(seed):
    """(text, kind, classes): a clean input (about one case in six) or one with one to three mutations."""
    rng = np.random.default_rng(seed)
    kind = ["fastq", "fasta2", "fastaw"][int(rng.integers(0, 3))]
    lines, roles = clean_lines(rng, kind)
    classes = []
    if rng.random() >= 1 / 6:
        for _ in range(int(rng.integers(1, 4))):
            cls = CLASSES[int(rng.integers(0, len(CLASSES)))]
            if cls != "truncated" and mutate(rng, lines, roles, cls):
                classes.append(cls)
            elif cls == "truncated":
                classes.append(cls)
    text = b"".join(l + b"\n" for l in lines)
    if "truncated" in classes:
        last = len(b"".join(l + b"\n" for l in lines[:[i for i, (_, r) in enumerate(roles) if r == "h"][-1]]))
        text = text[:int(rng.integers(last + 1, len(text)))]
        if rng.random() < 0.5:
            text += b"\n"
    elif rng.random() < 0.3:
        text = text[:-1]                                         # no final newline
    return text, kind, sorted(set(classes))


N_CASES = 2400
CASES = [make_case(1000 + i) for i in range(N_CASES)]


def fnv(b):
    h = 0xCBF29CE484222325
    for c in b:
        h = ((h ^ c) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


# ---------------------------------------------------------------------------------------------
# CPU: the model against the host reader and against the recorded reference
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dumper(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("fz") / "fastx_offsets_dump")
    r = subprocess.run(["g++", "-std=c++17", "-O2", os.path.join(ROOT, "tests", "fastx_offsets_dump.cpp"),
                        os.path.join(HOST, "fastx.cpp"), "-lz", "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def test_model_reads_the_clean_inputs_as_written():
    for text, kind, classes in CASES:
        if classes:
            continue
        recs = km.kseq_all(text)
        assert recs[-1] == -1 and all(r.plain or kind == "fastaw" for r in recs[:-1])
        for r in recs[:-1]:
            assert text[r.name_off:r.name_off + len(r.name)] == r.name
            assert r.is_fastq == (kind == "fastq")
            if kind != "fastaw":
                assert text[r.seq_off:r.seq_off + len(r.seq)] == r.seq


def test_model_kseq_edges():
    """Hand-worked kseq behaviour (kseq.h:182-224) the generator reaches only by chance."""
    f = lambda t: [(r.name, r.comment, r.seq, r.qual, r.ret) if r != -1 else -1 for r in km.kseq_all(t)]
    assert f(b"junk>a x\nAC\n\nGT\n@b\nA\n+\nI\n") == [(b"a", b"x", b"ACGT", b"", 4), (b"b", b"", b"A", b"I", 1), -1]
    assert f(b"@r1\n@CGT\n+\nIIII\n") == [(b"r1", b"", b"", b"", 0), (b"CGT", b"", b"", b"IIII", -2)]
    assert f(b"@a\nAC\r\n+\nII\r\n") == [(b"a", b"", b"AC", b"II", 2), -1]
    assert f(b"@a \r\nA\r\n+\nI\r\n") == [(b"a", b"\r", b"A", b"I", 1), -1]
    assert f(b"@a\n\r\n+\n\r\n") == [(b"a", b"", b"\r", b"\r", 1), -1]              # one byte: the '\r' stays (kseq.h:146)
    assert f(b">a\nACGT\n\r") == [(b"a", b"", b"ACGT\r", b"", 5), -1]                  # the line's only byte, at EOF
    assert f(b">a\nACGT\n\r\n") == [(b"a", b"", b"ACGT", b"", 4), -1]
    assert f(b"@a\nACGT\n+\nII\nII\nxx>b\nA\n") == [(b"a", b"", b"ACGT", b"IIII", 4), (b"b", b"", b"A", b"", 1), -1]
    assert f(b"@a\nACGT\n+") == [(b"a", b"", b"ACGT", b"", -2)]
    assert f(b"@a\nACGT\n+\nII") == [(b"a", b"", b"ACGT", b"II", -2)]
    assert f(b"@a\tb c\nA\n+\n@\n") == [(b"a", b"b c", b"A", b"@", 1), -1]
    assert f(b">") == [-1] and f(b"") == [-1] and f(b">a") == [(b"a", b"", b"", b"", 0), -1]
    r = km.reads_loop(b">a\n>b\n>c\n" + b"A" * 300 + b"\n>d\n" + b"C" * 400 + b"\n", True)
    assert not r.error and r.log_line == "4 reads (700 bp)"
    assert km.reads_loop(b"@r\0x\nACGT\n+\nIIII\n@r\0y\nACGT\n+\nIIII\n", False).error == ["Error: duplicate read name: r"]
    assert km.pass2_output(b"@r1\0x\nACGTAC\0T\n+\nIIIIIIII\n") == b"@r1\nACGTAC\n+\nIIIIIIII\n"
    assert km.pass2_output(b"@r1 \0c\nA\n+\nI\n") == b"@r1 \nA\n+\nI\n"


def test_model_equals_the_host_reader(dumper, tmp_path):
    """FastxReader (csrc/host/fastx.cpp) and the model read every fuzz input the same way: records, names (as C
    strings), every byte of comment, sequence and quality, the return that ends the file, and where the reader calls a
    record a slice of the input, the same slice."""
    paths = []
    for i, (text, _, _) in enumerate(CASES):
        p = tmp_path / ("c%d" % i)
        p.write_bytes(text)
        paths.append(str(p))
    out = []
    for k in range(0, len(paths), 400):
        r = subprocess.run([dumper] + paths[k:k + 400], capture_output=True)
        assert r.returncode == 0
        out += r.stdout.split(b"\n")[:-1]
    it = iter(out)
    for i, (text, kind, classes) in enumerate(CASES):
        recs = km.kseq_all(text)
        end = recs[-1] if recs[-1] == -1 else recs[-1].ret
        good = [r for r in recs if r != -1 and r.ret >= 0]
        for r in good:
            f = next(it).split(b"\t")
            ctx = (i, classes, text[:120], r)
            assert f[0] == r.cname, ctx
            assert [int(x) for x in f[1:4]] == [len(r.comment), len(r.seq), len(r.qual)], ctx
            assert [int(x, 16) for x in f[10:13]] == [fnv(r.comment), fnv(r.seq), fnv(r.qual)], ctx
            simple = r.plain and b"\0" not in r.name + r.comment + r.seq + r.qual
            assert f[4] == (b"1" if simple else b"0"), ctx
            if simple:
                assert int(f[9]) == r.name_off and int(f[6]) == r.seq_off, ctx
                if r.is_fastq:
                    assert int(f[7]) == r.qual_off, ctx
        assert next(it) == b"END %d" % end, (i, classes, text[:120])


# A fixed subset, run through the recorded reference CLI: the model must predict its verdict
REF_SUBSET = list(range(0, N_CASES, 60))


def _progress(err, what):
    """the last progress line of a reference run: "N reads (M bp)" / "<file> (M bp)", thousands separators removed"""
    hits = [l.strip() for line in err.splitlines() for l in line.split("\r") if what in l]
    return hits[-1].replace(",", "") if hits else None


@pytest.mark.parametrize("i", REF_SUBSET)
def test_model_predicts_the_reference_cli(i, tmp_path):
    text, kind, classes = CASES[i]
    path = tmp_path / "in.txt"
    path.write_bytes(text)
    rc, out, err = orc.run_refcli(["--min_length", "1", str(path)])
    m = km.reads_loop(text, False)
    lines = [l for l in err.splitlines() if l.strip()]
    if m.error:
        assert rc == 1 and lines[-len(m.error):] == m.error, (classes, err[-500:])
    else:
        assert rc == 0, err[-500:]
        assert _progress(err, "reads (") == m.log_line
        assert out == km.pass2_output(text, keep=lambda k: len(m.records[k].seq) >= 1)
    # the same bytes as a short-read file (kmers.cpp:88-134): hashing stops quietly at the first bad record
    reads = tmp_path / "reads.fastq"
    reads.write_bytes(b"@x\n" + b"ACGT" * 10 + b"\n+\n" + b"I" * 40 + b"\n")
    rc, out, err = orc.run_refcli(["-1", str(path), "--min_length", "1", str(reads)])
    n, bases, _ = km.reference_loop(text)
    assert rc == 0, err[-500:]
    counted = [l for l in err.splitlines() if "16-mers" in l and "Hashing" not in l]
    assert [int(l.split()[0].replace(",", "")) for l in counted] == [n]
    assert _progress(err, str(path)) == "%s (%d bp)" % (path, bases)


# ---------------------------------------------------------------------------------------------
# GPU: the device parser against the model
# ---------------------------------------------------------------------------------------------
def chunkings(text, fastq):
    """The whole text as one chunk, and the text cut the way plan_chunks() cuts it (about three chunks)."""
    out = [[0, len(text)]]
    cuts = km.plan_cuts(text, fastq, max(len(text) // 3, 1))
    if cuts and len(cuts) > 2:
        out.append(cuts)
    return out


def check_reads_chunks(ctx, text, fastq, cuts, model):
    """fl_reads_push_text over the chunks; every accepted record must be the model's. Returns the statuses."""
    recs = [r for r in model if r != -1]
    k, statuses = 0, []
    names, hashes = [], []
    for c in range(len(cuts) - 1):
        b, e = cuts[c], cuts[c + 1]
        is_last = c + 2 == len(cuts)
        r = ctx.push_text(text[b:e], fastq=fastq, is_last=is_last)
        statuses.append(r["status"])
        if r["status"] != "ok":
            break
        consumed = b + r["consumed"]
        for j in range(r["n"]):
            assert k < len(recs), "a record the reference does not read"
            m = recs[k]
            assert m.ret >= 0 and m.plain, ("accepted a record kseq reads otherwise", m)
            assert int(r["name_off"][j]) + b == m.name_off and int(r["name_len"][j]) == len(m.name), m
            assert int(r["comment_len"][j]) == len(m.comment), m
            assert int(r["len"][j]) == len(m.seq) and int(r["seq_off"][j]) + b == m.seq_off, m
            if fastq:
                assert int(r["qual_off"][j]) + b == m.qual_off, m
            names.append(m.cname)
            hashes.append(int(r["name_hash"][j]))
            k += 1
        assert k == 0 or recs[k - 1].end <= consumed
        assert k == len(recs) or recs[k].start >= consumed, ("the chunk ends inside a record", recs[k])
        if consumed != e:
            break
    for x in range(len(names)):              # equal hashes <=> equal names (as the reference compares them)
        for y in range(x):
            assert (hashes[x] == hashes[y]) == (names[x] == names[y])
    ctx.reset_reads()
    return statuses


def check_kmer_chunks(ctx, text, fastq, cuts, model, packed):
    """fl_kmers_add_text over the chunks: counts and bases must be kseq's for the records consumed; the records'
    sequences go to `packed` (the batch path), whose set must end up equal."""
    recs = [r for r in model if r != -1]
    k, statuses = 0, []
    for c in range(len(cuts) - 1):
        b, e = cuts[c], cuts[c + 1]
        r = ctx.kmers_add_text(text[b:e], fastq=fastq, is_last=c + 2 == len(cuts))
        statuses.append(r["status"])
        if r["status"] != "ok":
            break
        consumed = b + r["consumed"]
        mine = []
        while k < len(recs) and recs[k].start < consumed:
            mine.append(recs[k])
            k += 1
        assert all(m.ret >= 0 for m in mine), "accepted a chunk where kseq stops with -2"
        assert r["n"] == len(mine), (r, [m.name for m in mine])
        assert r["bases"] == sum(len(m.seq) for m in mine if len(m.seq) >= 16)
        assert not mine or mine[-1].end <= consumed
        seqs = [m.seq for m in mine if len(m.seq) >= 16]
        if seqs:
            packed.kmers_add(seqs, False)
        if consumed != e:
            break
    return statuses


@pytest.mark.gpu
def test_device_parser_accepts_only_what_kseq_reads():
    from filtlong_b200 import api
    rng = np.random.default_rng(5)
    genome = _seq(rng, 5000)
    phred = api.Context(api.make_params(min_length=1))
    kmer = api.Context(api.make_params(min_length=1))
    kmer.kmers_add([genome], False)
    kmer.kmers_count()
    text_k, packed = api.Context(api.make_params()), api.Context(api.make_params())
    os.environ["FL_FASTA_TWO_LINE"] = "1"
    try:
        text_k2 = api.Context(api.make_params())
    finally:
        del os.environ["FL_FASTA_TWO_LINE"]
    tally = collections.defaultdict(collections.Counter)
    for i, (text, kind, classes) in enumerate(CASES):
        model = km.kseq_all(text)
        fmt = {64: "fastq", 62: "fasta"}.get(text[0] if text else 0)
        if fmt is None:
            continue
        fastq = fmt == "fastq"
        for cuts in chunkings(text, fastq):
            runs = [("reads/kmer", check_reads_chunks(kmer, text, fastq, cuts, model))]
            if fastq:
                runs.append(("reads/phred", check_reads_chunks(phred, text, fastq, cuts, model)))
            runs.append(("ref/" + ("fastq" if fastq else "wrapped"), check_kmer_chunks(text_k, text, fastq, cuts, model, packed)))
            if not fastq:
                runs.append(("ref/fasta2", check_kmer_chunks(text_k2, text, fastq, cuts, model, packed)))
            for what, st in runs:
                ok = all(s == "ok" for s in st)
                for cls in classes or ["clean"]:
                    tally[cls]["ok" if ok else "fallback"] += 1
                if not classes and (what != "reads/kmer" or kind != "fastaw") and not (kind == "fastaw" and what == "ref/fasta2"):
                    assert ok, (i, kind, what, st, text[:200])      # a fix may not fall back on the common layout
    assert np.array_equal(packed.kmers_export(), np.union1d(text_k.kmers_export(), text_k2.kmers_export()))
    print("\nper mutation class: calls that the device accepted / handed back")
    for cls in ["clean"] + CLASSES:
        print("  %-20s ok %5d   fallback %5d" % (cls, tally[cls]["ok"], tally[cls]["fallback"]))
    for cls in ["clean"] + CLASSES:
        assert tally[cls]["fallback"] + tally[cls]["ok"] > 0, cls
    assert tally["clean"]["ok"] > 0 and tally["seq_lead"]["fallback"] > 0 and tally["nul"]["fallback"] > 0
    for c in (phred, kmer, text_k, text_k2, packed):
        c.close()


# ---------------------------------------------------------------------------------------------
# GPU: the CLI on every input path against the recorded reference
# ---------------------------------------------------------------------------------------------
def _reads(n, seed, lead=b"@"):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        s = _seq(rng, 120 + 7 * i)
        out.append(b"@r%d\n" % i + s + b"\n+\n" + bytes(rng.integers(40, 74, size=len(s)).astype(np.uint8)) + b"\n")
    return out


def cli_cases():
    """(name, reads bytes, as a -1 file too): the issue's table, the NUL cases and fuzz outputs the model picks."""
    r = _reads(10, 3)
    cases = [
        ("seq_at", r[0] + b"@r1\n@CGT\n+\nIIII\n" + r[2]),
        ("seq_plus", r[0] + b"@r1\n+CGT\n+\nIIII\n" + r[2]),
        ("seq_gt", r[0] + b"@r1\n>CGT\n+\nIIII\n" + r[2]),
        ("fasta_empty", b">a\n>b\n>c\n" + _seq(np.random.default_rng(1), 300) + b"\n>d\n" + _seq(np.random.default_rng(2), 400) + b"\n"),
        ("fourth_plus", b"".join(r[:3]) + b"@r3\n+CGTACGTACGTACGTACGT\n+\n" + b"I" * 19 + b"\n" + b"".join(r[4:])),
        ("nul", b"".join(r[:4]) + b"@r1x\0x\nACGTAC\0T\n+\nIIIIIIII\n" + b"".join(r[4:])),
        ("nul_comment", b"".join(r[:4]) + b"@n1 \0c\nACGTACGT\n+\nIII\0IIII\n" + b"".join(r[4:])),
        ("nul_dup", b"".join(r[:4]) + b"@dup\0a\nACGT\n+\nIIII\n@dup\0b\nACGT\n+\nIIII\n" + b"".join(r[4:])),
    ]
    # fuzz outputs: in every class, the first with one mutation that the model reads without error (FASTQ first, then
    # FASTA, which needs -a)
    seen = set()
    for i, (text, kind, classes) in sorted(enumerate(CASES), key=lambda c: (c[1][1] != "fastq", c[0])):
        if len(classes) != 1 or classes[0] in seen or km.reads_loop(text, True).error or not km.reads_loop(text, True).records:
            continue
        if not any(len(x.seq) >= 1 for x in km.reads_loop(text, True).records):
            continue
        seen.add(classes[0])
        cases.append(("fuzz%d_%s" % (i, classes[0]), text))
    return cases


CLI_CASES = cli_cases()


def _run(cmd, env=None):
    e = dict(os.environ, LC_ALL="C")
    e.pop("LANG", None)
    e.update(env or {})
    p = subprocess.run(cmd, capture_output=True, env=e)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


def _errors(err):
    return [l for l in err.splitlines() if l.startswith("Error") or l.startswith("  problem")]


def test_cli_cases_cover_the_table_and_each_class():
    names = [n for n, _ in CLI_CASES]
    assert len(names) >= 8 + 8, names


@pytest.mark.gpu
@pytest.mark.parametrize("case", [n for n, _ in CLI_CASES])
def test_cli_matches_the_reference_on_every_input_path(case, tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    text = dict(CLI_CASES)[case]
    fa = tmp_path / "asm.fasta"
    fa.write_bytes(b">asm\n" + _seq(np.random.default_rng(7), 3000) + b"\n")
    src = tmp_path / ("reads.fastq" if text[:1] == b"@" else "reads.fasta")
    src.write_bytes(text)
    good = tmp_path / "good.fastq"
    good.write_bytes(b"".join(_reads(6, 8)))
    runs = [["--min_length", "1", str(src)], ["-a", str(fa), "--min_length", "1", "-p", "90", str(src)],
            ["-1", str(src), "--min_length", "1", str(good)], ["-a", str(src), "--min_length", "1", str(good)]]
    for args in runs:
        rc_r, out_r, err_r = orc.run_refcli(args)
        for env, extra in (({"FL_CHUNK_MB": "1", "FL_CLI_TIMING": "1"}, []), ({"FL_HOST_PARSER": "1"}, []), ({"FL_CHUNK_MB": "1"}, ["--bgzip"])):
            rc, out, err = _run([CLI] + extra + args, env)
            if extra and rc == 0:
                out = gzip.decompress(out) if out else b""
            ctx = (case, args, env, err[-800:])
            assert rc == rc_r, ctx
            assert out == out_r, ctx
            assert _errors(err) == _errors(err_r), ctx
            if args[0] in ("-1", "-a") and args[1] == str(src):
                count = lambda e: [l.replace(",", "") for l in e.splitlines() if "16-mers" in l and "Hashing" not in l]
                assert count(err) == count(err_r), ctx

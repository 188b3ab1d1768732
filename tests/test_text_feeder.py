"""The feeder (SURVEY 8f-1..3): FASTQ / FASTA text parsed on the device (fl_reads_push_text) and the CLI's
input path built on it (mapped file -> pinned ring -> device; writev output from the mapping; duplicate
names through device-computed hashes). Results must equal the packed-arena path bit for bit, the record index
must equal a plain Python parse, anything outside the simple layout must be handed back (FALLBACK) untouched,
and the CLI's stdout must stay byte-identical to the reference binary's."""
import os
import subprocess

import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import util

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def fastq_text(reads, last_newline=True):
    t = b"".join(b"@" + n + b"\n" + s + b"\n+" + (n if i % 3 == 0 else b"") + b"\n" + q + b"\n" for i, (n, s, q) in enumerate(reads))
    return t if last_newline else t[:-1]


def make_reads(seed, n=120, genome=None):
    rng = np.random.default_rng(seed)
    genome = genome or util.rand_seq(rng, 50000)
    reads = [(("read_%d" % i).encode() + (b" comment %d\twith tab" % i if i % 4 == 1 else b""), s, q)
             for i, (_, s, q) in enumerate(util.long_reads(rng, genome, n, max_len=7000))]
    reads.append((b"x", b"ACGT", b"IIII"))
    reads.append((b"a_rather_long_name_" * 5, util.rand_seq(rng, 33), b"5" * 33))
    return genome, reads


@pytest.mark.parametrize("mode", ["phred", "kmer"])
@pytest.mark.parametrize("last_newline", [True, False])
def test_push_text_equals_packed_path_and_python_parse(mode, last_newline):
    genome, reads = make_reads(3)
    opts = dict(keep_percent=70.0) if mode == "phred" else dict(keep_percent=70.0, trim=True, split=120)
    text = fastq_text(reads, last_newline)
    ctx = api.Context(api.make_params(**opts))
    ref = api.Context(api.make_params(**opts))
    if mode == "kmer":
        for c in (ctx, ref):
            c.kmers_add([genome], False)
            c.kmers_count()
    # the text in three record-aligned chunks (the caller's job: fl_reads_push_text reports where whole records end)
    cuts, pos = [], 0
    idx = {k: [] for k in ("name_off", "name_len", "comment_len", "seq_off", "qual_off", "len", "name_hash")}
    while pos < len(text):
        piece = text[pos:pos + len(text) // 3 + 1000]
        is_last = pos + len(piece) >= len(text)
        if not is_last:                        # cut at a record boundary: last "\n@" followed by a well formed record
            k = piece.rfind(b"\n@")
            while True:
                rest = piece[k + 1:].split(b"\n")
                if len(rest) >= 4 and rest[2].startswith(b"+") and len(rest[1]) == len(rest[3]):
                    break
                k = piece.rfind(b"\n@", 0, k)
            piece = piece[:k + 1]
        r = ctx.push_text(piece, fastq=True, is_last=is_last)
        assert r["status"] == "ok" and r["consumed"] == len(piece)
        for k in idx:
            idx[k].append(r[k] + (pos if k.endswith("_off") else 0) if k.endswith("_off") else r[k])
        cuts.append(r["n"])
        pos += len(piece)
    idx = {k: np.concatenate(v) for k, v in idx.items()}
    assert sum(cuts) == len(reads) and len(cuts) >= 3
    for i, (n, s, q) in enumerate(reads):
        name, _, comment = n.partition(b" ")
        o = int(idx["name_off"][i])
        assert text[o:o + int(idx["name_len"][i])] == name
        assert int(idx["comment_len"][i]) == len(comment)
        if comment:
            assert text[o + len(name) + 1:o + len(name) + 1 + len(comment)] == comment
        assert int(idx["len"][i]) == len(s)
        assert text[int(idx["seq_off"][i]):int(idx["seq_off"][i]) + len(s)] == s
        assert text[int(idx["qual_off"][i]):int(idx["qual_off"][i]) + len(q)] == q
    # equal names <=> equal hashes (here: all distinct)
    assert len(set(idx["name_hash"].tolist())) == len(reads)
    ref.push(api.HostBatch([r[1] for r in reads], [r[2] for r in reads], want_seq=(mode == "kmer")))
    s1, s2 = ctx.finalize(-1), ref.finalize(-1)
    assert (s1.status, s1.target, s1.keeping, s1.total_bases) == (s2.status, s2.target, s2.keeping, s2.total_bases)
    a, b = ctx.row_results(), ref.row_results()
    for k in a:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    ra, rb = ctx.read_results(), ref.read_results()
    for k in ra:
        assert np.array_equal(ra[k].view(np.uint8), rb[k].view(np.uint8)), k
    ctx.close(); ref.close()


def test_push_text_fasta_and_fallbacks():
    genome, reads = make_reads(5, n=30)
    ctx = api.Context(api.make_params(keep_percent=80.0))
    fasta = b"".join(b">" + n + b"\n" + s + b"\n" for n, s, _ in reads)
    assert ctx.push_text(fasta, fastq=False)["status"] == "fallback"          # no reference: main.cpp:103-106 is the host's error
    ctx.kmers_add([genome], False)
    ctx.kmers_count()
    r = ctx.push_text(fasta, fastq=False)
    assert r["status"] == "ok" and r["n"] == len(reads) and [int(x) for x in r["len"]] == [len(s) for _, s, _ in reads]
    ctx.reset_reads()
    good = fastq_text(reads)
    crlf = good.replace(b"\n", b"\r\n")
    two_line_seq = b"@a\nACGT\nACGT\n+\nIIIIIIII\n"
    short_qual = b"@a\nACGTACGT\n+\nIIII\n@b\nACGT\n+\nIIII\n"
    blank = b"@a\nACGT\n+\nIIII\n\n@b\nACGT\n+\nIIII\n"
    no_name = b"@\nACGT\n+\nIIII\n"
    empty_seq = b"@a\n\n+\n\n"
    wrong_lead = b">a\nACGT\n+\nIIII\n"
    for bad in (crlf, two_line_seq, short_qual, blank, no_name, empty_seq, wrong_lead):
        r = ctx.push_text(bad, fastq=True)
        assert r["status"] == "fallback", bad[:40]
        assert ctx.counts()[0] == 0                      # nothing was scored
    # too small a record array: the needed size comes back, nothing scored
    r = ctx.push_text(good, fastq=True, cap=5)
    assert r["status"] == "erange" and r["n"] == len(reads) and ctx.counts()[0] == 0
    # a truncated final record in a chunk that is not the last: whole records are consumed, the rest is the caller's
    r = ctx.push_text(good + b"@tail\nACG", fastq=True, is_last=False)
    assert r["status"] == "ok" and r["n"] == len(reads) and r["consumed"] == len(good)
    ctx.close()


@pytest.mark.parametrize("multi", [False, True])
def test_kmers_add_text_builds_the_set_the_packed_path_builds(multi):
    """fl_kmers_add_text (the reference file as text: kmers.cpp:75-134 behind kseq) against fl_kmers_add_batch on the
    same sequences: identical 16-mer sets, one copy and >= 4 copies, with N runs, lower case, sequences shorter than
    16 (counted, adding nothing), chunked at record boundaries; and against the oracle's set."""
    rng = np.random.default_rng(41 + multi)
    genome = bytearray(util.rand_seq(rng, 30000))
    genome[5000:5040] = b"N" * 40
    genome[12000:12100] = bytes(genome[12000:12100]).lower()
    genome = bytes(genome)
    if multi:       # short reads, deep enough that many 16-mers are seen four times
        seqs = [genome[s:s + 150] for s in rng.integers(0, len(genome) - 150, size=3000)]
        seqs[7] = b"ACGTNACGT"                                        # < 16: counted, contributes nothing
        seqs[11] = b"acgtacgtacgtacgtacgtnnnnacgtacgtacgtacgtacgtacgtac"
        recs = [(b"r%d" % i, q, b"I" * len(q)) for i, q in enumerate(seqs)]
        text = fastq_text(recs)
    else:           # "contigs", unwrapped FASTA
        seqs = [genome[:9000], genome[9000:9010], genome[9010:30000], b"ACGTACGTACGTACGT", b"TTTTTTTTTTTTTTT"]
        text = b"".join(b">contig_%d some words\n" % i + q + b"\n" for i, q in enumerate(seqs))
    # the packed path's set first, its multiple-copy build state (49 GiB) released before the text path needs its own
    b = api.Context(api.make_params())
    b.kmers_add(seqs, multi)
    b_count, b_set = b.kmers_count(), b.kmers_export()
    b.kmers_release_build_state()
    a = api.Context(api.make_params())
    # three record-aligned chunks
    lines = text.split(b"\n")[:-1]
    lpr = 4 if multi else 2
    n_rec = len(lines) // lpr
    cuts = [0, n_rec // 3, 2 * n_rec // 3, n_rec]
    total_rec = total_bases = 0
    for i in range(3):
        piece = b"".join(l + b"\n" for l in lines[cuts[i] * lpr:cuts[i + 1] * lpr])
        if not piece:
            continue
        r = a.kmers_add_text(piece, fastq=multi, is_last=(i == 2), multiple_copies=multi)
        assert r["status"] == "ok" and r["consumed"] == len(piece), r
        total_rec += r["n"]
        total_bases += r["bases"]
    assert total_rec == len(seqs)
    assert total_bases == sum(len(q) for q in seqs if len(q) >= 16)
    assert a.kmers_count() == b_count > 0
    assert np.array_equal(a.kmers_export(), b_set)
    ok = orc.Kmers()
    (ok.add_short_reads if multi else ok.add_assembly)(seqs)
    assert np.array_equal(a.kmers_export(), np.sort(ok.dump()))
    # not the common layout: nothing is added, the caller parses on the host
    before = a.kmers_count()
    ragged = b">c\nACGTACGTACGTACGTACGT\nACGTACGT\nACGTACGTACGTACGTACGT\n"         # a middle line shorter than the first
    longer = b">c\nACGTACGTACGTACGTACGT\nACGTACGTACGTACGTACGTACGT\n"                 # the last line longer than the first
    crlf = b">c\r\nACGTACGTACGTACGTACGTACGT\r\n"
    blank = b">c\nACGTACGTACGTACGTACGT\n\nACGTACGTACGTACGTACGT\n"
    plus = b">c\nACGTACGTACGTACGTACGT\n+CGTACGTACGTACGTACGT\n"                        # kseq takes '+' for the quality separator
    nohead = b"ACGTACGTACGTACGTACGT\n>c\nACGTACGTACGTACGTACGT\n"
    for bad in (ragged, longer, crlf, blank, plus, nohead, b"@r\nACGTACGTACGTACGTAAAA\n+\nIIII\n"):
        r = a.kmers_add_text(bad, fastq=bad.startswith(b"@"), is_last=True, multiple_copies=multi)
        assert r["status"] == "fallback" and r["n"] == 0, bad
    assert a.kmers_count() == before
    a.close(); b.close()


@pytest.mark.parametrize("width", [1, 7, 31, 32, 60, 64, 70, 1000])
def test_kmers_add_text_wrapped_fasta(width):
    """A wrapped FASTA reference (every assembler writes them so) through fl_kmers_add_text: kseq joins a record's
    lines (kseq.h:199-203); the device maps base p to byte first + p + p / width. Against the packed path on the joined
    sequences, for line widths below, at and above the 32-base groups of the packer, with N runs and lower case, records
    of one line, of exactly k full lines, empty records, and a last line without newline."""
    rng = np.random.default_rng(100 + width)
    genome = bytearray(util.rand_seq(rng, 9000))
    genome[1000:1100] = b"N" * 100
    genome[2000:2300] = bytes(genome[2000:2300]).lower()
    genome[4000:4003] = b"RYK"
    genome = bytes(genome)
    seqs = [genome[:3001], genome[3001:3001 + 5 * width], genome[5000:5000 + max(width // 2, 1)], b"", genome[6000:6017], genome[7000:]]
    wrap = lambda q: b"".join(q[i:i + width] + b"\n" for i in range(0, len(q), width))
    text = b"".join(b">contig_%d len=%d\n" % (i, len(q)) + wrap(q) for i, q in enumerate(seqs))
    for last_newline in (True, False):
        a, b = api.Context(api.make_params()), api.Context(api.make_params())
        b.kmers_add([q for q in seqs if q], False)
        t = text if last_newline else text[:-1]
        # two chunks, cut at a record start
        cut = t.index(b">contig_2")
        r1 = a.kmers_add_text(t[:cut], fastq=False, is_last=False)
        r2 = a.kmers_add_text(t[cut:], fastq=False, is_last=True)
        assert r1["status"] == r2["status"] == "ok" and r1["consumed"] == cut and r2["consumed"] == len(t) - cut
        assert r1["n"] + r2["n"] == len(seqs)
        assert r1["bases"] + r2["bases"] == sum(len(q) for q in seqs if len(q) >= 16)
        assert a.kmers_count() == b.kmers_count() > 0
        assert np.array_equal(a.kmers_export(), b.kmers_export())
        a.close(); b.close()


def run(cmd, env=None):
    e = dict(os.environ, LC_ALL="C")
    e.pop("LANG", None)
    e.update(env or {})
    p = subprocess.run(cmd, capture_output=True, env=e)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


CLI_CASES = [
    ["--min_length", "1", "--keep_percent", "90", "FQ"],
    ["-t", "300000", "FQ"],
    ["-p", "60", "--min_mean_q", "70", "--window_size", "100", "FQ"],
    ["-t", "1g", "FQ"],
    ["-a", "FA", "-p", "90", "FQ"],
    ["-a", "FA", "-p", "80", "--trim", "--split", "100", "FQ"],
    ["-a", "FA", "--split", "30", "-t", "250000", "FQ"],
    ["-a", "FA", "-p", "70", "--trim", "--split", "80", "FASTA"],
]


@pytest.mark.parametrize("case", CLI_CASES, ids=lambda c: " ".join(c))
@pytest.mark.parametrize("last_newline", [True, False])
def test_cli_device_parse_path_is_byte_identical_to_the_reference(case, last_newline, tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    genome, reads = make_reads(11, n=200)
    fq = tmp_path / "reads.fastq"
    fq.write_bytes(fastq_text(reads, last_newline))
    fa = util.write_fasta(tmp_path / "asm.fasta", [("contig_1", genome[:30000]), ("contig_2", genome[30000:])], width=60)
    fasta = tmp_path / "reads.fasta"
    fasta.write_bytes(b"".join(b">" + n + b"\n" + s + b"\n" for n, s, _ in reads[:80]))
    sub = {"FQ": str(fq), "FA": fa, "FASTA": str(fasta)}
    args = [sub.get(a, a) for a in case]
    rc_r, out_r, err_r = orc.run_refcli(args)
    # tiny chunks so that the plan has many of them and the ring wraps
    rc_o, out_o, err_o = run([CLI] + args, {"FL_CLI_TIMING": "1", "FL_CHUNK_MB": "1"})
    assert rc_o == rc_r == 0, err_o[-2000:]
    assert "device parse" in err_o, "the host parser ran instead of the feeder"
    assert out_o == out_r
    rc_h, out_h, err_h = run([CLI] + args, {"FL_HOST_PARSER": "1"})
    assert rc_h == 0 and out_h == out_r
    # stdout a regular file: groups of reads are sized and written with pwrite() by several threads
    with open(tmp_path / "out.txt", "wb") as fh:
        fh.write(b"HEAD\n")
        fh.flush()
        e = dict(os.environ, LC_ALL="C", FL_CHUNK_MB="1")
        e.pop("LANG", None)
        assert subprocess.run([CLI] + args, stdout=fh, stderr=subprocess.DEVNULL, env=e).returncode == 0
        fh.write(b"TAIL\n")
    written = (tmp_path / "out.txt").read_bytes()
    assert written[:5] == b"HEAD\n" and written[-5:] == b"TAIL\n" and written[5:-5] == out_r
    tail = lambda e: [l.split("\r")[-1] for l in e.splitlines() if l.strip() and "[timing]" not in l and "bp)" not in l]
    assert tail(err_o) == tail(err_r)


def test_cli_duplicate_names_and_fallback_inputs(tmp_path):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    rng = np.random.default_rng(2)
    recs = [(b"r%d" % i, util.rand_seq(rng, 300), util.rand_qual(rng, 300)) for i in range(400)]
    dup = tmp_path / "dup.fastq"
    dup.write_bytes(fastq_text(recs + [(b"r37", util.rand_seq(rng, 100), b"I" * 100)] + recs[:3]))
    multi = tmp_path / "multi.fastq"                       # a two-line sequence in the middle: the feeder must hand the file back
    multi.write_bytes(fastq_text(recs[:100]) + b"@ml\nACGTACGT\nACGT\n+\nIIIIIIIIIIII\n" + fastq_text(recs[100:200]))
    for path in (dup, multi):
        args = ["-p", "50", str(path)]
        rc_r, out_r, err_r = orc.run_refcli(args)
        rc_o, out_o, err_o = run([CLI] + args, {"FL_CHUNK_MB": "1"})
        assert (rc_o, out_o) == (rc_r, out_r)
        assert [l for l in err_o.splitlines() if l.startswith("Error")] == [l for l in err_r.splitlines() if l.startswith("Error")]


def test_cli_gzip_input_is_inflated_once_and_parsed_on_the_device(tmp_path):
    """.gz reads (the README's usual input): one member, concatenated members, BGZF blocks (inflated by several host
    threads) all take the device-text path after ONE inflate into memory; a truncated file goes to the host reader,
    whose messages are the reference's. stdout is the reference binary's, byte for byte, every time."""
    import gzip
    from tests.test_gzmem import bgzf
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    genome, reads = make_reads(31, n=300)
    text = fastq_text(reads)
    fa = util.write_fasta(tmp_path / "asm.fasta", [("c", genome)])
    half = len(fastq_text(reads[:150]))
    files = {
        "one.fastq.gz": gzip.compress(text, 6),
        "two.fastq.gz": gzip.compress(text[:half], 1) + gzip.compress(text[half:], 9),
        "blocks.fastq.gz": bgzf(text, block=20000),
    }
    for name, data in files.items():
        path = tmp_path / name
        path.write_bytes(data)
        for case in (["-p", "70", str(path)], ["-a", fa, "-p", "80", "--trim", "--split", "100", str(path)]):
            rc_r, out_r, err_r = orc.run_refcli(case)
            rc_o, out_o, err_o = run([CLI] + case, {"FL_CLI_TIMING": "1", "FL_CHUNK_MB": "1", "FL_INFLATE_THREADS": "4"})
            assert rc_o == rc_r == 0, err_o[-2000:]
            assert "gzip input inflated" in err_o and "device parse" in err_o, err_o[-2000:]
            assert out_o == out_r and len(out_r) > 0
            rc_h, out_h, _ = run([CLI] + case, {"FL_GZ_HOST": "1"})            # the streaming host reader, for comparison
            assert rc_h == 0 and out_h == out_r
    broken = tmp_path / "truncated.fastq.gz"
    broken.write_bytes(files["one.fastq.gz"][:len(files["one.fastq.gz"]) // 2])
    rc_r, out_r, err_r = orc.run_refcli(["-p", "70", str(broken)])
    rc_o, out_o, err_o = run([CLI, "-p", "70", str(broken)], {"FL_CLI_TIMING": "1"})
    assert "gzip input inflated" not in err_o
    assert (rc_o, out_o) == (rc_r, out_r)
    assert [l for l in err_o.splitlines() if l.startswith("Error")] == [l for l in err_r.splitlines() if l.startswith("Error")]


REFERENCE_FILE_CASES = ["flat_fasta", "wrapped_fasta", "ragged_record_in_second_chunk", "short_reads_plain_and_gzip"]


@pytest.mark.parametrize("case", REFERENCE_FILE_CASES)
def test_cli_reference_files_take_the_device_text_path(case, tmp_path):
    """-a with an unwrapped or a wrapped FASTA and -1/-2 with plain and gzip FASTQ files go to the device as text
    (Kmers::add_reference -> fl_kmers_add_text); a file with a ragged record half way goes through the host reader from
    that chunk on. Same stdout and the same log lines as the reference binary every time."""
    import gzip
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    genome, reads = make_reads(51, n=200)
    fq = tmp_path / "reads.fastq"
    fq.write_bytes(fastq_text(reads))
    wrap = lambda q, w: b"".join(q[i:i + w] + b"\n" for i in range(0, len(q), w))
    if case == "flat_fasta":
        contigs = [(b"c1 first", genome[:20000]), (b"c2", genome[20000:20010]), (b"c3", genome[20010:])]
        fa = tmp_path / "flat.fasta"
        fa.write_bytes(b"".join(b">" + n + b"\n" + q + b"\n" for n, q in contigs))
        args, how = ["-a", str(fa), "-p", "80", "--trim", "--split", "100", str(fq)], ["device text"]
    elif case == "wrapped_fasta":
        fa = util.write_fasta(tmp_path / "wrapped.fasta", [("c1", genome[:20000]), ("c3", genome[20010:])], width=70)
        args, how = ["-a", fa, "-p", "80", "--trim", str(fq)], ["device text"]
    elif case == "ragged_record_in_second_chunk":
        # 40 wrapped records (1.3 MB: two 1 MB chunks), the 35th with a short line in the middle: the host reader takes
        # over in the second chunk
        recs = [b">rec%d\n" % i + wrap(genome[i * 100:i * 100 + 32000], 60) for i in range(40)]
        recs[34] = b">rec34\n" + genome[:60] + b"\n" + genome[60:90] + b"\n" + genome[90:150] + b"\n"
        fa = tmp_path / "half.fasta"
        fa.write_bytes(b"".join(recs))
        # (no --keep_percent here and below: this assembly covers 70 % of the genome and the short-read set is patchy, so
        # many rows tie at the bottom of the ranking and a cut-off there is the unstable-sort exception of DESIGN 5; without a
        # cut-off every read's trim / split coordinates are compared instead)
        args, how = ["-a", str(fa), "--min_length", "50", "--trim", str(fq)], ["host reader from byte"]
    else:
        rng = np.random.default_rng(9)
        sr = [genome[s:s + 150] for s in rng.integers(0, len(genome) - 150, size=4000)]
        s1 = tmp_path / "s1.fastq"
        s1.write_bytes(fastq_text([(b"p%d/1" % i, q, b"I" * 150) for i, q in enumerate(sr[:2000])]))
        s2 = tmp_path / "s2.fastq.gz"
        s2.write_bytes(gzip.compress(fastq_text([(b"p%d/2" % i, q, b"I" * 150) for i, q in enumerate(sr[2000:])])))
        args, how = ["-1", str(s1), "-2", str(s2), "--min_length", "50", "--trim", "--split", "50", str(fq)], ["device text", "device text"]
    tail = lambda e: [l.split("\r")[-1] for l in e.splitlines() if l.strip() and "[timing]" not in l and "bp)" not in l]
    count = lambda e: [l for l in e.splitlines() if "16-mers" in l and "Hashing" not in l]          # "N contigs / reads, M 16-mers"
    rc_r, out_r, err_r = orc.run_refcli(args)
    rc_o, out_o, err_o = run([CLI] + args, {"FL_CLI_TIMING": "1", "FL_CHUNK_MB": "1"})
    rc_h, out_h, err_h = run([CLI] + args, {"FL_HOST_PARSER": "1"})                                  # the host reader for everything
    assert rc_o == rc_r == rc_h == 0, err_o[-2000:]
    notes = [l for l in err_o.splitlines() if l.startswith("[timing] reference ") and (": device text" in l or ": host reader" in l)]
    assert len(notes) == len(how) and all(h in n for h, n in zip(how, notes)), notes
    assert count(err_h) == count(err_r), (count(err_h), count(err_r))
    assert count(err_o) == count(err_r), (count(err_o), count(err_r))
    assert out_h == out_r and len(out_r) > 0
    assert out_o == out_r
    assert tail(err_o) == tail(err_r)


def test_cli_sharded_over_gpus_prints_what_one_gpu_prints(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    genome, reads = make_reads(21, n=600)
    def again(n):
        name, sep, comment = n.partition(b" ")
        return name + b"_again" + sep + comment
    reads = reads + [(again(n), s, q) for n, s, q in reads[:50]]                # exact score ties across shards
    fq = tmp_path / "reads.fastq"
    fq.write_bytes(fastq_text(reads))
    fa = util.write_fasta(tmp_path / "asm.fasta", [("c", genome)])
    for case in (["-p", "60", str(fq)], ["-a", fa, "-p", "70", "--trim", "--split", "100", str(fq)]):
        rc1, out1, err1 = run([CLI] + case, {"FL_CHUNK_MB": "1"})
        rc2, out2, err2 = run([CLI, "--gpus", "2"] + case, {"FL_CHUNK_MB": "1", "NCCL_DEBUG": "VERSION"})   # NCCL chats on "stdout"
        assert rc1 == rc2 == 0, err2[-2000:]
        assert out1 == out2

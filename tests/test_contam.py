"""`filtlong --contam FILE [--max_contam P]`: remove the reads that come from a contaminant sequence.

A read's contaminant percentage c is the raw mean quality the reference gives it in k-mer mode with `-a FILE`
(100 * bases covered by a 16-mer of FILE / length); the read is removed when c > P. What these tests check: the set is
the one `-a FILE` builds; c is bit-identical to the oracle's k-mer-mode mean against that set; fl_finalize ranks only the
kept reads; and the CLI's stdout equals the reference's run on the input with the removed reads deleted, with `-p P`
turned into `-t T` over all the input's bases (main.cpp:229-237). Those reference runs are recorded in
tests/golden/contam_reference_runs.jsonl.xz; the CPU tests check them against the oracle. The argument errors need no
GPU."""
import gzip
import json
import lzma
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from tests import bam_util as bu
from tests import qtrim_model as qm
from tests import util
from tests.test_cli import CLI, log_lines, need_cli

TIMEOUT = 300
P_DEFAULT = 50.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORDED = os.path.join(ROOT, "tests", "golden", "contam_reference_runs.jsonl.xz")
_recorded_loaded = False


def run(args, stdin_data=None, env_extra=None):
    env = dict(os.environ, LC_ALL="C", **(env_extra or {}))
    env.pop("LANG", None)
    p = subprocess.run([CLI] + list(args), input=stdin_data, capture_output=True, env=env, timeout=TIMEOUT)
    return p.returncode, p.stdout, p.stderr


# ---- argument errors and help (no GPU) --------------------------------------------------------------------------------
ERRORS = [
    (["--max_contam", "20", "-p", "90", "FQ"], "Error: --max_contam needs --contam"),
    (["--contam", "FA", "--max_contam", "100", "FQ"], "Error: the value for --max_contam must be at least 0 and less than 100"),
    (["--contam", "FA", "--max_contam", "250.5", "-p", "90", "FQ"], "Error: the value for --max_contam must be at least 0 and less than 100"),
    (["--contam", "FA", "--max_contam", "-1", "FQ"], "Error: argument 'float' received invalid value type '-1'"),
    (["--contam", "MISSING", "FQ"], "Error: cannot find file: MISSING"),
    (["-a", "FA", "--contam", "MISSING", "-p", "90", "FQ"], "Error: cannot find file: MISSING"),
]


@need_cli
@pytest.mark.parametrize("args,message", ERRORS, ids=lambda x: " ".join(x) if isinstance(x, list) else None)
def test_argument_errors(args, message, tmp_path):
    fq = util.write_fastq(tmp_path / "x.fastq", [("r1", b"ACGT" * 10, b"I" * 40)])
    fa = util.write_fasta(tmp_path / "a.fasta", [("c", b"ACGT" * 10)])
    missing = str(tmp_path / "missing.fa")
    sub = {"FQ": fq, "FA": fa, "MISSING": missing}
    rc, out, err = run([sub.get(a, a) for a in args])
    assert (rc, out, err.decode()) == (1, b"", message.replace("MISSING", missing) + "\n")


@need_cli
def test_no_thresholds_message_is_unchanged(tmp_path):
    fq = util.write_fastq(tmp_path / "x.fastq", [("r1", b"ACGT" * 10, b"I" * 40)])
    rc, out, err = run([fq])
    assert rc == 1 and err.decode() == ("Error: no thresholds set, you must use one of the following options:\n"
                                        "target_bases, keep_percent, min_length, max_length, min_mean_q, min_window_q, trim, split\n")


@need_cli
def test_help_lists_the_contaminant_group():
    rc, out, err = run(["--help"])
    text = err.decode()
    assert rc == 0 and "--contam [file]" in text and "--max_contam [float]" in text
    assert text.index("score weights") < text.index("contaminant removal:") < text.index("--contam [file]") \
        < text.index("--max_contam") < text.index("read manipulation:")


# ---- fixtures ---------------------------------------------------------------------------------------------------------
def wrapped_fasta(name, seq, width=60):
    return b">" + name + b" contaminant\n" + b"".join(seq[i:i + width] + b"\n" for i in range(0, len(seq), width))


def make_inputs(seed=2024):
    """a sample genome, a lambda-sized contaminant (lowercase and N runs), and reads: from the genome, from the
    contaminant, chimeras of the two on both sides of 50 %, reads shorter than 16, and one with c == 50 exactly"""
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, 150000)
    contam = bytearray(util.rand_seq(rng, 48502))
    contam[1000:1600] = bytes(contam[1000:1600]).lower()
    contam[20000:20100] = b"N" * 100
    contam[30000:30040] = b"n" * 40
    contam = bytes(contam)
    reads = [(n, s, q) for n, s, q in util.long_reads(rng, genome, 260, max_len=12000, lower_frac=0.05)]
    cont = contam.upper().replace(b"N", b"A")
    for i, (n, s, q) in enumerate(util.long_reads(rng, cont, 50, max_len=6000, junk_frac=0.0, lower_frac=0.0)):
        reads.append(("contam_%d" % i, s, q))
    for i in range(60):                                     # chimeras: a contaminant share from about 10 % to 90 %
        L = int(rng.integers(800, 6000))
        share = rng.uniform(0.1, 0.9)
        a = int(L * share)
        cs = int(rng.integers(0, len(cont) - a))
        gs = int(rng.integers(0, len(genome) - (L - a)))
        seq = util.mutate(rng, cont[cs:cs + a] + genome[gs:gs + L - a], 0.02)
        reads.append(("chimera_%d" % i, seq, util.rand_qual(rng, len(seq), mean_q=rng.uniform(8, 25))))
    for i in range(6):
        seq = cont[100 * i:100 * i + int(rng.integers(1, 16))]
        reads.append(("tiny_%d" % i, seq, util.rand_qual(rng, len(seq))))
    half = cont[5000:5400] + util.rand_seq(rng, 400)
    reads.append(("exactly_half", half, util.rand_qual(rng, len(half), mean_q=20)))
    order = rng.permutation(len(reads))
    return genome, contam, [reads[i] for i in order]


def contam_percentages(contam, reads):
    k = orc.Kmers()
    k.add_assembly([contam])
    sc = orc.score([(s, q) for _, s, q in reads], orc.make_params(), k)
    return np.array([p.mean_q for p in sc.parents]), k


def fastq(reads):
    return b"".join(b"@" + n.encode() + b"\n" + s + b"\n+\n" + q + b"\n" for n, s, q in reads)


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("contam")
    genome, contam, reads = make_inputs()
    (d / "contam.fa").write_bytes(wrapped_fasta(b"lambda", contam))
    with gzip.open(d / "contam.fa.gz", "wb") as f:
        f.write(wrapped_fasta(b"lambda", contam))
    util.write_fasta(d / "sample.fa", [("chr", genome)], width=80)
    text = fastq(reads)
    (d / "reads.fastq").write_bytes(text)
    with gzip.open(d / "reads.fastq.gz", "wb") as f:
        f.write(text)
    c, k = contam_percentages(contam, reads)
    return dict(dir=d, genome=genome, contam=contam, reads=reads, text=text, c=c, kmers=k,
                fq=str(d / "reads.fastq"), gz=str(d / "reads.fastq.gz"), cfa=str(d / "contam.fa"), cgz=str(d / "contam.fa.gz"),
                sample=str(d / "sample.fa"), bases=sum(len(r[1]) for r in reads))


def test_fixture_covers_both_sides_of_the_threshold(inputs):
    """the oracle's percentages: reads are removed, reads with contaminant sequence are kept, one read sits exactly at
    50 % (kept: only c > P removes), and reads shorter than 16 bases score 0"""
    c, reads = inputs["c"], inputs["reads"]
    names = [r[0] for r in reads]
    assert c[names.index("exactly_half")] == 50.0
    chim = np.array([c[i] for i, n in enumerate(names) if n.startswith("chimera_")])
    assert (chim > 50).sum() >= 10 and ((chim > 5) & (chim <= 50)).sum() >= 10
    assert all(c[i] == 0.0 for i, n in enumerate(names) if n.startswith("tiny_"))
    assert (c > 20).sum() > (c > 50).sum() > 40


# ---- CLI configs: stdout equals the reference's run on the filtered input -----------------------------------------------
CONFIGS = [
    ["--contam", "C", "-p", "90"],
    ["--contam", "C", "--max_contam", "20", "-t", "1.5m", "--min_length", "1000"],
    ["--contam", "C", "-a", "S", "--trim", "--split", "500", "-p", "70"],   # at -p 80 the cut falls inside the class of 0 scores
    ["--contam", "C", "--trim_q", "10", "--trim", "--split", "500", "-p", "90"],
    ["--contam", "C"],
]


def resolve(config, inputs, contam=None):
    sub = {"C": contam or inputs["cfa"], "S": inputs["sample"]}
    return [sub.get(a, a) for a in config]


def filtered_args(config, input_bases):
    """the same options without --contam / --max_contam, and -p P as -t T = min(t, P/100 * all input bases)"""
    out, i, t, p = [], 0, None, None
    while i < len(config):
        a = config[i]
        if a in ("--contam", "--max_contam"):
            i += 2
        elif a == "-p":
            p, i = float(config[i + 1]), i + 2
        elif a == "-t":
            t, i = int(float(config[i + 1][:-1]) * 1e6) if config[i + 1].endswith("m") else int(config[i + 1]), i + 2
        elif a == "--trim":
            out, i = out + [a], i + 1
        else:
            out, i = out + config[i:i + 2], i + 2
    if p is not None or t is not None:
        out += ["-t", str(qm.derived_target(t, p, input_bases))]
    return out


def max_contam(config):
    return float(config[config.index("--max_contam") + 1]) if "--max_contam" in config else P_DEFAULT


def kept_reads(inputs, P):
    return [r for r, c in zip(inputs["reads"], inputs["c"]) if not c > P]


def reference_run(args):
    """The reference's run (oracle.run_refcli), replayed from RECORDED: the lines `FL_REFERENCE_RECORD=<file>` writes for
    these tests (recorded where oracle/_ref is built), xz-compressed, added to the oracle's replay store in memory."""
    global _recorded_loaded
    if not _recorded_loaded and not os.environ.get("FL_REFERENCE_RECORD"):
        store = orc._load_store()
        with lzma.open(RECORDED, "rt") as f:
            for line in f:
                if line.strip():
                    store.update(json.loads(line))
        _recorded_loaded = True
    return orc.run_refcli(args)


def reference_case(inputs, k, tmp):
    """(reference options, its input, its records) for config k: the input with the removed reads deleted and the same
    options, -p P as -t T. With --trim_q the reference has no such option: its input is then the FASTQ derived from the
    filtered input (one record per row, as tests/test_cli_qtrim.py states --trim_q), with --trim_q / --trim / --split
    dropped. No options left (--contam alone): the reference refuses to run, and stdout is the filtered input itself."""
    config = CONFIGS[k]
    kept = [(n, b"", s, q) for n, s, q in kept_reads(inputs, max_contam(config))]
    args = filtered_args(resolve(config, inputs), inputs["bases"])
    if "--trim_q" in config:
        Q, split = int(config[config.index("--trim_q") + 1]), int(config[config.index("--split") + 1])
        kept = qm.derived_reads(kept, Q, "--trim" in config, split)
        drop = {"--trim_q": 2, "--split": 2, "--trim": 1}
        out, i = [], 0
        while i < len(args):
            n = drop.get(args[i], 0)
            out, i = (out, i + n) if n else (out + args[i:i + 2], i + 2)
        args = out
    path = os.path.join(str(tmp), "reference_input_%d.fastq" % k)
    with open(path, "wb") as f:
        f.write(qm.fastq_bytes(kept))
    return args, path, kept


def model(inputs, args, records):
    """the oracle's rows for the reference's run of `args` on `records` (its parents, its finalised rows)"""
    kw, i, kmers = {}, 0, None
    while i < len(args):
        a = args[i]
        if a == "--trim":
            kw["trim"], i = True, i + 1
            continue
        v = args[i + 1]
        if a == "-a":
            kmers = orc.Kmers()
            kmers.add_assembly([inputs["genome"]])
        else:
            kw[{"-t": "target_bases", "--min_length": "min_length", "--split": "split"}[a]] = int(v)
        i += 2
    op = orc.make_params(**kw)
    sc = orc.finalize(orc.score([(r[2], r[3]) for r in records], op, kmers), op)
    names = []
    for row in sc.rows:
        n = records[row.parent][0]
        names.append(n if sc.parents[row.parent].n_child == 0 else "%s_%d-%d" % (n, row.start + 1, row.end))
    return sc, names


@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_reference_on_the_filtered_input_equals_the_model(inputs, k, tmp_path):
    """the recorded reference run on the filtered input keeps exactly the rows the oracle keeps; each config removes
    reads and keeps reads that hold contaminant sequence; no exact tie class of final scores straddles the cut"""
    P = max_contam(CONFIGS[k])
    c = inputs["c"]
    assert (c > P).sum() > 0 and ((c > 0) & ~(c > P)).sum() > 0
    args, path, records = reference_case(inputs, k, tmp_path)
    if not args:
        return
    sc, names = model(inputs, args, records)
    kept = [r.final_score for r in sc.rows if r.passed_final]
    dropped = [r.final_score for r in sc.rows if r.passed and not r.passed_final]
    assert kept and not (set(kept) & set(dropped))
    rc, out, err = reference_run(args + [path])
    assert rc == 0, err[-2000:]
    assert orc.fastq_names(out) == [n for n, r in zip(names, sc.rows) if r.passed_final]


@need_cli
@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_stdout_equals_the_reference_on_the_filtered_input(inputs, k, tmp_path):
    config = CONFIGS[k]
    args, path, records = reference_case(inputs, k, tmp_path)
    rc, out, err = run(resolve(config, inputs) + [inputs["fq"]])
    assert rc == 0, err[-2000:]
    assert len(out) > 0
    if args:
        rc_r, ref, err_r = reference_run(args + [path])
        assert rc_r == 0 and out == ref
    else:
        assert out == qm.fastq_bytes(records)
    if "--trim_q" in config:                                  # and this CLI's own --trim_q run on the filtered input
        filtered = tmp_path / "filtered.fastq"
        filtered.write_bytes(fastq(kept_reads(inputs, max_contam(config))))
        rc_q, out_q, err_q = run(filtered_args(resolve(config, inputs), inputs["bases"]) + [str(filtered)])
        assert rc_q == 0 and out_q == out, err_q[-2000:]
    P = max_contam(config)
    n_removed = int((inputs["c"] > P).sum())
    assert 0 < n_removed < len(inputs["reads"])
    lines = log_lines(err.decode())
    removed_bases = sum(len(r[1]) for r, c in zip(inputs["reads"], inputs["c"]) if c > P)
    assert "  %d reads (%d bp) with more than %g%% of bases in contaminant 16-mers" % (n_removed, removed_bases, P) in lines
    if k:
        return
    variants = [(config, inputs["gz"], None, None), (config, "-", inputs["text"], None),
                (config, inputs["fq"], None, {"FL_CHUNK_MB": "1"}), (config, inputs["fq"], None, {"FL_HOST_PARSER": "1"})]
    if gpu_count() >= 2:
        variants.append((["--gpus", "2"] + config, inputs["fq"], None, {"FL_CHUNK_MB": "1"}))
    for cfg, path, data, env in variants:
        rc, o, e = run(resolve(cfg, inputs, inputs["cgz"]) + [path], data, env)
        assert rc == 0 and o == out, (path, env, e[-2000:])
    rc, z, e = run(["--bgzip"] + resolve(config, inputs) + [inputs["fq"]])
    assert rc == 0 and gzip.decompress(z) == out


def gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 1


@need_cli
@pytest.mark.gpu
def test_bam_input(inputs, tmp_path):
    recs = [(n.encode(), s.upper(), bytes(x - 33 for x in q), b"") for n, s, q in inputs["reads"] if len(s) > 0]
    raw = bu.bam_of(recs, bu.header(refs=[(b"chr1", 150000)]))
    (tmp_path / "r.bam").write_bytes(bu.bgzf(raw))
    (tmp_path / "r.fastq").write_bytes(bu.to_fastq(raw))
    config = resolve(CONFIGS[0], inputs)
    rc_f, out_f, err_f = run(config + [str(tmp_path / "r.fastq")])
    rc_b, out_b, err_b = run(config + [str(tmp_path / "r.bam")])
    assert rc_f == rc_b == 0, err_b[-2000:]
    raw_out = gzip.decompress(out_b)
    assert raw_out[:bu.header_end(raw)] == raw[:bu.header_end(raw)]
    assert bu.to_fastq(raw_out) == out_f and len(out_f) > 0


@need_cli
@pytest.mark.gpu
def test_failed_file_is_the_complement(inputs, tmp_path):
    failed = tmp_path / "failed.fastq"
    config = resolve(CONFIGS[0], inputs)
    rc, out, err = run(config + ["--failed", str(failed), inputs["fq"]])
    assert rc == 0, err[-2000:]
    got = {r[0] for r in util.read_fastx(io_path(tmp_path, out))} | {r[0] for r in util.read_fastx(str(failed))}
    assert got == {r[0] for r in inputs["reads"]}
    kept = {r[0] for r in util.read_fastx(io_path(tmp_path, out))}
    assert not kept & {r[0] for r in util.read_fastx(str(failed))}
    removed = {r[0] for r, c in zip(inputs["reads"], inputs["c"]) if c > P_DEFAULT}
    assert removed and removed <= {r[0] for r in util.read_fastx(str(failed))}


def io_path(tmp_path, data):
    p = tmp_path / "stdout.fastq"
    p.write_bytes(data)
    return str(p)


@need_cli
@pytest.mark.gpu
def test_an_empty_contaminant_set_changes_nothing(inputs, tmp_path):
    fa = util.write_fasta(tmp_path / "short.fa", [("a", b"ACGTACGTAC"), ("b", b"ACGTACGTACGTACG")])
    rc0, out0, err0 = run(["-p", "90", inputs["fq"]])
    rc1, out1, err1 = run(["--contam", fa, "-p", "90", inputs["fq"]])
    assert rc0 == rc1 == 0 and out0 == out1 and len(out0) > 0
    assert "  2 contigs, 0 16-mers" in log_lines(err1.decode())
    assert "  0 reads (0 bp) with more than 50% of bases in contaminant 16-mers" in log_lines(err1.decode())


@need_cli
@pytest.mark.gpu
def test_log_and_verbose(inputs, tmp_path):
    rc, out, err = run(resolve(CONFIGS[0], inputs) + ["--verbose", inputs["fq"]])
    assert rc == 0
    text = err.decode()
    n = len(inputs["kmers"])
    lines = log_lines(text)
    i = lines.index("Hashing 16-mers from contaminant sequences")
    assert lines[i + 1].strip() == inputs["cfa"]
    assert "  1 contig, %d 16-mers" % n in lines
    p = -np.expm1(16 * np.log1p(-n / 4.0 ** 16))
    assert "  a random base lies in one of them with probability %.3g" % p in lines
    assert i < lines.index("Removing contaminant reads") < lines.index("Filtering long reads")
    table = text[text.index("Read name\tLength score"):]
    listed = {l.split("\t")[0].strip() for l in table.splitlines()[1:] if "\t" in l}
    removed = {r[0] for r, c in zip(inputs["reads"], inputs["c"]) if c > P_DEFAULT}
    assert listed and not listed & removed
    assert not [n for n in removed if "\n%s\n" % n in text]               # nor a per-read block
    assert len(listed) == len(inputs["reads"]) - len(removed)
    rc2, out2, _ = run(resolve(CONFIGS[0], inputs) + [inputs["fq"]])
    assert out == out2


# ---- the C ABI ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_set_equals_the_reference_set(inputs):
    from filtlong_b200 import api
    text = open(inputs["cfa"], "rb").read()
    want = inputs["kmers"].dump()
    with api.Context() as a, api.Context() as b, api.Context() as h:
        r = a.contam_add_text(text, fastq=False)
        assert r["status"] == "ok" and r["n"] == 1
        b.kmers_add_text(text, fastq=False)
        h.contam_add([inputs["contam"]])                               # the host-batch path
        got = a.contam_export()
        assert np.array_equal(got, want) and np.array_equal(b.kmers_export(), want)
        assert np.array_equal(h.contam_export(), want)
        assert a.kmers_count() == 0                                    # not a reference: still Phred mode


def _push_all(ctx, reads, how):
    from filtlong_b200 import api
    import torch
    seqs, quals = [r[1] for r in reads], [r[2] for r in reads]
    if how == "push":
        ctx.push(api.HostBatch(seqs, quals, want_seq=True))
    elif how == "push_text":
        r = ctx.push_text(fastq(reads))
        assert r["status"] == "ok"
    elif how == "push_device":
        hb = api.HostBatch(seqs, quals, want_seq=False)
        asc = np.zeros(max(hb.padded_bases, 1), np.uint8)
        for i, s in enumerate(seqs):
            asc[int(hb.off[i]):int(hb.off[i]) + len(s)] = np.frombuffer(s, np.uint8)
        dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
               dict(off=hb.off.view(np.int64), len=hb.len, qual=hb.qual, ascii=asc).items()}
        ctx.push_device(api.device_batch(hb.n, hb.padded_bases, dev["off"], dev["len"], qual=dev["qual"], ascii=dev["ascii"]))
        torch.cuda.synchronize()
    elif how == "push_bam":
        recs = [(n.encode(), s.upper(), bytes(x - 33 for x in q), b"") for n, s, q in reads]
        raw = bu.bam_of(recs, bu.header(refs=[(b"chr1", 1000)]))
        recs_at = list(bu.records(raw))
        so = [r["seq_off"] for r in recs_at]
        qo = [r["qual_off"] for r in recs_at]
        ctx.push_bam(raw, so, qo, [len(r[1]) for r in reads])


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["push", "push_text", "push_device", "push_bam"])
@pytest.mark.parametrize("with_reference", [False, True])
def test_percentages_are_the_oracle_mean(inputs, how, with_reference):
    from filtlong_b200 import api
    P = 30.0
    reads = [r for r in inputs["reads"] if len(r[1]) > 0]
    if how == "push":
        reads = reads + [("empty", b"", b"")]
    c = contam_percentages(inputs["contam"], reads)[0]
    with api.Context(api.make_params(max_contam=P, keep_percent=90)) as ctx:
        if with_reference:
            ctx.kmers_add_text(open(inputs["sample"], "rb").read(), fastq=False)
        ctx.contam_add_text(open(inputs["cfa"], "rb").read(), fastq=False)
        _push_all(ctx, reads, how)
        pct, removed, counts = ctx.contam_results()
    assert len(pct) == len(reads)
    assert np.array_equal(pct.view(np.uint64)[~np.isnan(c)], c.view(np.uint64)[~np.isnan(c)])
    assert np.array_equal(np.isnan(pct), np.isnan(c)) and (how != "push" or np.isnan(pct[-1]))
    assert np.array_equal(removed, c > P)
    assert counts["reads"] == int((c > P).sum()) > 0
    assert counts["bases"] == sum(len(r[1]) for r, x in zip(reads, c) if x > P)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(keep_percent=90.0), dict(target_bases=1500000, min_length=1000),
                                dict(keep_percent=80.0, trim=True, split=500)])
def test_finalize_ranks_only_the_kept_reads(inputs, kw):
    from filtlong_b200 import api
    from tests import select_model
    reads = inputs["reads"]
    kept = kept_reads(inputs, P_DEFAULT)
    ref = kw.get("trim", False)
    total = inputs["bases"]

    def ctx_for(rs, contam):
        ctx = api.Context(api.make_params(**kw))
        if ref:
            ctx.kmers_add_text(open(inputs["sample"], "rb").read(), fastq=False)
        if contam:
            ctx.contam_add_text(open(inputs["cfa"], "rb").read(), fastq=False)
        ctx.push(api.HostBatch([r[1] for r in rs], [r[2] for r in rs], want_seq=True))
        return ctx

    with ctx_for(reads, True) as a, ctx_for(kept, False) as b:
        sa, sb = a.finalize(total), b.finalize(total)
        ra, rb = a.row_results(), b.row_results()
        _, removed, counts = a.contam_results()
        parent_removed = removed[ra["parent"]]
        assert counts["rows"] == int(parent_removed.sum()) > 0
        assert not ra["passed_final"][parent_removed].any()
        for k in ("start", "end", "mean_q", "window_q", "passed_final"):
            assert np.array_equal(ra[k][~parent_removed], rb[k]), k
        for f in ("min_q", "max_q", "status", "target", "passed_bases", "keeping", "total_bases", "rows_bases"):
            assert getattr(sa, f) == getattr(sb, f), f
        select_model.check_stats(sa, rb["mean_q"])

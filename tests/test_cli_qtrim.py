"""`filtlong --trim_q Q --trim / --split N`: trimming and splitting on Phred qualities when there is no reference.

The option's statement, and what these tests check: stdout equals what the same build prints in plain Phred mode on the
DERIVED FASTQ -- one record per row (the row's name, the parent's comment, the substring's bases and qualities) -- with
the same thresholds and `-p P` replaced by `-t T`, T = min(t, P/100 * input bases) (main.cpp:229-237). The reference's
own run on each derived FASTQ is recorded in tests/golden/qtrim_reference_runs.jsonl.xz; the CPU test checks it against the
model, the GPU tests check this CLI against it. The argument errors are checked before any read is scored and need no
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
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORDED = os.path.join(ROOT, "tests", "golden", "qtrim_reference_runs.jsonl.xz")
_recorded_loaded = False


def reference_run(args):
    """The reference's run on a derived FASTQ (oracle.run_refcli). The runs are replayed from RECORDED, which holds the
    lines that `FL_REFERENCE_RECORD=<file>` writes for these tests (recorded where oracle/_ref is built), xz-compressed;
    they are added to the oracle's replay store in memory, and nothing is written."""
    global _recorded_loaded
    if not _recorded_loaded and not os.environ.get("FL_REFERENCE_RECORD"):
        store = orc._load_store()
        with lzma.open(RECORDED, "rt") as f:
            for line in f:
                if line.strip():
                    store.update(json.loads(line))
        _recorded_loaded = True
    return orc.run_refcli(args)


def run(args, stdin_data=None, env_extra=None):
    env = dict(os.environ, LC_ALL="C", **(env_extra or {}))
    env.pop("LANG", None)
    p = subprocess.run([CLI] + list(args), input=stdin_data, capture_output=True, env=env, timeout=TIMEOUT)
    return p.returncode, p.stdout, p.stderr


# ---- argument errors (no GPU) -----------------------------------------------------------------------------------------
ERRORS = [
    (["--trim_q", "10", "--trim", "-a", "FA", "FQ"], "Error: --trim_q cannot be used with an assembly or read reference"),
    (["--trim_q", "10", "--split", "50", "-1", "FQ", "FQ"], "Error: --trim_q cannot be used with an assembly or read reference"),
    (["--trim_q", "10", "--trim", "-2", "FQ", "FQ"], "Error: --trim_q cannot be used with an assembly or read reference"),
    (["--trim_q", "10", "-p", "90", "FQ"], "Error: --trim_q needs --trim or --split"),
    (["--trim_q", "0", "--trim", "FQ"], "Error: the value for --trim_q must be an integer from 1 to 93"),
    (["--trim_q", "94", "--trim", "FQ"], "Error: the value for --trim_q must be an integer from 1 to 93"),
    (["--trim_q", "-5", "--trim", "FQ"], "Error: the value for --trim_q must be an integer from 1 to 93"),
    (["--trim_q", "7.5", "--trim", "FQ"], "Error: the value for --trim_q must be an integer from 1 to 93"),
    (["--trim_q", "1k", "--trim", "FQ"], "Error: the value for --trim_q must be an integer from 1 to 93"),
    (["--trim_q", "", "--trim", "FQ"], "Error: the value for --trim_q must be an integer from 1 to 93"),
    (["--trim", "FQ"], "Error: assembly or read reference is required to use --trim"),
    (["--split", "100", "-p", "90", "FQ"], "Error: assembly or read reference is required to use --split"),
]


@need_cli
@pytest.mark.parametrize("args,message", ERRORS, ids=lambda x: " ".join(x) if isinstance(x, list) else None)
def test_argument_errors(args, message, tmp_path):
    fq = util.write_fastq(tmp_path / "x.fastq", [("r1", b"ACGT" * 10, b"I" * 40)])
    fa = util.write_fasta(tmp_path / "a.fasta", [("c", b"ACGT" * 10)])
    rc, out, err = run([fq if a == "FQ" else (fa if a == "FA" else a) for a in args])
    assert (rc, out, err.decode()) == (1, b"", message + "\n")


@need_cli
def test_help_lists_trim_q():
    rc, out, err = run(["--help"])
    text = err.decode()
    assert "--trim_q [int]" in text
    assert text.index("read manipulation:") < text.index("--trim_q") < text.index("other:")


# ---- inputs and their derived FASTQs ----------------------------------------------------------------------------------
CONFIGS = [
    ["--trim_q", "10", "--trim", "--split", "500", "-p", "90"],
    ["--trim_q", "7", "--split", "32", "-t", "1500000"],
    ["--trim_q", "20", "--trim", "-p", "80", "--window_size", "100"],
    ["--trim_q", "12", "--trim", "--split", "1", "--min_mean_q", "80", "-p", "95", "-t", "2000000"],
]


def make_reads(seed=77, n=400):
    """(name, comment, seq, qual): long reads with low-quality blocks spliced into their qualities"""
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, 80000)
    out = []
    for i, (name, seq, qual) in enumerate(util.long_reads(rng, genome, n, max_len=15000, lower_frac=0.0)):
        q = bytearray(qual)
        for _ in range(int(rng.integers(0, 4))):
            ln = int(rng.integers(1, 900))
            s = int(rng.integers(0, max(len(q), 1)))
            q[s:s + ln] = bytes(rng.integers(33, 39, size=len(q[s:s + ln])).astype(np.uint8))
        out.append((name, b"ch=%d x" % i if i % 3 == 0 else b"", seq, bytes(q)))
    return out


def options(config):
    """(Q, trim, split, oracle / model keyword thresholds) of a config"""
    Q, trim, split, kw, i = None, False, None, {}, 0
    names = {"-p": "keep_percent", "-t": "target_bases", "--min_mean_q": "min_mean_q", "--window_size": "window_size"}
    while i < len(config):
        a = config[i]
        if a == "--trim":
            trim, i = True, i + 1
            continue
        v = config[i + 1]
        if a == "--trim_q":
            Q = int(v)
        elif a == "--split":
            split = int(v)
        else:
            kw[names[a]] = float(v) if a in ("-p", "--min_mean_q") else int(v)
        i += 2
    return Q, trim, split, kw


def derived_args(config, input_bases):
    """the plain Phred run on the derived FASTQ: no --trim_q / --trim / --split, -p P as -t T"""
    Q, trim, split, kw = options(config)
    out, i = [], 0
    while i < len(config):
        if config[i] == "--trim":
            i += 1
        elif config[i] in ("--trim_q", "--split", "-p", "-t"):
            i += 2
        else:
            out += config[i:i + 2]
            i += 2
    if "keep_percent" in kw or "target_bases" in kw:
        out += ["-t", str(qm.derived_target(kw.get("target_bases"), kw.get("keep_percent"), input_bases))]
    return out


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("qtrim_cli")
    reads = make_reads()
    text = qm.fastq_bytes(reads)
    (d / "reads.fastq").write_bytes(text)
    with gzip.open(d / "reads.fastq.gz", "wb") as f:
        f.write(text)
    bases = sum(len(r[2]) for r in reads)
    cases = []
    for k, config in enumerate(CONFIGS):
        Q, trim, split, kw = options(config)
        derived = qm.derived_reads(reads, Q, trim, split)
        path = d / ("derived_%d.fastq" % k)
        path.write_bytes(qm.fastq_bytes(derived))
        sc = qm.score_rows([(r[2], r[3]) for r in reads], Q, dict(kw, trim=trim, split=split))
        cases.append(dict(config=config, derived=derived, path=str(path), args=derived_args(config, bases), sc=sc))
    return dict(dir=d, reads=reads, fq=str(d / "reads.fastq"), gz=str(d / "reads.fastq.gz"), text=text, cases=cases)


def expected_stdout(case):
    return qm.fastq_bytes([r for r, row in zip(case["derived"], case["sc"].rows) if row.passed_final])


@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_reference_on_the_derived_fastq_equals_the_model(inputs, k):
    """the recorded reference run on the derived FASTQ keeps exactly the rows the model keeps; no exact tie class of
    final scores straddles the cut, so the selection is not decided by the order of a sort"""
    case = inputs["cases"][k]
    rows = case["sc"].rows
    assert len(rows) == len(case["derived"])
    assert sum(len(c) for c in case["sc"].children) > 50               # the config does trim or split reads
    kept = [r.final_score for r in rows if r.passed_final]
    dropped = [r.final_score for r in rows if r.passed and not r.passed_final]
    assert kept and not (set(kept) & set(dropped))
    rc, out, err = reference_run(case["args"] + [case["path"]])
    assert rc == 0, err[-2000:]
    assert out == expected_stdout(case)


# ---- the CLI on the GPU -----------------------------------------------------------------------------------------------
def gpu_count():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 1


@need_cli
@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_stdout_equals_the_plain_run_on_the_derived_fastq(inputs, k):
    case = inputs["cases"][k]
    rc, ref, err = reference_run(case["args"] + [case["path"]])
    rc_d, out_d, err_d = run(case["args"] + [case["path"]])
    assert rc_d == 0, err_d[-2000:]
    rc_q, out_q, err_q = run(case["config"] + [inputs["fq"]])
    assert rc_q == 0, err_q[-2000:]
    assert out_q == out_d and ref == out_q and len(out_q) > 0
    if k:
        return
    variants = [(case["config"] + [inputs["gz"]], None, None), (case["config"] + ["-"], inputs["text"], None),
                (case["config"] + [inputs["fq"]], None, {"FL_CHUNK_MB": "1"}), (case["config"] + [inputs["fq"]], None, {"FL_HOST_PARSER": "1"})]
    if gpu_count() >= 2:
        variants.append((["--gpus", "2"] + case["config"] + [inputs["fq"]], None, {"FL_CHUNK_MB": "1"}))
    for args, data, env in variants:
        rc, out, err = run(args, data, env)
        assert rc == 0 and out == out_q, (args[-1], env, err[-2000:])
    rc, z, err = run(["--bgzip"] + case["config"] + [inputs["fq"]])
    assert rc == 0 and gzip.decompress(z) == out_q


@need_cli
@pytest.mark.gpu
def test_bam_input_gives_the_records_of_its_fastq_equivalent(inputs, tmp_path):
    recs = [(n.encode(), s.upper(), bytes(x - 33 for x in q), (bu.aux_z(b"RG", b"rg1") if i % 2 else b"") +
             bu.aux_z(b"MM", b"C+m?,0,1;")) for i, (n, _, s, q) in enumerate(inputs["reads"][:250])]
    raw = bu.bam_of(recs, bu.header(refs=[(b"chr1", 80000)]))
    (tmp_path / "r.bam").write_bytes(bu.bgzf(raw))
    (tmp_path / "r.fastq").write_bytes(bu.to_fastq(raw))
    config = CONFIGS[0]
    rc_f, out_f, err_f = run(config + [str(tmp_path / "r.fastq")])
    rc_b, out_b, err_b = run(config + [str(tmp_path / "r.bam")])
    assert rc_f == rc_b == 0, err_b[-2000:]
    raw_out = gzip.decompress(out_b)
    assert raw_out[:bu.header_end(raw)] == raw[:bu.header_end(raw)]
    assert bu.to_fastq(raw_out) == out_f and len(out_f) > 0
    children = [r for r in bu.records(raw_out) if b"-" in r["name"].rsplit(b"_", 1)[-1]]
    assert children and all([t for t, _ in bu.aux_fields(r["aux"])] in ([], [b"RG"]) for r in children)


@need_cli
@pytest.mark.gpu
def test_failed_file_is_the_complement(inputs, tmp_path):
    case = inputs["cases"][0]
    failed = tmp_path / "failed.fastq"
    rc, out, err = run(case["config"] + ["--failed", str(failed), inputs["fq"]])
    assert rc == 0, err[-2000:]
    assert out == expected_stdout(case)
    assert failed.read_bytes() == qm.fastq_bytes([r for r, row in zip(case["derived"], case["sc"].rows) if not row.passed_final])


@need_cli
@pytest.mark.gpu
def test_verbose_prints_the_model_ranges(inputs):
    case = inputs["cases"][1]
    Q, trim, split, _ = options(case["config"])
    rc, out, err = run(case["config"] + ["--verbose", inputs["fq"]])
    assert rc == 0 and out == expected_stdout(case)
    want = []
    for m in qm.read_rows([(r[2], r[3]) for r in inputs["reads"]], Q, trim, split):
        if m["bad"]:
            want.append("bad ranges = " + ", ".join("%d-%d" % b for b in m["bad"]))
        if m["children"]:
            want.append("child ranges = " + ", ".join("%d-%d" % c for c in m["children"]))
    got = [l.strip() for l in log_lines(err.decode()) if l.strip().startswith(("bad ranges = ", "child ranges = "))]
    assert got == want and len(want) > 0

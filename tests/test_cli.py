"""The `filtlong` drop-in command line (filtlong_b200/bin/filtlong) against the unmodified
reference binary (oracle/_ref/filtlong_ref, its runs replayed from tests/golden): byte-identical stdout, and the stderr log lines the
reference's own tests assert (test/test_sort.py, test_trim.py, test_split.py,
test_error_messages.py, test_unit_suffixes.py). Argument errors need no GPU; everything that
scores reads is marked gpu."""
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")
need_cli = pytest.mark.skipif(not os.path.exists(CLI), reason="CLI not built")


def run(binary, args, cwd=None):
    env = dict(os.environ, LC_ALL="C")
    env.pop("LANG", None)
    p = subprocess.run([binary] + list(args), capture_output=True, env=env, cwd=cwd)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


def log_lines(err):
    """stderr without progress redraws (\\r...) and blank lines."""
    out = []
    for line in err.replace("\r", "\n").split("\n"):
        line = line.rstrip()
        if line:
            out.append(line)
    return out


def final_lines(err):
    """Keeps, for every run of progress redraws, only the last one."""
    lines = []
    for chunk in err.split("\n"):
        parts = chunk.split("\r")
        last = parts[-1].rstrip()
        if last:
            lines.append(last)
    return lines


ERROR_CASES = [
    [], ["--help"], ["-h"], ["--version"],
    ["--target_bases=100", "X"], ["--bogus", "X"], ["-x", "X"], ["X", "X", "-t", "10"], ["-t", "X"], ["-t"],
    ["--target_bases"], ["-p", "50", "-t"], ["-q", "-1", "X"], ["--window_size", "10k", "-t", "5", "X"],
    ["-t", "1e3", "X"], ["--min_length", "99999999999", "X"], ["--version", "--bogus"], ["-t", "0", "X"],
    ["-t", "-10", "X"], ["--target_bases", "-10", "X"], ["-l", "0", "X"], ["-L", "-5", "X"],
    ["-t", "5", "nonexist.fq"], ["-a", "nonexist.fa", "-t", "5", "X"], ["-1", "nonexist.fq", "-t", "5", "X"],
    ["--keep_percent", "100", "X"], ["--keep_percent", "0", "X"], ["-p", "abc", "X"], ["--trim", "X"],
    ["--split", "100", "X"], ["X"], ["-t", "5"], ["--min_mean_q", "0", "X"], ["--min_window_q", "0", "X"],
    ["--length_weight", "-1", "-t", "5", "X"], ["--split", "0", "-a", "X", "X"], ["--window_size", "0", "-t", "5", "X"],
    ["--window_size", "-3", "-t", "5", "X"], ["-t", "5k", "--split", "1x", "-a", "X", "X"], ["-t", "k", "X"],
    ["-t", "", "X"], ["-t", "5", "-t", "6", "-l", "1.5K", "--max_length", "2MB", "--bogus2", "X"],
    ["-ht", "5"], ["-t5", "--min_length", "1e2", "X"],
]


@need_cli
@pytest.mark.parametrize("case", ERROR_CASES, ids=lambda c: " ".join(c) or "noargs")
def test_argument_handling_matches_reference(case, tmp_path):
    """No read is scored in any of these: exit code and stderr must match the reference verbatim
    (help text only by the substrings the reference's tests check)."""
    fq = util.write_fastq(tmp_path / "x.fastq", [("r1", b"ACGT" * 10, b"I" * 40)])
    args = [fq if a == "X" else a for a in case]
    rc_r, out_r, err_r = orc.run_refcli(args, cwd=tmp_path)
    rc_o, out_o, err_o = run(CLI, args, cwd=tmp_path)
    assert rc_o == rc_r
    assert out_o == out_r
    if "usage:" in err_r:
        assert "usage:" in err_o and "Filtlong:" in err_o          # test_error_messages.py:59-62
    else:
        assert err_o == err_r


def make_inputs(tmp_path, seed=5, n=150):
    rng = np.random.default_rng(seed)
    genome = util.rand_seq(rng, 60000)
    reads = util.long_reads(rng, genome, n, max_len=9000)
    reads.append(("with_comment extra words\there", util.rand_seq(rng, 900), util.rand_qual(rng, 900)))
    reads.append(("junk_only", util.rand_seq(rng, 800), b"5" * 800))
    reads.append(("sandwich", util.rand_seq(rng, 60) + genome[9000:9400] + util.rand_seq(rng, 300) + genome[12000:12500], b"7" * 1260))
    fq = tmp_path / "reads.fastq"
    with open(fq, "wb") as f:
        for i, (name, seq, qual) in enumerate(reads):
            nl = b"\r\n" if i % 7 == 3 else b"\n"                       # some CRLF records
            f.write(b"@" + name.encode() + nl + seq + nl + b"+" + (name.encode() if i % 5 == 0 else b"") + nl + qual + nl)
    fa = util.write_fasta(tmp_path / "asm.fasta", [("contig_1", genome[:35000]), ("contig_2", genome[35000:])], width=60)
    r1, r2 = util.short_reads(rng, genome, 9000)
    s1 = util.write_fastq(tmp_path / "s1.fastq", r1)
    s2 = util.write_fastq(tmp_path / "s2.fastq.gz", r2)
    fasta_reads = util.write_fasta(tmp_path / "reads.fasta", [(n, s) for n, s, _ in reads[:60]], width=80)
    return str(fq), fa, s1, s2, fasta_reads


RUN_CASES = [
    ["--min_length", "1", "--keep_percent", "90", "FQ"],                       # BASELINE config 1 shape
    ["-t", "300000", "FQ"],
    ["-p", "60", "--min_mean_q", "70", "--window_size", "100", "FQ"],
    ["-t", "1g", "FQ"],                                                         # not enough reads
    ["-t", "1000", "-l", "100000", "FQ"],                                       # already below target
    ["-a", "FA", "-p", "90", "FQ"],
    ["-a", "FA", "-p", "80", "--trim", "--split", "100", "FQ"],
    ["-a", "FA", "--trim", "FQ"],
    ["-a", "FA", "--split", "30", "-t", "250000", "--length_weight", "2", "--mean_q_weight", "0.5", "FQ"],
    ["-1", "S1", "-2", "S2", "-p", "85", "--trim", "--split", "250", "FQ"],
    ["-a", "FA", "-1", "S1", "-2", "S2", "-p", "85", "FQ"],
    ["-a", "FA", "-p", "70", "--trim", "--split", "80", "FASTA"],
    ["-a", "FA", "-p", "80", "--trim", "--split", "100", "--verbose", "FQ"],
    ["-p", "80", "--verbose", "FQ"],
]


@need_cli
@pytest.mark.gpu
@pytest.mark.parametrize("case", RUN_CASES, ids=lambda c: " ".join(c))
def test_cli_output_matches_reference(case, tmp_path):
    fq, fa, s1, s2, fasta_reads = make_inputs(tmp_path)
    sub = {"FQ": fq, "FA": fa, "S1": s1, "S2": s2, "FASTA": fasta_reads}
    args = [sub.get(a, a) for a in case]
    rc_r, out_r, err_r = orc.run_refcli(args)
    rc_o, out_o, err_o = run(CLI, args)
    assert rc_o == rc_r == 0, err_o[-2000:]
    assert out_o == out_r, "stdout differs"
    if "--verbose" in case:
        # per-read blocks and the score table print the same numbers at 2 decimals
        assert [l for l in log_lines(err_o) if "bp)" not in l] == [l for l in log_lines(err_r) if "bp)" not in l]
    else:
        assert final_lines(err_o) == final_lines(err_r)


@need_cli
@pytest.mark.gpu
def test_cli_runtime_errors_match_reference(tmp_path):
    good = [("a", b"ACGT" * 30, b"I" * 120), ("b", b"ACGT" * 30, b"I" * 120)]
    dup = util.write_fastq(tmp_path / "dup.fastq", good + [("a", b"ACGT" * 20, b"I" * 80)])
    bad = tmp_path / "bad.fastq"
    bad.write_bytes(b"@a\nACGTACGT\n+\nIIIIIIII\n@b\nACGTACGT\n+\nIIIIIII\n")
    fa = util.write_fasta(tmp_path / "reads.fasta", [("a", b"ACGT" * 30)])
    mixed = tmp_path / "mixed.fastq"
    mixed.write_bytes(b"@a\nACGTACGT\n+\nIIIIIIII\n>b\nACGTACGT\n")
    ref_bad = os.path.join(util.REF_FIXTURES, "test_bad_fastq.fastq")             # the reference suite's test_bad_fastq
    for args in (["-t", "100", dup], ["-t", "100", str(bad)], ["-t", "100", fa], ["-t", "100", str(mixed)],
                 ["--target_bases", "1000", ref_bad]):
        rc_r, out_r, err_r = orc.run_refcli(args)
        rc_o, out_o, err_o = run(CLI, args)
        assert (rc_o, out_o) == (rc_r, out_r)
        assert final_lines(err_o) == final_lines(err_r)

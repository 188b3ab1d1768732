"""The short-read 16-mer build on the device against the exact models of tests/bloom_model.py, on inputs designed to
reach each path of the Bloom false-positive rule (kmers.cpp:142-166): through every entry point that adds short
reads, with the set resolved between any two batches, and through the CLI against recorded runs of the reference.

Every multiple-copy context holds 49 GiB of build state: each test opens one at a time and closes it."""
import os
import subprocess

import numpy as np
import pytest

from filtlong_b200 import api
from oracle import oracle as orc
from tests import bloom_model as bm

pytestmark = pytest.mark.gpu

DESIGNS = bm.designs()
BY_NAME = {d.name: d for d in DESIGNS}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def units(reads):
    """the reads one by one, except that runs of reads under 16 bases (fillers) stay together"""
    out, in_run = [], False
    for seq in reads:
        if len(seq) < 16 and in_run:
            out[-1].append(seq)
        else:
            out.append([seq])
            in_run = len(seq) < 16
    return out


def fastq(reads, first=0):
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (first + i, s, b"I" * len(s)) for i, s in enumerate(reads))


def check_set(ctx, d):
    want = sorted(bm.model_set(d.files, d.assembly))
    assert ctx.kmers_export().tolist() == want
    named = [k for k, _, _ in d.expect.values()]
    assert ctx.kmers_contains(named).tolist() == [m for _, m, _ in d.expect.values()]


def add_assembly(ctx, d):
    if d.assembly:
        ctx.kmers_add(d.assembly, False)


@pytest.mark.parametrize("name", list(BY_NAME))
def test_one_batch(name):
    d = BY_NAME[name]
    with api.Context(api.make_params(min_length=1)) as ctx:
        add_assembly(ctx, d)
        ctx.kmers_add(d.files[0] + d.files[1], True)
        check_set(ctx, d)


@pytest.mark.parametrize("name", list(BY_NAME))
def test_one_batch_per_read_resolved_between_batches(name):
    """fl_kmers_finalize after every batch: the set so far is the model's set of the reads so far (the closed form of a
    prefix of the stream), and resolving it mid-stream does not change the final set"""
    d = BY_NAME[name]
    with api.Context(api.make_params(min_length=1)) as ctx:
        add_assembly(ctx, d)
        done = [[], []]
        named = [k for k, _, _ in d.expect.values()]
        for f in (0, 1):
            for u in units(d.files[f]):
                ctx.kmers_add(u, True)
                done[f] += u
                if any(len(s) >= 16 for s in u):
                    want = bm.model_set(done, d.assembly)
                    assert ctx.kmers_count() == len(want)
                    assert ctx.kmers_contains(named).tolist() == [k in want for k in named]
        check_set(ctx, d)


def test_mid_stream_count_shows_the_false_positive_16mer():
    d = BY_NAME["covered_before_first_sighting"]
    x = d.expect["covered"][0]
    reads = d.files[0]
    third = [i for i, s in enumerate(reads) if s == bm.kmer_seq(x)][2]
    with api.Context(api.make_params(min_length=1)) as ctx:
        ctx.kmers_add(reads[:third], True)
        assert not ctx.kmers_contains([x])[0]
        ctx.kmers_add(reads[third:third + 1], True)
        assert ctx.kmers_contains([x])[0]                 # in at its third sighting
        ctx.kmers_add(reads[third + 1:], True)
        check_set(ctx, d)


@pytest.mark.parametrize("per_record", [False, True], ids=["whole_files", "chunk_per_record"])
@pytest.mark.parametrize("name", list(BY_NAME))
def test_text(name, per_record):
    """fl_kmers_add_text on each file as FASTQ, whole or cut at every record boundary (a run of fillers stays whole)"""
    d = BY_NAME[name]
    with api.Context(api.make_params(min_length=1)) as ctx:
        if d.assembly:
            r = ctx.kmers_add_text(b"".join(b">c%d\n%s\n" % (i, s) for i, s in enumerate(d.assembly)), fastq=False)
            assert r["status"] == "ok"
        for f in (0, 1):
            pieces = units(d.files[f]) if per_record else [d.files[f]]
            first = 0
            for i, u in enumerate(pieces):
                text = fastq(u, first)
                first += len(u)
                r = ctx.kmers_add_text(text, fastq=True, is_last=i + 1 == len(pieces), multiple_copies=True)
                assert r["status"] == "ok" and r["consumed"] == len(text) and r["n"] == len(u)
        check_set(ctx, d)


@pytest.mark.parametrize("name", list(BY_NAME))
def test_device_batches(name):
    torch = pytest.importorskip("torch")
    d = BY_NAME[name]
    with api.Context(api.make_params(min_length=1)) as ctx:
        add_assembly(ctx, d)
        for reads in d.files:
            if not reads:
                continue
            hb = api.HostBatch(reads, None, want_seq=True, want_nmask=True)
            t = {k: torch.from_numpy(getattr(hb, k)).cuda() for k in ("off", "len", "seq2b", "nmask")}
            ctx.kmers_add_device(api.device_batch(hb.n, hb.padded_bases, t["off"], t["len"], seq2b=t["seq2b"], nmask=t["nmask"]),
                                 True)
            torch.cuda.synchronize()
        check_set(ctx, d)


def test_multiple_copy_adds_are_refused_after_the_build_state_is_released():
    """the counts of earlier adds are gone after fl_kmers_release_build_state: a 16-mer seen twice before and twice after
    would be missed, so every multiple-copy entry point refuses; assembly adds still go in"""
    torch = pytest.importorskip("torch")
    x = bm.kmer_seq(0x12345678)
    y = bm.kmer_seq(0x0F0F1234)
    with api.Context(api.make_params(min_length=1)) as ctx:
        ctx.kmers_add([x, x], True)
        assert ctx.kmers_count() == 0
        ctx.kmers_release_build_state()
        with pytest.raises(api.FLError, match="after fl_kmers_release_build_state"):
            ctx.kmers_add([x, x], True)
        with pytest.raises(api.FLError, match="after fl_kmers_release_build_state"):
            ctx.kmers_add_text(fastq([x, x]), fastq=True, multiple_copies=True)
        hb = api.HostBatch([x], None, want_seq=True, want_nmask=True)
        t = {k: torch.from_numpy(getattr(hb, k)).cuda() for k in ("off", "len", "seq2b", "nmask")}
        with pytest.raises(api.FLError, match="after fl_kmers_release_build_state"):
            ctx.kmers_add_device(api.device_batch(hb.n, hb.padded_bases, t["off"], t["len"], seq2b=t["seq2b"], nmask=t["nmask"]), True)
        assert ctx.kmers_count() == 0
        ctx.kmers_add([y], False)
        r = ctx.kmers_add_text(b">c\n%s\n" % x, fastq=False)
        assert r["status"] == "ok"
        want = sorted({bm.seq_kmer(y), bm.rc(bm.seq_kmer(y)), bm.seq_kmer(x), bm.rc(bm.seq_kmer(x))})
        assert ctx.kmers_export().tolist() == want
    with api.Context(api.make_params(min_length=1)) as ctx:     # released before any multiple-copy add: nothing is lost
        ctx.kmers_release_build_state()
        ctx.kmers_add([x] * 4, True)
        assert ctx.kmers_export().tolist() == sorted({bm.seq_kmer(x), bm.rc(bm.seq_kmer(x))})


CLI_CASES = {
    "defaults": ({}, False, False),
    "chunks_of_1MiB": ({"FL_CHUNK_MB": "1"}, False, False),
    "host_parser": ({"FL_HOST_PARSER": "1"}, False, False),
    "gzip": ({}, True, False),
    "gzip_chunks_of_1MiB": ({"FL_CHUNK_MB": "1"}, True, False),
    "crlf_record": ({}, False, True),
    "crlf_record_chunks_of_1MiB": ({"FL_CHUNK_MB": "1"}, False, True),
}


@pytest.mark.skipif(not os.path.exists(CLI), reason="CLI not built")
@pytest.mark.parametrize("case", list(CLI_CASES))
def test_cli_against_the_reference(case, tmp_path):
    """the combined designs as -a / -1 / -2 files: the "N reads, M 16-mers" line, and stdout (--min_mean_q 1 keeps the
    long reads whose designed 16-mer is in the set) byte for byte, against the recorded reference CLI"""
    env_extra, gz, crlf = CLI_CASES[case]
    paths = bm.write_combined(str(tmp_path), DESIGNS, gz=gz, crlf=crlf)
    args = bm.cli_args(paths)
    rc_r, out_r, err_r = orc.run_refcli(args)
    env = dict(os.environ, LC_ALL="C", **env_extra)
    env.pop("LANG", None)
    p = subprocess.run([CLI] + args, capture_output=True, env=env)
    err = p.stderr.decode(errors="replace")
    assert p.returncode == rc_r == 0, err[-2000:]
    assert bm.count_line(err) == bm.count_line(err_r)
    assert p.stdout == out_r

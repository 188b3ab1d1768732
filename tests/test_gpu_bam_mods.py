"""BAM output built on the device (fl_bam_build, the CLI's BAM pass 2) and `--keep_mods`: records byte for byte against
tests/bam_mods_model.py with the flag and against bam_util.expected_output without it, and the CLI's output against the
BGZF of the model's stream, member for member."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from filtlong_b200 import api
from tests import bam_mods_model as mm
from tests import bam_util as bu
from tests import util
from tests.test_bam_mods_model import INVALID, random_mm, random_read, results_for

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "filtlong_b200", "bin", "filtlong")


def items_of(raw, res):
    """fl_bam_build items for results over the whole stream (records at their own offsets) and the records"""
    items = [(0, -1, bu.header_end(raw))]
    for r, (n_child, rows) in zip(bu.records(raw), res):
        if n_child == 0:
            if rows[0][2]:
                items.append((r["start"], -1, r["size"]))
            continue
        items += [(r["start"], s, e) for s, e, passed in rows if passed and e - s > 0]
    return items


@pytest.fixture(scope="module")
def ctx():
    with api.Context() as c:
        yield c


@pytest.mark.parametrize("keep_mods", [False, True])
def test_build_equals_the_model(ctx, keep_mods):
    rng = np.random.default_rng(31)
    reads = [random_read(rng, i, lo=1, hi=2500) for i in range(400)]
    reads += [(b"bad_%s" % k.encode(), b"ACGTCCGACGTC", b"\x10" * 12, bu.aux_z(b"RG", b"rg1") + v) for k, v in sorted(INVALID.items())]
    long_seq = util.rand_seq(rng, 40000).upper()
    mmv = b"C+m?" + b"".join(b",%d" % d for d in rng.integers(0, 3, size=2000)) + b";"
    reads.append((b"long", long_seq, None, bu.aux_z(b"RG", b"rg1") + bu.aux_z(b"MM", mmv) + bu.aux_b(b"ML", b"C", [7] * 2000)))
    raw = bu.bam_of(reads)
    res = results_for(rng, reads[:-1])
    L5 = len(reads[5][1])
    res[5] = (2, [(0, L5 // 2, 0), (L5 // 2, L5, 0)])                     # a parent with no kept child
    cuts = list(range(0, 40001, 37)) + [40000]
    res.append((len(cuts) - 1, [(cuts[k], cuts[k + 1], 1) for k in range(len(cuts) - 1)]))   # one read in many children
    for k in range(10, 40):                                               # children of length 1 at odd and even starts
        L = len(reads[k][1])
        res[k] = (2, [(L // 2, L // 2 + 1, 1), (L - 1, L, 1)]) if L > 2 else res[k]
    want, counts = mm.expected_output(raw, res, keep_mods)
    if not keep_mods:
        assert want == bu.expected_output(raw, res)
    got, got_counts = ctx.bam_build(raw, items_of(raw, res), keep_mods)
    assert got == want
    assert got_counts == counts
    assert (counts[0] > 0) == keep_mods


def pack_seq_np(seq):
    codes = np.zeros(256, np.uint8)
    for i, c in enumerate(bu.SEQ_CODES):
        codes[c] = i
    x = codes[np.frombuffer(seq, np.uint8)]
    if x.size % 2:
        x = np.append(x, 0)
    return ((x[0::2] << 4) | x[1::2]).astype(np.uint8).tobytes()


def test_record_larger_than_64_mib(ctx):
    rng = np.random.default_rng(8)
    L = 46_000_001
    seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=L)].tobytes()
    qual = rng.integers(1, 60, size=L).astype(np.uint8).tobytes()
    body = bu.FIXED.pack(-1, -1, 4, 255, 4680, 0, 4, L, -1, -1, 0) + b"big\0" + pack_seq_np(seq) + qual + bu.aux_z(b"RG", b"rg1")
    rec = len(body).to_bytes(4, "little") + body
    assert len(rec) > 64 << 20
    raw = bu.header() + rec
    start = bu.header_end(raw)
    got, _ = ctx.bam_build(raw, [(0, -1, start), (start, 3, 5_000_004), (start, 5_000_004, L)], True)
    kids = bu.records(bu.header() + got[start:])
    assert [k["name"] for k in kids] == [b"big_4-5000004", b"big_5000005-%d" % L]
    assert kids[0]["seq"] == seq[3:5_000_004] and kids[1]["seq"] == seq[5_000_004:]
    assert kids[0]["qual"] == qual[3:5_000_004] and kids[1]["qual"] == qual[5_000_004:]
    assert got[:start] == raw[:start]


# ---- the CLI ----
def run(cmd, env=None):
    e = dict(os.environ, LC_ALL="C")
    e.pop("LANG", None)
    e.update(env or {})
    p = subprocess.run([str(c) for c in cmd], capture_output=True, env=e)
    return p.returncode, p.stdout, p.stderr.decode(errors="replace")


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    if not os.path.exists(CLI):
        pytest.skip("CLI not built")
    d = tmp_path_factory.mktemp("modcli")
    rng = np.random.default_rng(41)
    genome = util.rand_seq(rng, 60000)
    reads = []
    for i, (name, seq, qual) in enumerate(util.long_reads(rng, genome, 400, max_len=12000)):
        seq = seq.upper()
        mmv, ml = random_mm(rng, seq)
        aux = (bu.aux_z(b"RG", b"rg1") if i % 3 else b"") + bu.aux_f(b"qs", 12.5)
        if i % 11 == 4:
            aux += INVALID[sorted(INVALID)[i % len(INVALID)]]
        elif i % 13 != 6:
            aux += bu.aux_z(b"MM", mmv) + bu.aux_b(b"ML", b"C", ml) + (bu.aux_i(b"MN", len(seq)) if i % 2 else b"")
        reads.append((name.encode(), seq, bytes(x - 33 for x in qual), aux))
    raw = bu.bam_of(reads)
    (d / "in.bam").write_bytes(bu.bgzf(raw))
    fa = util.write_fasta(d / "asm.fasta", [("contig_1", genome[:40000]), ("contig_2", genome[40000:])], width=60)
    return dict(dir=d, raw=raw, fa=fa)


def results_from_fastq(raw, fq_out):
    """per input record, (n_child, rows) as bam_util.expected_output takes them, from what the CLI wrote on the file's
    FASTQ equivalent: a read kept whole, or its children by their names name_<s+1>-<e>"""
    recs = bu.records(raw)
    names = {r["name"] for r in recs}
    whole, kids = set(), {}
    for line in fq_out.split(b"\n")[0::4]:
        if not line:
            continue
        n = line[1:]
        if n in names:
            whole.add(n)
            continue
        parent, se = n.rsplit(b"_", 1)
        s, e = (int(x) for x in se.split(b"-"))
        kids.setdefault(parent, []).append((s - 1, e, 1))
    return [(len(kids[r["name"]]), kids[r["name"]]) if r["name"] in kids else (0, [(0, r["len"], int(r["name"] in whole))])
            for r in recs]


CLI_CASES = [["-a", "FA", "--trim", "--split", "16", "-p", "80"], ["--trim_q", "10", "--trim", "--split", "500", "-p", "90"]]


@pytest.mark.parametrize("case", CLI_CASES, ids=lambda c: " ".join(c))
def test_cli_keep_mods(files, case, tmp_path):
    d, raw = files["dir"], files["raw"]
    args = [files["fa"] if a == "FA" else a for a in case]
    (tmp_path / "in.fastq").write_bytes(bu.to_fastq(raw))
    rc, fq_out, _ = run([CLI] + args + ["--failed", tmp_path / "failed.fastq", tmp_path / "in.fastq"])
    assert rc == 0
    res, fres = results_from_fastq(raw, fq_out), results_from_fastq(raw, (tmp_path / "failed.fastq").read_bytes())
    # without the flag: the model of RG-only children, its members cut every 65,280 bytes of the stream
    rc, plain, err_plain = run([CLI] + args + [d / "in.bam"])
    assert rc == 0, err_plain[-2000:]
    assert plain == api.bgzf_compress(bu.expected_output(raw, res))
    assert "modification tags" not in err_plain
    # with it: the re-based tags, on stdout and on --failed, and the log line
    rc, out, err = run([CLI] + args + ["--keep_mods", "--failed", tmp_path / "failed.bam", d / "in.bam"])
    assert rc == 0, err[-2000:]
    want, counts = mm.expected_output(raw, res, True)
    assert out == api.bgzf_compress(want)
    assert counts[0] > 0 and counts[1] > 0
    line = "  modification tags: re-based on %d child reads, dropped from %d whose parent's MM/ML/MN tags are invalid\n" % tuple(counts)
    assert line in err
    assert err.replace(line, "") == err_plain
    fwant, _ = mm.expected_output(raw, fres, True)
    assert (tmp_path / "failed.bam").read_bytes() == api.bgzf_compress(fwant)
    import torch
    if torch.cuda.device_count() >= 2:
        rc, out2, _ = run([CLI] + args + ["--keep_mods", "--gpus", "2", d / "in.bam"], env={"FL_CHUNK_MB": "1"})
        assert rc == 0 and out2 == out


def test_cli_keep_mods_errors(files, tmp_path):
    d = files["dir"]
    rc, out, err = run([CLI, "--keep_mods", "-p", "90", d / "in.bam"])
    assert rc == 1 and out == b"" and "Error: --keep_mods needs --trim or --split" in err
    fq = tmp_path / "r.fastq"
    fq.write_bytes(bu.to_fastq(files["raw"]))
    rc, out, err = run([CLI, "--keep_mods", "--trim_q", "10", "--trim", fq])
    assert rc == 1 and out == b"" and "Error: --keep_mods needs BAM input" in err
    assert "Scoring long reads" not in err


# ---- fl_bam_writer: one stream in several batches ----
def batch_of(raw, items):
    """the bytes of one batch and its items, as the CLI's sink makes them: raw pieces copied, a record copied once for
    its consecutive children"""
    buf, out, last = bytearray(), [], None
    for off, s, e in items:
        if s < 0:
            out.append((len(buf), -1, e))
            buf += raw[off:off + e]
            last = None
            continue
        if off != last:
            size = 4 + int.from_bytes(raw[off:off + 4], "little")
            at = len(buf)
            buf += raw[off:off + size]
            last = off
        out.append((at, s, e))
    return bytes(buf), out


@pytest.mark.parametrize("keep_mods", [False, True])
def test_writer_joins_batches_into_the_members_of_one_stream(ctx, keep_mods):
    rng = np.random.default_rng(53)
    reads = [random_read(rng, i, lo=1, hi=2500) for i in range(700)]
    reads += [(b"bad_%s" % k.encode(), b"ACGTCCGACGTC", b"\x10" * 12, bu.aux_z(b"RG", b"rg1") + v) for k, v in sorted(INVALID.items())]
    raw = bu.bam_of(reads)
    res = results_for(rng, reads)
    want, counts = mm.expected_output(raw, res, keep_mods)
    items = items_of(raw, res)
    recs = {r["start"]: r for r in bu.records(raw)}
    size = [e if s < 0 else len(mm.child_record(raw, recs[o], s, e, keep_mods)[0]) for o, s, e in items]
    assert sum(size) == len(want) > 8 * api.capi.FL_BGZF_BLOCK
    B = api.capi.FL_BGZF_BLOCK
    # split the first whole record that crosses a block boundary there, so that one batch ends exactly on it
    at = 0
    for k, (o, s, e) in enumerate(items):
        if k > 4 and s < 0 and at // B < (at + e) // B and (at + e) % B:
            cut = ((at + e) // B) * B - at
            items[k:k + 1] = [(o, -1, cut), (o + cut, -1, e - cut)]
            exact = k + 1
            break
        at += size[k]
    else:
        pytest.fail("no whole record crosses a block boundary")
    size[exact - 1:exact] = [items[exact - 1][2], items[exact][2]]
    assert sum(size[:exact]) % B == 0
    # a record's children on both sides of a cut
    split = next(k for k in range(exact + 1, len(items) - 1) if items[k][1] >= 0 and items[k + 1][1] >= 0 and items[k][0] == items[k + 1][0])
    cuts = sorted({1, 3, exact, split + 1} | set(range(exact + 7, len(items), 40)))
    bounds = [0] + [c for c in cuts if 0 < c < len(items)] + [len(items)]
    w = api.BamWriter(ctx)
    got, got_counts = b"", [0, 0]
    try:
        for a, b in zip(bounds, bounds[1:]):
            batch, its = batch_of(raw, items[a:b])
            z, c = w.push(batch, its, keep_mods)
            if b in (1, 3):                                              # less than one block so far: nothing out yet
                assert z == b""
            got += z
            got_counts = [x + y for x, y in zip(got_counts, c)]
            done = len(gzip.decompress(got)) if got else 0               # whole blocks only, the rest held back
            assert done % B == 0 and sum(size[:b]) - done < B
            if b == exact:                                               # this batch ends on a block boundary: nothing held
                assert done == sum(size[:b])
        z, c = w.push(b"", [], keep_mods, last=True)                     # the last push compresses what is held
        got += z
        got_counts = [x + y for x, y in zip(got_counts, c)]
    finally:
        w.close()
    assert got == api.bgzf_compress(want, append_eof=False)
    assert got_counts == counts


@pytest.mark.parametrize("bad", ["l_read_name_0", "l_seq_past_block", "child_past_l_seq", "item_past_batch"])
def test_build_refuses_records_that_do_not_fit(ctx, bad):
    good = bu.record(b"r", b"ACGTACGTAC", bytes(range(1, 11)), bu.aux_z(b"RG", b"rg1"))
    rec = {"l_read_name_0": bu.record(b"r", b"ACGTACGTAC", None, l_read_name=0),
           "l_seq_past_block": bu.record(b"r", b"ACGTACGTAC", None, l_seq=4000)}.get(bad, good)
    raw = bu.header() + rec
    at = bu.header_end(raw)
    items = [(at, 2, 11 if bad == "child_past_l_seq" else 8)] if bad != "item_past_batch" else [(at, -1, len(rec) + 1)]
    with pytest.raises(Exception, match="fl_bam_build"):
        ctx.bam_build(raw, items, True)
    assert ctx.bam_build(bu.header() + good, [(at, 2, 8)], True)[0] == bu.child_record(bu.header() + good, bu.records(bu.header() + good)[0], 2, 8)

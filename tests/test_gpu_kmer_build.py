"""The one-copy 16-mer build (`k_kmers_add<false>`, the -a assembly set and the --contam set) on the designed contigs
of tests/kmer_build_design.py, through every packer in front of it, against the model of tests/kmer_build_model.py
bit for bit: the exported set, its count, and for text the records and bases fl_kmers_add_text reports.

Reference set: host batches (fl_kmers_add_batch), FASTQ text, FASTA text through the wrapped-FASTA index (one line per
record, and wrapped at 1 .. 1000 bases a line) and through the two-line index (FL_FASTA_TWO_LINE=1), device batches of
2-bit codes + non-ACGT mask and of ASCII. Contaminant set: host batches and FASTQ / wrapped FASTA text. Each in one
batch and in record-aligned chunks cut just before and just after the long contigs. The device batches carry junk in
their padding (every byte class, ACGT included), which no 16-mer may read.

No text path declines any byte class of the design (every add below must return "ok"). The FASTQ and two-line FASTA
indexes decline a record with an empty sequence (kseq reads it, their slices cannot): their files leave those out.

Every context holds 2.5 GiB of tables: each test opens one at a time and closes it."""
import functools

import numpy as np
import pytest

from filtlong_b200 import api
from tests import kmer_build_design as kd
from tests import kmer_build_model as kbm

pytestmark = pytest.mark.gpu

REF_PATHS = ["host", "fastq", "fasta", "fasta_two_line"] + ["wrapped_%d" % w for w in kd.WIDTHS] + ["device_2bit", "device_ascii"]
CONTAM_PATHS = ["contam_host", "contam_fastq", "contam_wrapped_60"]
JUNK = np.frombuffer(kd.OTHER_BYTES + b"ACGTacgt", dtype=np.uint8)


def contigs_of(path):
    """the contigs a path adds: the design, with the line-end contigs of its width for wrapped FASTA, and without the
    empty sequences for the indexes that decline them"""
    if path.startswith(("wrapped_", "contam_wrapped_")):
        return kd.design().contigs + kd.wrapped_extra(int(path.rsplit("_", 1)[1]))[0]
    if path in ("fastq", "fasta_two_line", "contam_fastq"):
        return [s for s in kd.design().contigs if s]
    return kd.design().contigs


@functools.lru_cache(maxsize=None)
def _base_model(drop_empty):
    return kbm.build([s for s in kd.design().contigs if s] if drop_empty else kd.design().contigs)


@functools.lru_cache(maxsize=None)
def model(path):
    """(members, records, bases) of what `path` adds, the design's part computed once"""
    if path.startswith(("wrapped_", "contam_wrapped_")):
        members, n, bases = _base_model(False)
        em, en, eb = kbm.build(kd.wrapped_extra(int(path.rsplit("_", 1)[1]))[0])
        return np.union1d(members, em), n + en, bases + eb
    return _base_model(path in ("fastq", "fasta_two_line", "contam_fastq"))


def junk_padding(hb, rng):
    """junk codes and non-ACGT bits on every padding base of a packed host batch"""
    pad = np.zeros(hb.padded_bases, dtype=bool)
    for o, L in zip(hb.off, hb.len):
        pad[int(o) + int(L):int(o) + int(kd.padded(int(L)))] = True
    codes = np.where(pad, rng.integers(0, 4, size=hb.padded_bases), 0).astype(np.uint32)
    other = (pad & (rng.random(hb.padded_bases) < 0.5)).astype(np.uint32)
    hb.seq2b |= (codes.reshape(-1, 16) << np.arange(30, -1, -2, dtype=np.uint32)).sum(axis=1, dtype=np.uint32)
    hb.nmask |= (other.reshape(-1, 32) << np.arange(32, dtype=np.uint32)).sum(axis=1, dtype=np.uint32)


def add_device(ctx, torch, seqs, rng, ascii):
    hb = api.HostBatch(seqs, None, want_seq=not ascii, want_nmask=not ascii)
    t = {k: torch.from_numpy(getattr(hb, k)).cuda() for k in ("off", "len")}
    if ascii:
        arena = JUNK[rng.integers(0, len(JUNK), size=max(hb.padded_bases, 64))]
        for o, s in zip(hb.off, seqs):
            arena[int(o):int(o) + len(s)] = np.frombuffer(s, dtype=np.uint8)
        t["ascii"] = torch.from_numpy(arena).cuda()
    else:
        junk_padding(hb, rng)
        t["seq2b"], t["nmask"] = torch.from_numpy(hb.seq2b).cuda(), torch.from_numpy(hb.nmask).cuda()
    ctx.kmers_add_device(api.device_batch(hb.n, hb.padded_bases, t["off"], t["len"], seq2b=t.get("seq2b"), nmask=t.get("nmask"),
                                          ascii=t.get("ascii")), False)
    torch.cuda.synchronize()


def add(ctx, path, pieces):
    """adds the pieces through `path`; (records, bases) the text entry points report (None for batches)"""
    torch = pytest.importorskip("torch") if path.startswith("device_") else None
    rng = np.random.default_rng(5)
    n = bases = 0
    first = 0
    for i, seqs in enumerate(pieces):
        last = i + 1 == len(pieces)
        text = fastq = None
        if path in ("host", "contam_host"):
            (ctx.kmers_add(seqs, False) if path == "host" else ctx.contam_add(seqs))
        elif path.startswith("device_"):
            add_device(ctx, torch, seqs, rng, path == "device_ascii")
        elif path in ("fastq", "contam_fastq"):
            text, fastq = kd.fastq(seqs, first), True
        elif path in ("fasta", "fasta_two_line"):
            text, fastq = kd.fasta(seqs, None, first), False
        else:
            text, fastq = kd.fasta(seqs, int(path.rsplit("_", 1)[1]), first), False
        first += len(seqs)
        if text is None:
            continue
        r = (ctx.contam_add_text if path.startswith("contam_") else ctx.kmers_add_text)(text, fastq=fastq, is_last=last)
        assert r["status"] == "ok" and r["consumed"] == len(text) and r["n"] == len(seqs), (path, i, r)
        n += r["n"]
        bases += r["bases"]
    return (n, bases) if path not in ("host", "contam_host") and not path.startswith("device_") else None


def open_ctx(path, monkeypatch):
    if path == "fasta_two_line":
        monkeypatch.setenv("FL_FASTA_TWO_LINE", "1")            # read when the context is created
    ctx = api.Context(api.make_params())
    monkeypatch.delenv("FL_FASTA_TWO_LINE", raising=False)
    return ctx


def substitutions(members, rng, n=2000):
    """every single-base substitution of a sample of the members"""
    m = members[rng.choice(len(members), size=min(n, len(members)), replace=False)].astype(np.uint32)
    out = [m ^ (np.uint32(x) << np.uint32(2 * i)) for i in range(16) for x in (1, 2, 3)]
    return np.concatenate(out)


@pytest.mark.parametrize("chunked", [False, True], ids=["one_batch", "chunks"])
@pytest.mark.parametrize("path", REF_PATHS)
def test_reference_set(path, chunked, monkeypatch):
    seqs = contigs_of(path)
    members, n, bases = model(path)
    pieces = kd.chunks(seqs, kd.design().cuts) if chunked else [seqs]
    with open_ctx(path, monkeypatch) as ctx:
        reported = add(ctx, path, pieces)
        if reported is not None:
            assert reported == (n, bases)
        assert ctx.kmers_count() == len(members)
        assert np.array_equal(ctx.kmers_export(), members)
        assert ctx.kmers_contains(members).all()
        q = substitutions(members, np.random.default_rng(len(path)))
        assert np.array_equal(ctx.kmers_contains(q), np.isin(q, members))
        assert ctx.contam_count() == 0


@pytest.mark.parametrize("chunked", [False, True], ids=["one_batch", "chunks"])
@pytest.mark.parametrize("path", CONTAM_PATHS)
def test_contaminant_set(path, chunked, monkeypatch):
    seqs = contigs_of(path)
    members, n, bases = model(path)
    pieces = kd.chunks(seqs, kd.design().cuts) if chunked else [seqs]
    with open_ctx(path, monkeypatch) as ctx:
        reported = add(ctx, path, pieces)
        if reported is not None:
            assert reported == (n, bases)
        assert ctx.contam_count() == len(members)
        assert np.array_equal(ctx.contam_export(), members)
        assert ctx.kmers_count() == 0


@pytest.mark.parametrize("path", ["fastq", "fasta_two_line"])
def test_an_empty_sequence_is_declined_by_the_slicing_indexes(path, monkeypatch):
    """a record with an empty sequence: the FASTQ and two-line FASTA indexes add nothing and hand the chunk back (the
    CLI then reads it on the host); the wrapped-FASTA index takes it"""
    seqs = [s for s in kd.design().contigs[:200] if s][:20]
    seqs.insert(10, b"")
    with open_ctx(path, monkeypatch) as ctx:
        text = kd.fastq(seqs) if path == "fastq" else kd.fasta(seqs)
        r = ctx.kmers_add_text(text, fastq=path == "fastq", is_last=True)
        assert r["status"] == "fallback" and r["n"] == 0
        assert ctx.kmers_count() == 0
    with open_ctx("fasta", monkeypatch) as ctx:
        r = ctx.kmers_add_text(kd.fasta(seqs), fastq=False, is_last=True)
        assert r["status"] == "ok" and r["n"] == len(seqs)
        assert np.array_equal(ctx.kmers_export(), kbm.build(seqs)[0])

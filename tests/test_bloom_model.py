"""The short-read build's two models (tests/bloom_model.py) against each other, against the C restatement of the
reference (oracle/filtlong_oracle.c) and against recorded runs of the unmodified reference, on random streams and on
inputs designed to reach each path of the Bloom false-positive rule. No GPU."""
import hashlib

import numpy as np
import pytest

from oracle import oracle as orc
from tests import bloom_model as bm

DESIGNS = bm.designs()
BY_NAME = {d.name: d for d in DESIGNS}


def test_hash_and_its_inverse_against_the_c_restatement():
    L = orc.lib()
    assert L.orc_bloom_table_bits() == bm.TABLE_BITS
    rng = np.random.default_rng(1)
    keys = rng.integers(0, 1 << 32, size=200, dtype=np.uint64).astype(np.uint32)
    np_bits = bm.bloom_bits_np(keys)
    for i, k in enumerate(keys.tolist()):
        assert [L.orc_bloom_hash(k, j) % bm.TABLE_BITS for j in range(13)] == bm.bloom_bits(k) == np_bits[i].tolist()
    for b, j in zip(rng.integers(0, bm.TABLE_BITS, size=200).tolist(), rng.integers(0, 13, size=200).tolist()):
        for wrap in (0, 1, 2):
            c = bm.cover(b, j, wrap)
            if c is not None:
                assert L.orc_bloom_hash(c, j) == b + wrap * bm.TABLE_BITS


def test_add_stream_encoding():
    """forward A0 C1 G2 T3 (any case, anything else 0) with the first base on top; the reverse 16-mer with the newest
    base on top and anything but ACGT as 0; reads under 16 bases add nothing"""
    L = orc.lib()
    for c in range(256):
        assert bm.FWD.get(c, 0) == L.orc_base_fwd(bytes([c]))
        assert bm.REV.get(c, 0) << 30 == L.orc_base_rev(bytes([c]))
    rng = np.random.default_rng(2)
    seq = bytes(rng.choice(np.frombuffer(b"ACGTacgt", np.uint8), size=40))
    adds = bm.read_adds(seq)
    assert len(adds) == 25
    for p, (f, r) in enumerate(adds):
        assert f == bm.seq_kmer(seq[p:p + 16]) and r == bm.rc(f)
    n = bytearray(seq); n[20] = ord("N")
    for p, (f, r) in enumerate(bm.read_adds(bytes(n))):
        if p <= 20 < p + 16:          # N: A on the forward strand, 0 (not T's complement) on the reverse one
            assert f == bm.seq_kmer(seq[p:20] + b"A" + seq[21:p + 16])
            assert r == bm.rc(f) & ~(3 << (2 * (20 - p)))
    assert bm.add_stream([[b"ACGT" * 3, b"A" * 15], [b"C" * 16]]) == [bm.seq_kmer(b"C" * 16), bm.seq_kmer(b"G" * 16)]


@pytest.mark.parametrize("seed", range(6))
def test_models_agree_on_random_streams_with_a_small_table(seed):
    """a 4,096-bit table: false positives on first sightings are everywhere, so both clauses and both outcomes of
    cnt == 3 are reached many times; `members` (an assembly's 16-mers) are skipped by both"""
    rng = np.random.default_rng(seed)
    pool = rng.integers(0, 1 << 32, size=400, dtype=np.uint64).tolist()
    stream = [pool[i] for i in rng.integers(0, len(pool), size=1500)]
    members = set(pool[:15])
    trace, detail = {}, {}
    seq = bm.sequential_set(stream, members, table_bits=4096, trace=trace)
    cf = bm.closed_form_set(stream, members, table_bits=4096, detail=detail)
    assert seq == cf
    assert {x: v[2] for x, v in detail.items()} == trace          # FP on the first sighting: the same 16-mers
    three = [(x in cf, v[2]) for x, v in detail.items() if v[0] == 3]
    assert (True, True) in three and (False, False) in three
    assert any(v[0] == 2 and v[2] for v in detail.values())       # FP but only two sightings: out
    real = {}
    bm.closed_form_set(stream, members, detail=real)
    assert not any(v[2] for v in real.values())                   # the same stream with the real table: no FP at all


def _check_design(files, assembly, expect):
    stream = bm.add_stream(files)
    members = bm.assembly_set(assembly)
    trace, detail = {}, {}
    seq = bm.sequential_set(stream, members, trace=trace)
    cf = bm.closed_form_set(stream, members, detail=detail)
    assert seq == cf
    assert {x: v[2] for x, v in detail.items()} == trace
    for label, (k, member, path) in expect.items():
        assert (k in cf) == member, label
        if path is not None:
            cnt, covered = path
            assert detail[k][0] == cnt and detail[k][3] == covered, (label, detail[k])
    return cf


@pytest.mark.parametrize("name", list(BY_NAME))
def test_design_reaches_its_path(name):
    """both models give the same set; every named 16-mer has its membership, its sightings and its count of Bloom
    bits set before its first sighting -- e.g. a 16-mer seen three times is in only with all 13"""
    d = BY_NAME[name]
    _check_design(d.files, d.assembly, d.expect)


def test_designs_keep_their_paths_in_one_input():
    files, asm = bm.combined(DESIGNS)
    _check_design(files, asm, {"%s:%s" % (d.name, k): v for d in DESIGNS for k, v in d.expect.items()})


def test_designed_16mers():
    for x, j, jj in bm.SELF_COVER:
        assert x != bm.rc(x) and bm.bloom_bits(x)[j] == bm.bloom_bits(bm.rc(x))[jj]
    for x, c, j in bm.NEIGHBOUR_COVER:
        read = b"ACGT"[c:c + 1] + bm.kmer_seq(x)
        (f0, r0), (f1, _) = bm.read_adds(read)
        assert f1 == x and r0 != x and bm.bloom_bits(x)[j] in bm.bloom_bits(r0)
    d = BY_NAME["n_mask_cover"]
    w = d.files[0][12]
    assert b"N" in w and bm.read_adds(w)[0][1] == d.n_cover and bm.rc(bm.read_adds(w)[0][0]) != d.n_cover
    assert all(bm.rc(k) == k for k, _, _ in BY_NAME["palindromes"].expect.values())
    runs, run = [], 0                                             # FASTQ bytes of the filler runs (>= 10 per record + bases)
    for seq in BY_NAME["chunk_seams"].files[0]:
        if len(seq) < 16:
            run += 10 + 2 * len(seq)
        elif run:
            runs, run = runs + [run], 0
    assert len(runs) == 2 and min(runs) > 1 << 20


@pytest.mark.parametrize("name", list(BY_NAME))
def test_c_restatement_builds_the_models_set(name):
    d = BY_NAME[name]
    ok = orc.Kmers()
    ok.add_assembly(d.assembly)
    for f in d.files:
        ok.add_short_reads(f)
    assert ok.dump().tolist() == sorted(bm.model_set(d.files, d.assembly))


def _sha(kmers):
    return hashlib.sha256(np.array(sorted(kmers), dtype="<u4").tobytes()).hexdigest()


@pytest.mark.parametrize("with_assembly", [True, False])
def test_recorded_reference_builds_the_models_set(with_assembly, tmp_path):
    """the unmodified reference's link harness (its runs replayed from tests/golden) on the combined designs: the set's
    size and the SHA-256 of its sorted members"""
    paths = bm.write_combined(str(tmp_path), DESIGNS)
    files, asm = bm.combined(DESIGNS)
    want = bm.model_set(files, asm if with_assembly else [])
    ref = orc.run_refdump(bm.cli_args(paths, with_assembly), kmers_out=True)
    assert ref["n_kmers"] == len(want)
    assert ref["kmers_sha256"] == _sha(want)


@pytest.mark.parametrize("gz,crlf", [(False, False), (True, False), (False, True)])
def test_recorded_reference_cli_counts_the_models_set(gz, crlf, tmp_path):
    """the reference CLI's "N reads, M 16-mers" line on the combined files (the line the GPU tests hold the CLI to)"""
    paths = bm.write_combined(str(tmp_path), DESIGNS, gz=gz, crlf=crlf)
    files, asm = bm.combined(DESIGNS)
    rc, out, err = orc.run_refcli(bm.cli_args(paths))
    assert rc == 0
    n_reads = len(files[0]) + len(files[1])
    assert bm.count_line(err) == "%d reads, %d 16-mers" % (n_reads, len(bm.model_set(files, asm)))   # C locale: no separators
    # --min_mean_q 1 keeps the long reads whose designed 16-mer is in the set
    assert orc.fastq_names(out) == ["%s:%s" % (d.name, label) for d in DESIGNS for label, (_, member, _) in d.expect.items() if member]

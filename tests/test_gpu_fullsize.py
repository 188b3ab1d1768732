"""GPU tests at BASELINE.json's FULL sizes (config 2: 20 Gbases Phred, config 3: 20 Gbases vs a
10 Mbp assembly), where the oracle cannot follow. Parity is carried by size-independent properties:

* two independent exact implementations of the same scores must agree bit-for-bit on every one of
  the 2 M reads (Phred: lattice warp kernels vs one-thread-per-chain work items; k-mer: the position-anchored
  table with and without the L2 pre-filter, and the plain bitmap);
* results must not depend on how the read set is cut into batches;
* the first few thousand reads, regenerated on the host with the same counter-based generator,
  must match the oracle bit-for-bit;
* the selection must satisfy the reference's prefix-walk invariants (main.cpp:251-257): every kept
  row scores at least as high as every passed row that was dropped, kept bases reach the target and
  would not reach it without the lowest-scoring kept row;
* the rescaling and the selection must be exactly the restatement of tests/select_model.py, fed with
  the device's own statistics and scores (parity.check_rescale_exact / check_selection_exact).
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests import parity

pytestmark = pytest.mark.gpu

SAMPLE = 3000


def _env(**kw):
    class E:
        def __enter__(self):
            self.old = {k: os.environ.get(k) for k in kw}
            os.environ.update({k: str(v) for k, v in kw.items()})

        def __exit__(self, *a):
            for k, v in self.old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    return E()


def _selection_invariants(rows, summ, target):
    passed = rows["passed"].astype(bool)
    kept = rows["passed_final"].astype(bool)
    length = (rows["end"] - rows["start"]).astype(np.int64)
    assert not np.any(kept & ~passed)                      # a failed read never comes back (main.cpp:251)
    assert summ.status == 3
    kept_bases = int(length[kept].sum())
    assert kept_bases == summ.keeping
    assert kept_bases >= target                            # the crossing read is kept (main.cpp:252-254)
    fs = rows["final_score"]
    lo_kept = fs[kept].min()
    dropped = passed & ~kept
    assert fs[dropped].max() <= lo_kept                    # descending-score prefix
    # without the rows at the lowest kept score the target is not reached (bases_so_far < target there)
    assert kept_bases - int(length[kept & (fs == lo_kept)].sum()) < target


def _phred_setup(torch, bench, api, capi, dev):
    w = bench.phred_workload(0, 2000000, 20 * 10 ** 9)
    t_len = torch.from_numpy(w["len"]).to(dev)
    t_off = torch.from_numpy(w["off"].view(np.int64)).to(dev)
    t_qbar = torch.from_numpy(w["qbar"]).to(dev)
    d_qual = torch.empty(w["padded"] + 64, dtype=torch.uint8, device=dev)
    return w, t_len, t_off, t_qbar, d_qual


def test_config2_phred_full_size():
    import torch
    import bench
    from filtlong_b200 import api, capi, sharding
    from oracle import oracle as orc

    dev = torch.device("cuda", 0)
    L = capi.lib()
    w, t_len, t_off, t_qbar, d_qual = _phred_setup(torch, bench, api, capi, dev)
    target = 5 * 10 ** 9
    params = api.make_params(target_bases=target)
    results = {}
    for tag, mode, nbatch in (("lattice", 1, 1), ("items", 0, 1), ("lattice_batched", 1, 5)):
        with _env(FL_PHRED_MODE=mode):
            ctx = api.Context(params)
        if tag == "lattice":
            capi.check(ctx.h, L.fl_synth_qual_device(ctx.h, w["seed"], w["n"], t_off.data_ptr(), t_len.data_ptr(),
                                                     t_qbar.data_ptr(), w["read_base"], d_qual.data_ptr()), "synth_qual")
            ctx.sync()
        keep = []
        for lo, hi in sharding.shard_by_bases(w["len"], nbatch):
            base = int(w["off"][lo])
            end = int(w["off"][hi]) if hi < w["n"] else w["padded"]
            rel = torch.from_numpy((w["off"][lo:hi] - np.uint64(base)).view(np.int64)).to(dev)
            keep.append(rel)
            b = api.device_batch(hi - lo, end - base, rel, t_len[lo:hi], qual=d_qual[base:])
            ctx.push_device(b)
        summ = ctx.finalize(w["bases"])
        results[tag] = (ctx.read_results(), ctx.row_results(), summ)
        ctx.close()
    rr, rows, summ = results["lattice"]
    assert len(rr["mean_q"]) == w["n"]
    for other in ("items", "lattice_batched"):
        r2, rows2, s2 = results[other]
        for k in ("mean_q", "window_q"):
            assert np.array_equal(rr[k].view(np.uint64), r2[k].view(np.uint64)), (other, k)
        assert np.array_equal(rr["passed"], r2["passed"])
        assert np.array_equal(rows["final_score"].view(np.uint64), rows2["final_score"].view(np.uint64)), other
        assert np.array_equal(rows["passed_final"], rows2["passed_final"]), other
        assert (s2.status, s2.target, s2.keeping) == (summ.status, summ.target, summ.keeping)
    _selection_invariants(rows, summ, target)
    parity.check_rescale_exact(rows, summ, params)
    parity.check_selection_exact(rows, summ, params)
    # the first reads AND the 50 longest ones (the 1 Mbase reads, where the lattice sum crosses the most
    # binades) against the oracle, regenerated on the host one read at a time (the generator is keyed by
    # the read's global index)
    idx = np.concatenate([np.arange(SAMPLE), np.argsort(-w["len"].astype(np.int64), kind="stable")[:50]])
    assert int(w["len"][idx].max()) == 1000000
    reads = []
    for i in idx:
        n = np.array([w["len"][i]], dtype=np.int32)
        q = np.zeros(int(n[0]) + 64, dtype=np.uint8)
        L.fl_synth_qual_host(w["seed"], 1, capi.ptr(np.zeros(1, dtype=np.uint64)), capi.ptr(n), capi.ptr(w["qbar"][i:i + 1].copy()),
                             w["read_base"] + int(i), capi.ptr(q))
        reads.append((b"A" * int(n[0]), q[:int(n[0])].tobytes()))
    sc = orc.score(reads, orc.make_params(target_bases=target), None)
    parity.check_reads_vs_oracle({k: v[idx] for k, v in rr.items()}, sc)


def _to_dev(torch, dev, x):
    x = x.view(np.int64) if x.dtype == np.uint64 else (x.view(np.int32) if x.dtype == np.uint32 else x)
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _synth_reads(torch, dev, ctx, w, d_genome):
    from filtlong_b200 import capi
    t_len, t_off = _to_dev(torch, dev, w["len"]), _to_dev(torch, dev, w["off"])
    keep = [_to_dev(torch, dev, w[k]) for k in ("start", "strand", "err", "junk_pos", "junk_len", "adap5", "adap3")]
    d_seq = torch.zeros(w["padded"] // 16 + 8, dtype=torch.int32, device=dev)
    desc = capi.SynthReads()
    desc.n, desc.flags, desc.genome_bases = w["n"], w["flags"], w["genome_bases"]
    desc.off, desc.len = t_off.data_ptr(), t_len.data_ptr()
    desc.start, desc.strand, desc.err_ppm, desc.junk_pos, desc.junk_len, desc.adap5, desc.adap3 = [t.data_ptr() for t in keep]
    capi.check(ctx.h, capi.lib().fl_synth_reads_device(ctx.h, w["seed"], d_genome.data_ptr(), C.byref(desc), w["read_base"],
                                                       d_seq.data_ptr()), "synth_reads")
    ctx.sync()
    return t_off, t_len, d_seq


def _host_reads(w, idx, genome_arena):
    """Reads idx of workload w as ASCII, from the HOST generator (one read at a time: keyed by global index)."""
    from filtlong_b200 import capi
    S = capi.synth_host_lib()
    out = []
    for i in idx:
        i = int(i)
        lens = np.array([w["len"][i]], dtype=np.int32)
        off = np.zeros(1, dtype=np.uint64)
        padded = (int(lens[0]) + 63) & ~63
        d = capi.SynthReads()
        arrs = [np.ascontiguousarray(w[k][i:i + 1]) for k in ("start", "strand", "err", "junk_pos", "junk_len", "adap5", "adap3")]
        d.n, d.flags, d.genome_bases = 1, w["flags"], w["genome_bases"]
        d.off, d.len = capi.ptr(off), capi.ptr(lens)
        d.start, d.strand, d.err_ppm, d.junk_pos, d.junk_len, d.adap5, d.adap3 = [capi.ptr(a) for a in arrs]
        arena = np.zeros(padded // 16 + 8, dtype=np.uint32)
        S.fl_synth_reads_host(w["seed"], capi.ptr(genome_arena), C.byref(d), w["read_base"] + i, capi.ptr(arena))
        txt = np.zeros(padded + 64, dtype=np.uint8)
        S.fl_synth_ascii_host(1, capi.ptr(off), capi.ptr(lens), capi.ptr(arena), None, capi.ptr(txt))
        out.append((txt[:int(lens[0])].tobytes(), None))
    return out


def test_config3_kmer_full_size():
    """BASELINE config 3 as written: the 16-mer set is hashed from 10 M synthetic 2 x 150 bp reads with the
    >= 4-copy rule (-1/-2), then 20 Gbases of ONT reads are scored against it (+ --trim --split 500, config 4)."""
    import torch
    import bench
    from filtlong_b200 import api, capi
    from oracle import oracle as orc

    dev = torch.device("cuda", 0)
    L = capi.lib()
    gb = 10 ** 7
    w = bench.kmer_workload(0, 2000000, 20 * 10 ** 9, 1, gb, 0.03, 0.15, seed=3)
    iw = bench.illumina_workload(gb, 5 * 10 ** 6)
    target = 5 * 10 ** 9
    params = api.make_params(target_bases=target, keep_percent=90.0, trim=True, split=500)
    d_genome = torch.zeros(gb // 16 + 8, dtype=torch.int32, device=dev)
    results = {}
    exported = None
    for tag, filt, anch in (("filter", 1, 1), ("direct", 0, 1), ("bitmap", 1, 0)):
        with _env(FL_FILTER=filt, FL_ANCHOR=anch):
            ctx = api.Context(params)
        if tag == "filter":
            capi.check(ctx.h, L.fl_synth_genome_device(ctx.h, 2, gb, d_genome.data_ptr()), "synth_genome")
            t_off, t_len, d_seq = _synth_reads(torch, dev, ctx, w, d_genome)
            s_off, s_len, d_sr = _synth_reads(torch, dev, ctx, iw, d_genome)
            ctx.kmers_add_device(api.device_batch(iw["n"], iw["padded"], s_off, s_len, seq2b=d_sr), True)   # kmers.cpp:50-58,142-166
            n_kmers = ctx.kmers_count()
            ctx.kmers_release_build_state()
            del d_sr
            torch.cuda.empty_cache()
            exported = ctx.kmers_export()
            bm_ptr, bm_bytes = ctx.kmers_bitmap_dev()
            bitmap = torch.empty(bm_bytes, dtype=torch.uint8, device=dev)
            # device-to-device copy of the finished bitmap through torch's CUDA array interface
            class _Raw:
                __cuda_array_interface__ = {"shape": (bm_bytes,), "typestr": "|u1", "data": (bm_ptr, False), "version": 2}
            bitmap.copy_(torch.as_tensor(_Raw(), device=dev))
        else:
            # same set for the other probe layouts: hand the finished bitmap over (what a sharded run does)
            p2, nb2 = ctx.kmers_bitmap_dev()

            class _Raw2:
                __cuda_array_interface__ = {"shape": (nb2,), "typestr": "|u1", "data": (p2, False), "version": 2}
            torch.as_tensor(_Raw2(), device=dev).copy_(bitmap)
            torch.cuda.synchronize()
            ctx.kmers_bitmap_changed()
            n_kmers = ctx.kmers_count()
        ctx.push_device(api.device_batch(w["n"], w["padded"], t_off, t_len, seq2b=d_seq))
        summ = ctx.finalize(w["bases"])
        results[tag] = (ctx.read_results(), ctx.row_results(), summ, n_kmers)
        ctx.close()
    rr, rows, summ, n_kmers = results["filter"]
    # the set: every 16-mer of the genome with >= 4 sightings among 150x reads -- nearly all of the genome's
    # distinct 16-mers, and (0.2 % substitutions, 4 copies needed) next to nothing else
    S = capi.synth_host_lib()
    g = np.zeros(gb // 16 + 8, dtype=np.uint32)
    S.fl_synth_genome_host(2, gb, capi.ptr(g))
    gw = g[:gb // 16].astype(np.uint64)
    both = (gw[:-1] << np.uint64(32)) | gw[1:]
    fw = np.concatenate([((both >> np.uint64(32 - 2 * k)) & np.uint64(0xFFFFFFFF)).astype(np.uint32) for k in range(16)])
    x = ~fw                                                    # reverse complement: complement, then reverse the 2-bit fields
    x = ((x >> 2) & 0x33333333) | ((x & 0x33333333) << 2)
    x = ((x >> 4) & 0x0F0F0F0F) | ((x & 0x0F0F0F0F) << 4)
    rc = x.byteswap()
    genome_set = np.unique(np.concatenate([fw, rc]))
    assert len(exported) == n_kmers
    inter = np.intersect1d(exported, genome_set, assume_unique=True).size
    assert inter >= 0.99 * genome_set.size, (inter, genome_set.size)
    assert n_kmers - inter <= 2e-3 * n_kmers, (n_kmers, inter)      # the same substitution seen in >= 4 of ~150 covering reads: rare, not absent
    for other in ("direct", "bitmap"):
        r2, rows2, s2, n2 = results[other]
        assert n_kmers == n2
        for k in ("mean_q", "window_q"):
            assert np.array_equal(rr[k].view(np.uint64), r2[k].view(np.uint64)), (other, k)
        for k in ("first_base_in_kmer", "last_base_in_kmer", "n_bad", "n_child", "passed"):
            assert np.array_equal(rr[k], r2[k]), (other, k)
        for k in ("start", "end", "passed_final"):
            assert np.array_equal(rows[k], rows2[k]), (other, k)
        assert (s2.status, s2.target, s2.keeping) == (summ.status, summ.target, summ.keeping)
    # children tile their parent without overlap, in coordinate order (read.cpp:119-130)
    assert np.all(rows["end"] >= rows["start"])
    same_parent = rows["parent"][1:] == rows["parent"][:-1]
    assert np.all(rows["start"][1:][same_parent] >= rows["end"][:-1][same_parent])
    assert int((rows["end"] - rows["start"]).astype(np.int64).sum()) == summ.rows_bases
    _selection_invariants(rows, summ, summ.target)
    parity.check_rescale_exact(rows, summ, params)
    parity.check_selection_exact(rows, summ, params)
    # the first reads and the 50 longest against the oracle (host-regenerated reads; the oracle's Kmers is
    # loaded with the exported set: the CPU cannot hash 10 M short reads inside a test)
    idx = np.concatenate([np.arange(400), np.argsort(-w["len"].astype(np.int64), kind="stable")[:50]])
    reads = _host_reads(w, idx, g)
    ok = orc.Kmers()
    ok.insert(exported)
    assert len(ok) == n_kmers
    sc = orc.score(reads, orc.make_params(target_bases=target, keep_percent=90.0, trim=True, split=500), ok)
    parity.check_reads_vs_oracle({k: v[idx] for k, v in rr.items()}, sc)
    # ... and their child ranges / per-child statistics
    for j, i in enumerate(idx):
        row = int(rr["row_start"][i])
        p, kids = sc.parents[j], sc.children[j]
        for r in (kids if kids else [p]):
            assert (rows["start"][row], rows["end"][row]) == (r.start, r.end), (i, row)
            assert rows["mean_q"][row] == r.mean_q and rows["window_q"][row] == r.window_q, (i, row)
            row += 1


def test_sharded_kmer_run_equals_single_context_run():
    """Config 5's shape at test size: the read set cut into two contiguous shards on two contexts (both on
    GPU 0, driven through the split-phase protocol), the 16-mer set built from an assembly with runs of N on
    one context and handed to the others as a bitmap: must select exactly what one context selects."""
    import torch
    import bench
    from filtlong_b200 import api, capi, sharding
    from oracle import oracle as orc

    dev = torch.device("cuda", 0)
    L = capi.lib()
    nc, cb = 8, 500000
    w = bench.kmer_workload(0, 20000, 2 * 10 ** 8, nc, cb, 0.01, 0.12, seed=4)
    target = 5 * 10 ** 7
    kw = dict(target_bases=target, trim=True, split=300)
    params = api.make_params(**kw)
    one = api.Context(params)
    pc = (cb + 63) & ~63
    d_asm = torch.zeros(nc * pc // 16 + 8, dtype=torch.int32, device=dev)
    d_nm = torch.zeros(nc * pc // 32 + 8, dtype=torch.int32, device=dev)
    capi.check(one.h, L.fl_synth_assembly_device(one.h, 4, nc, cb, 20000, d_asm.data_ptr(), d_nm.data_ptr()), "synth_assembly")
    a_off = _to_dev(torch, dev, np.arange(nc, dtype=np.uint64) * np.uint64(pc))
    a_len = _to_dev(torch, dev, np.full(nc, cb, dtype=np.int32))
    one.kmers_add_device(api.device_batch(nc, nc * pc, a_off, a_len, seq2b=d_asm, nmask=d_nm), False)
    n_k = one.kmers_count()
    t_off, t_len, d_seq = _synth_reads(torch, dev, one, w, d_asm)
    one.push_device(api.device_batch(w["n"], w["padded"], t_off, t_len, seq2b=d_seq))
    s1 = one.finalize(-1)
    rows1 = one.row_results()
    # two shards, two contexts; the second gets the finished bitmap
    ctxs = [api.Context(params), api.Context(params)]
    p0, nb = one.kmers_bitmap_dev()

    class _Src:
        __cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (p0, False), "version": 2}
    for c in ctxs:
        pd, _ = c.kmers_bitmap_dev()

        class _Dst:
            __cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (pd, False), "version": 2}
        torch.as_tensor(_Dst(), device=dev).copy_(torch.as_tensor(_Src(), device=dev))
        torch.cuda.synchronize()
        c.kmers_bitmap_changed()
        assert c.kmers_count() == n_k
    cuts = sharding.shard_by_bases(w["len"], 2)
    keep = []
    for c, (lo, hi) in zip(ctxs, cuts):
        base = int(w["off"][lo])
        end = int(w["off"][hi]) if hi < w["n"] else w["padded"]
        rel = _to_dev(torch, dev, w["off"][lo:hi] - np.uint64(base))
        keep.append(rel)
        c.push_device(api.device_batch(hi - lo, end - base, rel, t_len[lo:hi], seq2b=d_seq[base // 16:]))
    # the split-phase protocol with the all-reduces done by hand on the device buffers: the transport-agnostic
    # form of what fl_finalize does over NCCL (that path is exercised on >= 2 GPUs by test_nccl_two_ranks)
    from tests import util
    summaries = util.split_phase_finalize(ctxs, w["bases"])
    rows2 = [c.row_results() for c in ctxs]
    cat = {k: np.concatenate([r[k] for r in rows2]) for k in ("start", "end", "passed_final", "mean_q", "window_q", "final_score")}
    for k in ("start", "end", "passed_final"):
        assert np.array_equal(cat[k], rows1[k]), k
    for k in ("mean_q", "window_q"):
        assert np.array_equal(cat[k].view(np.uint64), rows1[k].view(np.uint64)), k
    assert np.allclose(cat["final_score"], rows1["final_score"], rtol=1e-9, atol=0, equal_nan=True)
    assert (summaries[0].status, summaries[0].target, summaries[0].keeping) == (s1.status, s1.target, s1.keeping)
    # and a sample against the oracle (assembly text from the host generator)
    S = capi.synth_host_lib()
    g = np.zeros(nc * pc // 16 + 8, dtype=np.uint32); nm = np.zeros(nc * pc // 32 + 8, dtype=np.uint32)
    S.fl_synth_assembly_host(4, nc, cb, 20000, capi.ptr(g), capi.ptr(nm))
    txt = np.zeros(nc * pc + 64, dtype=np.uint8)
    S.fl_synth_ascii_host(nc, capi.ptr(np.arange(nc, dtype=np.uint64) * np.uint64(pc)), capi.ptr(np.full(nc, cb, dtype=np.int32)),
                          capi.ptr(g), capi.ptr(nm), capi.ptr(txt))
    ok = orc.Kmers()
    ok.add_assembly([txt[c * pc:c * pc + cb].tobytes() for c in range(nc)])
    assert len(ok) == n_k
    idx = np.arange(300)
    sc = orc.score(_host_reads(w, idx, g), orc.make_params(**kw), ok)
    parity.check_reads_vs_oracle({k: v[idx] for k, v in one.read_results().items()}, sc)
    for c in ctxs + [one]:
        c.close()

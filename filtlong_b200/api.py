"""Thin Python convenience layer over the C ABI (tests / bench plumbing; the product's host side
is the C++ facade in filtlong_b200/csrc/host/). Nothing here computes scores: packing goes through
the library's own host packer and every number comes back from the CUDA kernels."""
import ctypes as C

import numpy as np

from . import capi
from .capi import FLError, make_params  # noqa: F401


class HostBatch:
    """A batch of sequences in the arena layout of include/filtlong_b200.h (host memory)."""

    def __init__(self, seqs, quals=None, want_seq=True, want_nmask=False):
        L = capi.lib()
        n = len(seqs)
        self.n = n
        self.len = np.array([len(s) for s in seqs], dtype=np.int32)
        padded = np.array([L.fl_padded_len(int(x)) for x in self.len], dtype=np.uint64)
        self.off = np.zeros(n, dtype=np.uint64)
        if n:
            self.off[1:] = np.cumsum(padded)[:-1]
        self.padded_bases = int(padded.sum())
        self.seq2b = np.zeros(max(self.padded_bases // 16, 1), dtype=np.uint32) if want_seq else None
        self.nmask = np.zeros(max(self.padded_bases // 32, 1), dtype=np.uint32) if want_nmask else None
        have_q = quals is not None and any(q is not None for q in quals)
        self.qual = np.zeros(max(self.padded_bases, 1), dtype=np.uint8) if have_q else None
        for i, s in enumerate(seqs):
            q = quals[i] if have_q else None
            L.fl_pack_sequence(s, q, len(s), int(self.off[i]), capi.ptr(self.seq2b), capi.ptr(self.qual),
                               capi.ptr(self.nmask))
        self.total_bases = int(self.len.sum())

    def c_batch(self):
        b = capi.Batch()
        b.n = self.n
        b.padded_bases = self.padded_bases
        b.off, b.len = capi.ptr(self.off), capi.ptr(self.len)
        b.seq2b, b.qual, b.nmask = capi.ptr(self.seq2b), capi.ptr(self.qual), capi.ptr(self.nmask)
        return b


def device_batch(n, padded_bases, off, length, seq2b=None, qual=None, nmask=None, ascii=None):
    """fl_batch whose pointers are device pointers (torch tensors or raw ints)."""
    b = capi.Batch()
    b.n = n
    b.padded_bases = padded_bases
    b.off, b.len = capi.ptr(off), capi.ptr(length)
    b.seq2b, b.qual, b.nmask = capi.ptr(seq2b), capi.ptr(qual), capi.ptr(nmask)
    b.ascii = capi.ptr(ascii)
    return b


class Context:
    def __init__(self, params=None, device=0):
        self.L = capi.lib()
        self.params = params if params is not None else make_params()
        h = C.c_void_p()
        rc = self.L.fl_ctx_create(C.byref(self.params), device, C.byref(h))
        if rc != 0:
            raise FLError("fl_ctx_create failed (%d): %s" % (rc, self.L.fl_last_error(None).decode()))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.fl_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc, what):
        capi.check(self.h, rc, what)

    def set_stream(self, stream_ptr):
        self._ck(self.L.fl_ctx_set_stream(self.h, stream_ptr), "fl_ctx_set_stream")

    def sync(self):
        self._ck(self.L.fl_ctx_sync(self.h), "fl_ctx_sync")

    def set_params(self, params):
        self.params = params
        self._ck(self.L.fl_ctx_set_params(self.h, C.byref(params)), "fl_ctx_set_params")

    def launch_count(self):
        return int(self.L.fl_ctx_launch_count(self.h))

    KERNELS = {"score_phred": 0, "probe_paint": 1, "kmer_stats": 2, "kmers_add": 3,
               "qual_mask": 4, "row_scan": 5, "qual_gather": 6, "qual_children": 7, "contam": 8, "bam_build": 9, "bgzf": 10}

    def enable_timing(self, on=True):
        self._ck(self.L.fl_ctx_enable_timing(self.h, int(on)), "fl_ctx_enable_timing")

    def reset_timing(self):
        self._ck(self.L.fl_ctx_reset_timing(self.h), "fl_ctx_reset_timing")

    def kernel_time(self, name):
        ms, n = C.c_double(), C.c_uint64()
        self._ck(self.L.fl_ctx_kernel_time(self.h, self.KERNELS[name], C.byref(ms), C.byref(n)), "fl_ctx_kernel_time")
        return ms.value, n.value

    def phred_paths(self):
        """k_phred_win's path counters (fl_ctx_phred_paths): {path: (reads, bases)} and the exact steps walked."""
        out = np.zeros(9, dtype=np.uint64)
        self._ck(self.L.fl_ctx_phred_paths(self.h, out.ctypes.data), "fl_ctx_phred_paths")
        paths = {k: (int(out[2 * i]), int(out[2 * i + 1])) for i, k in enumerate(("candidates", "full_walk", "reject_byte", "reject_low"))}
        return paths, int(out[8])

    # ---- Kmers (kmers.h:28-55) ----
    def kmers_add(self, seqs, multiple_copies, chunk=200000):
        for i in range(0, len(seqs), chunk):
            hb = HostBatch(seqs[i:i + chunk], None, want_seq=True, want_nmask=True)
            b = hb.c_batch()
            self._ck(self.L.fl_kmers_add_batch(self.h, C.byref(b), int(multiple_copies)), "fl_kmers_add_batch")

    def kmers_add_device(self, batch, multiple_copies):
        self._ck(self.L.fl_kmers_add_batch_device(self.h, C.byref(batch), int(multiple_copies)),
                 "fl_kmers_add_batch_device")

    def kmers_count(self):
        n = C.c_uint64()
        self._ck(self.L.fl_kmers_finalize(self.h, C.byref(n)), "fl_kmers_finalize")
        return n.value

    def kmers_contains(self, kmers):
        k = np.ascontiguousarray(kmers, dtype=np.uint32)
        out = np.zeros(k.size, dtype=np.uint8)
        self._ck(self.L.fl_kmers_contains(self.h, capi.ptr(k), k.size, capi.ptr(out)), "fl_kmers_contains")
        return out.astype(bool)

    def kmers_export(self):
        n = self.kmers_count()
        out = np.zeros(max(n, 1), dtype=np.uint32)
        got = C.c_uint64()
        self._ck(self.L.fl_kmers_export(self.h, capi.ptr(out), n, C.byref(got)), "fl_kmers_export")
        return out[:n]

    def kmers_bitmap_dev(self):
        p, nb = C.c_void_p(), C.c_uint64()
        self._ck(self.L.fl_kmers_bitmap_dev(self.h, C.byref(p), C.byref(nb)), "fl_kmers_bitmap_dev")
        return p.value, nb.value

    def kmers_bitmap_changed(self):
        self._ck(self.L.fl_kmers_bitmap_changed(self.h), "fl_kmers_bitmap_changed")

    def kmers_release_build_state(self):
        self._ck(self.L.fl_kmers_release_build_state(self.h), "fl_kmers_release_build_state")

    def kmers_probe_info(self):
        """(pre-filter in use, its flavour bits, log2 of its words, anchored table in use): fl_kmers_probe_info."""
        info = (C.c_int32 * 4)()
        self._ck(self.L.fl_kmers_probe_info(self.h, info), "fl_kmers_probe_info")
        return dict(pre_filter=bool(info[0]), filter_kind=int(info[1]), filter_log2_words=int(info[2]), anchored=bool(info[3]))

    # ---- contaminant set (--contam) ----
    def contam_add(self, seqs, chunk=200000):
        for i in range(0, len(seqs), chunk):
            hb = HostBatch(seqs[i:i + chunk], None, want_seq=True, want_nmask=True)
            b = hb.c_batch()
            self._ck(self.L.fl_contam_add_batch(self.h, C.byref(b)), "fl_contam_add_batch")

    def contam_add_text(self, data: bytes, fastq=True, is_last=True):
        """fl_contam_add_text on one chunk of a contaminant file (FASTQ / FASTA text)."""
        n, nb, used, st = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_int()
        buf = np.frombuffer(data, dtype=np.uint8)
        self._ck(self.L.fl_contam_add_text(self.h, capi.ptr(buf), len(data), 1 if fastq else 2, int(is_last),
                                           C.byref(n), C.byref(nb), C.byref(used), C.byref(st)), "fl_contam_add_text")
        return dict(status="fallback" if st.value else "ok", n=n.value, bases=nb.value, consumed=used.value)

    def contam_count(self):
        n = C.c_uint64()
        self._ck(self.L.fl_contam_finalize(self.h, C.byref(n)), "fl_contam_finalize")
        return n.value

    def contam_export(self):
        n = self.contam_count()
        out = np.zeros(max(n, 1), dtype=np.uint32)
        got = C.c_uint64()
        self._ck(self.L.fl_contam_export(self.h, capi.ptr(out), n, C.byref(got)), "fl_contam_export")
        return out[:n]

    def contam_configure(self, k, max_kmers=0):
        """fl_contam_configure: k-mers of k = 16..32 bases, a set of k > 16 sized for max_kmers canonical k-mers."""
        self._ck(self.L.fl_contam_configure(self.h, int(k), int(max_kmers)), "fl_contam_configure")

    def contam_export64(self):
        """the canonical members of a set of k > 16, sorted"""
        n = C.c_uint64()
        self._ck(self.L.fl_contam_export64(self.h, None, 0, C.byref(n)), "fl_contam_export64")
        out = np.zeros(max(n.value, 1), dtype=np.uint64)
        got = C.c_uint64()
        self._ck(self.L.fl_contam_export64(self.h, capi.ptr(out), n.value, C.byref(got)), "fl_contam_export64")
        return np.sort(out[:n.value])

    def contam_contains64(self, fwd_kmers):
        """per forward k-mer (2-bit codes, first base high): in a set of k > 16 on either strand"""
        q = np.ascontiguousarray(fwd_kmers, dtype=np.uint64)
        out = np.zeros(max(len(q), 1), dtype=np.uint8)
        self._ck(self.L.fl_contam_contains64(self.h, capi.ptr(q), len(q), capi.ptr(out)), "fl_contam_contains64")
        return out[:len(q)].astype(bool)

    def contam_probe_lengths(self, n_bins=16):
        """(members by sectors read per look-up, buckets by sectors an absent k-mer's look-up reads); last bin = or more"""
        h = np.zeros(2 * n_bins, dtype=np.uint64)
        self._ck(self.L.fl_contam_probe_lengths(self.h, capi.ptr(h), n_bins), "fl_contam_probe_lengths")
        return h[:n_bins], h[n_bins:]

    def contam_broadcast(self, root=0):
        self._ck(self.L.fl_contam_broadcast(self.h, root), "fl_contam_broadcast")

    def contam_results(self):
        """Per input read: (percent of bases in contaminant 16-mers, removed), and the removed reads / bases / rows."""
        n, _, _ = self.counts()
        pct, rem = np.zeros(max(n, 1)), np.zeros(max(n, 1), np.uint8)
        cc = capi.ContamCounts()
        self._ck(self.L.fl_results_contam(self.h, capi.ptr(pct), capi.ptr(rem), C.byref(cc)), "fl_results_contam")
        return pct[:n], rem[:n].astype(bool), dict(reads=cc.reads, bases=cc.bases, rows=cc.rows)

    # ---- sharded read set (one context per GPU, NCCL behind the C ABI) ----
    @staticmethod
    def comm_unique_id():
        buf = (C.c_uint8 * 128)()
        rc = capi.lib().fl_comm_unique_id(buf)
        if rc != 0:
            raise FLError("fl_comm_unique_id failed (%d): NCCL not available" % rc)
        return bytes(buf)

    def comm_init(self, id128, rank, nranks):
        buf = (C.c_uint8 * 128).from_buffer_copy(id128)
        self._ck(self.L.fl_comm_init(self.h, buf, rank, nranks), "fl_comm_init")

    def comm_destroy(self):
        self._ck(self.L.fl_comm_destroy(self.h), "fl_comm_destroy")

    def kmers_broadcast(self, root=0):
        self._ck(self.L.fl_kmers_broadcast(self.h, root), "fl_kmers_broadcast")

    def allreduce_i64(self, values):
        a = np.ascontiguousarray(values, dtype=np.int64)
        self._ck(self.L.fl_comm_allreduce_i64_host(self.h, capi.ptr(a), a.size), "fl_comm_allreduce_i64_host")
        return a

    def collective_count(self):
        return int(self.L.fl_comm_collective_count(self.h))

    # ---- Read (read.h:29-65) ----
    def push(self, host_batch):
        b = host_batch.c_batch()
        self._ck(self.L.fl_reads_push(self.h, C.byref(b)), "fl_reads_push")

    def push_text(self, data: bytes, fastq=True, is_last=True, cap=None):
        """fl_reads_push_text on one chunk of FASTQ / FASTA text. Returns a dict with status, n, consumed and
        the record index arrays (chunk-relative offsets)."""
        n_cap = cap if cap is not None else max(data.count(b"\n") // (4 if fastq else 2) + 2, 8)
        arr = dict(name_off=np.zeros(n_cap, np.uint64), name_len=np.zeros(n_cap, np.uint32), comment_len=np.zeros(n_cap, np.uint32),
                   seq_off=np.zeros(n_cap, np.uint64), qual_off=np.zeros(n_cap, np.uint64), len=np.zeros(n_cap, np.int32),
                   name_hash=np.zeros(n_cap, np.uint64))
        rec = capi.TextRecords(cap=n_cap, **{k: capi.ptr(v) for k, v in arr.items()})
        n, used, st = C.c_uint64(), C.c_uint64(), C.c_int()
        buf = np.frombuffer(data, dtype=np.uint8)
        rc = self.L.fl_reads_push_text(self.h, capi.ptr(buf), len(data), 1 if fastq else 2, int(is_last), C.byref(rec), C.byref(n),
                                       C.byref(used), C.byref(st))
        if rc == -5:
            return dict(status="erange", n=n.value)
        self._ck(rc, "fl_reads_push_text")
        out = {k: v[:n.value] for k, v in arr.items()}
        out.update(status="fallback" if st.value else "ok", n=n.value, consumed=used.value)
        return out

    def push_bam(self, chunk: bytes, seq_off, qual_off, length, reverse=None):
        """fl_reads_push_bam on a chunk of inflated BAM records: per record the chunk-relative offsets of SEQ and QUAL
        and l_seq. reverse (optional): per record, true when it stores its read reverse-complemented
        (fl_reads_push_bam_strand)."""
        so = np.ascontiguousarray(seq_off, dtype=np.uint32)
        qo = np.ascontiguousarray(qual_off, dtype=np.uint32)
        ln = np.ascontiguousarray(length, dtype=np.int32)
        buf = np.frombuffer(chunk, dtype=np.uint8)
        if reverse is None:
            self._ck(self.L.fl_reads_push_bam(self.h, capi.ptr(buf), buf.size, ln.size, capi.ptr(so), capi.ptr(qo), capi.ptr(ln)),
                     "fl_reads_push_bam")
            return
        rv = np.ascontiguousarray(reverse, dtype=np.uint8)
        if rv.size != ln.size:
            raise ValueError("push_bam: one reverse flag per record")
        self._ck(self.L.fl_reads_push_bam_strand(self.h, capi.ptr(buf), buf.size, ln.size, capi.ptr(so), capi.ptr(qo), capi.ptr(ln),
                                                 capi.ptr(rv)), "fl_reads_push_bam_strand")

    def kmers_add_text(self, data: bytes, fastq=True, is_last=True, multiple_copies=False):
        """fl_kmers_add_text on one chunk of a reference file (FASTQ / FASTA text)."""
        n, nb, used, st = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_int()
        buf = np.frombuffer(data, dtype=np.uint8)
        self._ck(self.L.fl_kmers_add_text(self.h, capi.ptr(buf), len(data), 1 if fastq else 2, int(is_last), int(multiple_copies),
                                          C.byref(n), C.byref(nb), C.byref(used), C.byref(st)), "fl_kmers_add_text")
        return dict(status="fallback" if st.value else "ok", n=n.value, bases=nb.value, consumed=used.value)

    def push_device(self, batch):
        self._ck(self.L.fl_reads_push_device(self.h, C.byref(batch)), "fl_reads_push_device")

    def reset_reads(self):
        self._ck(self.L.fl_reads_reset(self.h), "fl_reads_reset")

    def counts(self):
        a, b, t = C.c_uint64(), C.c_uint64(), C.c_int64()
        self._ck(self.L.fl_reads_count(self.h, C.byref(a), C.byref(b), C.byref(t)), "fl_reads_count")
        return a.value, b.value, t.value

    def finalize(self, total_bases=-1):
        s = capi.Summary()
        self._ck(self.L.fl_finalize(self.h, total_bases, C.byref(s)), "fl_finalize")
        return s

    def read_results(self):
        n, _, _ = self.counts()
        m = max(n, 1)
        r = dict(length=np.zeros(m, np.int32), mean_q=np.zeros(m), window_q=np.zeros(m), length_score=np.zeros(m),
                 passed=np.zeros(m, np.uint8), first_base_in_kmer=np.zeros(m, np.int32),
                 last_base_in_kmer=np.zeros(m, np.int32), n_bad=np.zeros(m, np.int32), n_child=np.zeros(m, np.int32),
                 row_start=np.zeros(m, np.uint64))
        o = capi.ReadResults(**{k: capi.ptr(v) for k, v in r.items()})
        self._ck(self.L.fl_results_reads(self.h, C.byref(o)), "fl_results_reads")
        return {k: v[:n] for k, v in r.items()}

    # ---- BGZF output (fl_bgzf_compress*) ----
    def bgzf_compress(self, data, append_eof=True):
        """data (bytes-like) compressed as BGZF on the device: bytes that any gzip reader inflates back to data."""
        src = np.frombuffer(data, dtype=np.uint8)
        out = np.empty(int(self.L.fl_bgzf_bound(src.size)), dtype=np.uint8)
        n = C.c_uint64()
        self._ck(self.L.fl_bgzf_compress(self.h, capi.ptr(src), src.size, capi.ptr(out), out.size, int(append_eof), C.byref(n)),
                 "fl_bgzf_compress")
        return out[:n.value].tobytes()

    def bgzf_compress_device(self, dev_in, n, dev_out, cap, append_eof=True):
        """Device buffers (torch tensors or raw pointers); returns the compressed size, or None when cap is too small."""
        m = C.c_uint64()
        rc = self.L.fl_bgzf_compress_device(self.h, capi.ptr(dev_in), n, capi.ptr(dev_out), cap, int(append_eof), C.byref(m))
        if rc == capi.FL_ERANGE:
            return None
        self._ck(rc, "fl_bgzf_compress_device")
        return m.value

    # ---- BAM output (fl_bam_build) ----
    def bam_build(self, batch, items, keep_mods=False):
        """The uncompressed BAM records of items over the bytes `batch`: items are (off, s, e) -- s < 0 copies bytes
        [off, off + e), else the child [s, e) of the record at off. Returns (bytes, [kept, invalid])."""
        src = np.frombuffer(batch, dtype=np.uint8)
        it = bam_items(items)
        counts = np.zeros(2, np.uint64)
        n = C.c_uint64()
        cap = 0
        while True:
            out = np.empty(max(cap, 1), dtype=np.uint8)
            rc = self.L.fl_bam_build(self.h, capi.ptr(src), src.size, capi.ptr(it), it.size, int(keep_mods), capi.ptr(out), cap,
                                     C.byref(n), capi.ptr(counts))
            if rc != capi.FL_ERANGE:
                break
            cap = n.value
            counts[:] = 0
        self._ck(rc, "fl_bam_build")
        return out[:n.value].tobytes(), [int(x) for x in counts]

    def row_results(self):
        _, n, _ = self.counts()
        m = max(n, 1)
        r = dict(parent=np.zeros(m, np.uint32), start=np.zeros(m, np.int32), end=np.zeros(m, np.int32),
                 mean_q=np.zeros(m), window_q=np.zeros(m), length_score=np.zeros(m), norm_mean=np.zeros(m),
                 norm_window=np.zeros(m), final_score=np.zeros(m), passed=np.zeros(m, np.uint8),
                 passed_final=np.zeros(m, np.uint8))
        o = capi.RowResults(**{k: capi.ptr(v) for k, v in r.items()})
        self._ck(self.L.fl_results_rows(self.h, C.byref(o)), "fl_results_rows")
        return {k: v[:n] for k, v in r.items()}


def bam_items(items):
    """(off, s, e) tuples as an array of fl_bam_item"""
    it = np.zeros(len(items), dtype=[("off", "<u8"), ("s", "<i4"), ("e", "<i4")])
    for k, (o, s_, e_) in enumerate(items):
        it[k] = (o, s_, e_)
    return it


class BamWriter:
    """fl_bam_writer on a context: one BGZF-compressed BAM stream, built and compressed batch by batch."""

    def __init__(self, ctx):
        self.ctx, self.h = ctx, C.c_void_p()
        ctx._ck(ctx.L.fl_bam_writer_create(ctx.h, C.byref(self.h)), "fl_bam_writer_create")

    def push(self, batch, items, keep_mods=False, last=False):
        """fl_bam_writer_push: the members of the whole blocks so far (all of them when last), and [kept, invalid]"""
        src = np.frombuffer(batch, dtype=np.uint8)
        it = bam_items(items)
        cap = int(self.ctx.L.fl_bgzf_bound(capi.FL_BGZF_BLOCK + 2 * src.size + 300 * len(items)))
        n = C.c_uint64()
        while True:                          # a push that does not fit changes nothing but the counts: again, with room
            out = np.empty(max(cap, 1), dtype=np.uint8)
            counts = np.zeros(2, np.uint64)
            rc = self.ctx.L.fl_bam_writer_push(self.h, capi.ptr(src), src.size, capi.ptr(it), it.size, int(keep_mods), int(last),
                                               capi.ptr(out), cap, C.byref(n), capi.ptr(counts))
            if rc != capi.FL_ERANGE:
                break
            cap = n.value
        self.ctx._ck(rc, "fl_bam_writer_push")
        return out[:n.value].tobytes(), [int(x) for x in counts]

    def close(self):
        if self.h:
            self.ctx.L.fl_bam_writer_destroy(self.h)
            self.h = None



def bgzf_compress(data, append_eof=True, device=0):
    """One-shot BGZF compression of host bytes on a fresh context (what `filtlong --bgzip` does to its output)."""
    with Context(device=device) as ctx:
        return ctx.bgzf_compress(data, append_eof)


def score_and_filter(reads, params, assembly=None, short_reads=None, device=0):
    """One-shot helper mirroring the reference's main(): build Kmers, score every read, finalize.
    reads: list of (seq, qual|None); assembly: list of seqs; short_reads: list of lists of seqs
    (file order, i.e. -1 then -2). Returns (context, summary)."""
    ctx = Context(params, device)
    if assembly:
        ctx.kmers_add(list(assembly), False)                 # main.cpp:54-56
    if short_reads:
        for f in short_reads:                                # main.cpp:57-58, file order
            ctx.kmers_add(list(f), True)
    ctx.kmers_count()
    hb = HostBatch([r[0] for r in reads], [r[1] for r in reads], want_seq=True)
    ctx.push(hb)
    summary = ctx.finalize(hb.total_bases)
    return ctx, summary

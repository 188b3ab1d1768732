// filtlong_b200/csrc/fl_internal.cuh -- shared declarations of the CUDA library (sm_90a only).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/filtlong_b200.h"

#define FL_BLOOM_BITS 1917295480ull   // bloom_filter.h:108-160 with kmers.cpp:32-34's parameters
#define FL_BLOOM_K 13
#define FL_ORDER_BUCKETS 1024
#define FL_COMM_MAX_RANKS 64
#define FL_SELECT_DIGIT_BITS 13           // the cut-off key is found 13 bits at a time: 5 levels for a 64-bit key
#define FL_SELECT_BINS (1 << FL_SELECT_DIGIT_BITS)
#define FL_COMM_SCRATCH_BYTES (FL_SELECT_BINS * 8 + 4096 * 8)

// ---------------------------------------------------------------------------------------------
// error plumbing: CUDA failures become FL_ECUDA + message, never exceptions
// ---------------------------------------------------------------------------------------------
#define FL_CUDA(ctx, call)                                                                     \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            (ctx)->set_error(std::string(#call) + ": " + cudaGetErrorString(e__));             \
            return FL_ECUDA;                                                                   \
        }                                                                                      \
    } while (0)

// every public entry point runs on its context's device (one process may hold one context per GPU)
#define FL_ENTER_NOFLUSH(c)                           \
    do {                                              \
        if (!(c)) return FL_EINVAL;                   \
        FL_CUDA((c), cudaSetDevice((c)->device));     \
    } while (0)

// every entry point but fl_reads_push first finishes a batch whose second half was deferred (fl_score_complete)
#define FL_ENTER(c)                                             \
    do {                                                        \
        FL_ENTER_NOFLUSH(c);                                    \
        if ((c)->kmer_pending) {                                \
            int rc_pending__ = fl_score_complete(c);            \
            if (rc_pending__ != FL_OK) return rc_pending__;     \
        }                                                       \
    } while (0)

#define FL_TRY(expr)                \
    do {                            \
        int rc__ = (expr);          \
        if (rc__ != FL_OK) return rc__; \
    } while (0)

// A grow-only device array. Growth synchronises the stream, so steady-state batches (same or
// smaller size than the largest seen) never allocate.
template <typename T>
struct DevVec {
    T *p = nullptr;
    size_t cap = 0;
    ~DevVec() { release(); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    // ensure capacity >= n elements, preserving the first `keep` elements
    cudaError_t reserve(size_t n, size_t keep, cudaStream_t s) {
        if (n <= cap) return cudaSuccess;
        size_t ncap = cap * 2 > n ? cap * 2 : n;
        if (ncap < 1024) ncap = 1024;
        T *np = nullptr;
        cudaError_t e = cudaMalloc(&np, ncap * sizeof(T));
        if (e != cudaSuccess) return e;
        if (keep && p) {
            e = cudaMemcpyAsync(np, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, s);
            if (e != cudaSuccess) return e;
        }
        e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) return e;
        if (p) cudaFree(p);
        p = np;
        cap = ncap;
        return cudaSuccess;
    }
};

// Device-side view of a batch (all pointers device memory).
struct BatchView {
    uint32_t n;
    uint64_t padded_bases;
    const uint64_t *off;
    const int32_t *len;
    const uint32_t *seq2b;
    const uint8_t *qual;
    const uint32_t *nmask;
    const uint8_t *ascii;
};

// State of the weighted radix select, lives in device memory (one instance per context).
struct SelectState {
    unsigned long long prefix;       // key bits decided so far (most significant digits)
    unsigned long long cum_before;   // passed bases (all ranks) with a strictly better key prefix
    long long target;                // main.cpp:229-237
    long long passed_bases;          // global
    long long total_bases;           // global
    int status;                      // fl_summary.status
    int active;                      // 1 while digits are still being resolved (status 3 and target > 0)
    unsigned long long tie_key;      // full key of the tie class at the cut-off
    unsigned long long tie_base;     // bases the tie class may still take: target - cum_before
};

#define FL_HSCALAR_ROWS 40
#define FL_SCALAR_PHRED_PATHS 30         // d_scalars[30, 39): k_phred_win's path counters (fl_ctx_phred_paths)
#define FL_SCALAR_CONTAM 20              // d_scalars[20, 23): removed reads, their bases, their rows (fl_results_contam)

// A 16-mer set and the tables the probe kernel reads. A context holds two: the reference set (read.cpp:35 decides the
// scoring mode by it) and the contaminant set (--contam), built, finalised and probed by the same code.
struct KmerSet {
    uint32_t *bitmap = nullptr;          // 2^32 bits, direct-address membership
    uint64_t n = 0;                      // members, valid while !stale
    bool stale = false;                  // the bitmap changed since n and the tables below were derived (fl_kmers_recount)
    // optional L2-resident pre-filter of the set (built when the set is small enough to make it selective)
    unsigned long long *filter = nullptr;
    // Flavour of the pre-filter (fl_device.cuh): bit 2 = one word per table group of four 16-mers; bit 3 = one word per pair
    // of neighbours; bit 4 = four bits per member instead of two (bits 0 and 1 are unused: former experiments). Chosen from
    // the set's size when the set is finalised (fl_kmers_recount).
    int filter_kind = 2;
    bool use_filter = false;
    uint32_t *anchor = nullptr;          // position-anchored membership table (2 GiB), see fl_anchor_slot
    bool use_anchor = false;
    bool added = false;                  // something was added (fl_contam_configure comes first)
    // k = 16: the bitmap and tables above. k = 17..32 (the contaminant set only, fl_contam_configure): a hash set of
    // canonical k-mers, 4 slots per bucket, then two counters: distinct members, palindromes (fl_contam_k.cu)
    int k = 16;
    unsigned long long *table = nullptr;
    uint64_t n_buckets = 0;
    uint64_t limit = 0;                  // the most members the table may hold (its load limit)
    void release() {
        if (bitmap) cudaFree(bitmap);
        if (filter) cudaFree(filter);
        if (anchor) cudaFree(anchor);
        if (table) cudaFree(table);
        bitmap = nullptr; filter = nullptr; anchor = nullptr; table = nullptr;
    }
};

struct fl_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    fl_params p{};
    std::string err;
    uint64_t launches = 0;
    int sm_count = 148;

    // ---- Kmers ----
    KmerSet ref;                         // -a / -1 / -2
    KmerSet contam;                      // --contam: reads covered by it beyond max_contam percent are removed
    // how the pre-filter and the anchored table of either set are chosen (tuning knobs, fl_kmers_recount)
    unsigned filter_log2_words = 22;     // 2^22 x 8 B = 32 MiB (sizes: see filter_min_bits_per_key)
    int filter_kind_request = -1;        // FL_FILTER_KIND (-1 = chosen from the set's size)
    uint64_t filter_group4_max = 6000000, filter_pair_max = 22000000;   // largest sets keyed by group / by pair (FL_FILTER_G4_MAX, FL_FILTER_PAIR_MAX)
    int anchor_enabled = 1;              // FL_ANCHOR=0 probes the bitmap itself (profiling, cross-checks)
    int filter_enabled = 1;              // FL_FILTER=0 disables (profiling)
    // The filter is used while it has at least this many bits per member: 40 keeps it to sets of <= 6.7 M members (the
    // group-keyed regime). Measured on an H100 80GB HBM3 at 400 W, config 3's set (20 M members) against 10 Gbp of reads,
    // probe ms: no filter 84.8; pair-keyed 16 / 32 / 64 MiB 101.5 / 115.9 / 148.7; per 16-mer 32 / 64 MiB 194.7 / 279.4.
    // Smaller sets were not measured on the H100.
    int filter_min_bits_per_key = 40;
    // multiple-copy build state of the reference set (kmers.cpp:142-166 in closed form, see fl_kmers.cu)
    uint32_t *d_seen[4] = {nullptr, nullptr, nullptr, nullptr};   // ">= 1,2,3,4 sightings" bitmaps
    unsigned long long *d_tfirst = nullptr;    // first add-stream index per k-mer (2^32 entries)
    unsigned long long *d_bittime = nullptr;   // first time each Bloom bit was set
    uint64_t add_counter = 0;                  // global add-stream index (kmers.cpp:109-120 order)
    bool multi_pending = false;
    bool multi_released = false;               // the state above was freed after adds: later multiple-copy adds are refused

    // ---- Phred LUTs ----
    double *d_lut = nullptr;   // [0..256) q, [256..512) a = q / window_size
    unsigned long long tie_binades = 0;     // bit e: some Phred table value ties when added to a sum in [2^e, 2^(e+1))
    unsigned long long tie_many = 0;        // bit e: more than one table value ties there
    unsigned char tie_char[64] = {0};       // the one that does, when exactly one
    unsigned long long tie_binades_a = 0;   // bit e: some window-table value ties when w is in [2^-e, 2^(1-e))
    bool fasta_two_line_only = false;       // fl_kmers_add_text: FASTA records of one sequence line only, no wrapped ones (FL_FASTA_TWO_LINE)
    int phred_mode = 1;                     // 1: k_phred_sum + k_phred_win (default); 0: work-item kernels (FL_PHRED_MODE)
    int phred_occupancy = 0;                // blocks per SM launched for the Phred kernels, 0 = the kernel's own default (FL_PHRED_OCC)
    int lut_window = -1;
    bool phred_attr_set = false, phred_items_attr_set = false;   // cudaFuncSetAttribute is per DEVICE: kept per context

    // ---- staging for host batches ----
    // two slots: the host->device copy of batch i+1 (copy_stream) overlaps the kernels of batch i
    struct Staging {
        DevVec<uint64_t> off;
        DevVec<int32_t> len;
        DevVec<uint32_t> seq, nmask;
        DevVec<uint8_t> qual, ascii;
        cudaEvent_t consumed = nullptr;   // recorded on the compute stream after the last kernel that reads this slot
        bool in_use = false;
    } stg[2];
    int stg_next = 0;
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copied = nullptr;

    // ---- per-batch scratch ----
    DevVec<uint32_t> sc_pack_seq, sc_pack_nmask;   // 2-bit codes / non-ACGT mask packed on the device from an ASCII DEVICE batch
    DevVec<uint32_t> sc_mask;        // 1 bit per padded base: base covered by a reference 16-mer (or a good 16-run, --trim_q)
    DevVec<uint32_t> sc_cmask;       // the same for the contaminant set
    // --trim_q: the batch's child rows as a view of their own (fl_qtrim.cu): offsets, lengths, gathered quality bytes
    DevVec<unsigned long long> sc_qoff;
    DevVec<int32_t> sc_qlen;
    DevVec<uint8_t> sc_qual;
    DevVec<unsigned long long> sc_sink;   // fl_phred_pass over rows: the per-read record fields it does not want go here
    DevVec<uint32_t> sc_order;       // rows in descending-length bucket order
    DevVec<uint32_t> tx_nl, tx_u32;  // fl_reads_push_text: newline positions; per-record name / comment / sequence / quality extents
    DevVec<int32_t> sc_items;        // length of each k_kmer_window item: the batch's reads, then its rows
    DevVec<unsigned long long> sc_u64a, sc_u64b, sc_u64c;
    DevVec<uint32_t> sc_u32a;
    DevVec<unsigned long long> sc_scan;   // block sums of fl_exclusive_scan_u64
    uint32_t *d_buckets = nullptr;         // 256 bucket counters + 256 cursors (fl_order_by_length)
    unsigned long long *d_scalars = nullptr;   // small device scalars (counts, cursors); [30, 39): FL_SCALAR_PHRED_PATHS
    unsigned long long *h_scalars = nullptr;   // pinned mirror
    // second half of a batch with --trim / --split (k-mer mode or --trim_q), deferred by fl_reads_push (fl_score.cu:
    // score_back)
    bool kmer_pending = false;
    bool pending_qual = false;              // the deferred batch is a --trim_q batch (no k-mer set)
    BatchView kmer_pending_view{};
    int kmer_pending_slot = -1;             // staging slot to release once the deferred kernels are queued
    cudaEvent_t ev_rows = nullptr;          // the batch's row count has reached h_scalars[FL_HSCALAR_ROWS]

    // ---- results: one entry per INPUT READ ----
    uint64_t n_reads = 0;
    int64_t total_bases = 0;
    DevVec<int32_t> r_len, r_first, r_last, r_nbad, r_nchild;
    DevVec<double> r_mean, r_window;
    DevVec<uint8_t> r_passed;
    DevVec<unsigned long long> r_rowstart;
    // with a non-empty contaminant set only: percent of the read's bases in its 16-mers, and c > max_contam
    DevVec<double> r_contam;
    DevVec<uint8_t> r_removed;

    // ---- results: one entry per reads2 ROW ----
    uint64_t n_rows = 0;
    DevVec<uint32_t> w_parent;
    DevVec<int32_t> w_start, w_end;
    DevVec<double> w_mean, w_window, w_nmean, w_nwindow, w_final;
    DevVec<uint8_t> w_passed, w_pfinal;
    DevVec<uint8_t> w_excl;          // with a non-empty contaminant set only: the row's read was removed (not ranked)
    DevVec<unsigned long long> w_key;
    bool finalized = false;

    // ---- finalize scratch ----
    SelectState *d_sel = nullptr;
    double *d_norm = nullptr;            // sums4, min1, max1, sq1 (+ padding)
    unsigned long long *d_hist = nullptr;  // 256 bins + tie/keeping scalars
    DevVec<double> sc_f64;

    // ---- sharded read set: one NCCL communicator per context (fl_comm.cu) ----
    void *comm = nullptr;                // ncclComm_t
    int comm_rank = 0, comm_nranks = 1;
    unsigned char *d_comm = nullptr;     // FL_COMM_SCRATCH_BYTES of send / receive buffers for the collectives of fl_finalize
    uint64_t collectives = 0;            // NCCL calls issued so far
    bool select_attr_set = false;

    // ---- BGZF compression (fl_bgzf.cu): its own buffers, so that it never touches the scored reads ----
    DevVec<uint8_t> bz_slots;                  // one 64 KiB member slot per block of a launch
    DevVec<uint32_t> bz_sizes;                 // member sizes of a launch
    DevVec<unsigned long long> bz_offs;        // their output offsets
    DevVec<unsigned long long> bz_state;       // [0] bytes written so far, [1] the output buffer was too small
    DevVec<uint8_t> bz_hin, bz_hout;           // fl_bgzf_compress: the host buffers' device copies
    bool inflate_attr_set = false;            // fl_gzip_inflate: k_inf_decode's shared memory limit is raised
    bool bgzf_attr_set = false;

    // ---- optional per-kernel timing (fl_ctx_enable_timing) ----
    bool timing = false;
    struct TimedLaunch { cudaEvent_t a, b; int which; };
    std::vector<TimedLaunch> timed;
    double kernel_ms[FL_KERNEL_COUNT] = {};
    uint64_t kernel_launches[FL_KERNEL_COUNT] = {};

    void set_error(const std::string &m) { err = m; }
};

// RAII bracket: records CUDA events on the launching stream around one kernel launch
struct KernelTimer {
    fl_ctx *c;
    fl_ctx::TimedLaunch t{};
    bool on;
    KernelTimer(fl_ctx *ctx, int which) : c(ctx), on(ctx->timing) {
        if (!on) return;
        t.which = which;
        if (cudaEventCreate(&t.a) != cudaSuccess || cudaEventCreate(&t.b) != cudaSuccess) { on = false; return; }
        cudaEventRecord(t.a, c->stream);
    }
    ~KernelTimer() {
        if (!on) return;
        cudaEventRecord(t.b, c->stream);
        c->timed.push_back(t);
    }
};

static inline unsigned fl_blocks(size_t n, unsigned threads) { return (unsigned)((n + threads - 1) / threads); }

// ---- implemented in fl_scan.cu ----
int fl_exclusive_scan_u64(fl_ctx *ctx, const unsigned long long *in, unsigned long long *out, size_t n,
                          unsigned long long *total_dev /* may be null */);
// rows 0..n-1 ordered by descending length bucket into order[] (lengths may be null when
// start/end are given: length = end - start)
int fl_order_by_length(fl_ctx *ctx, const int32_t *len, size_t n, uint32_t *order);
// same with caller-computed bucket keys in [0, FL_ORDER_BUCKETS): highest key first
int fl_order_by_key(fl_ctx *ctx, const uint32_t *key, size_t n, uint32_t *order);

// ---- implemented in fl_api.cu ----
// text -> 2-bit codes (+ non-ACGT mask when nmask != null), kmers.cpp:176-196 on the device
int fl_pack_ascii_device(fl_ctx *ctx, const uint8_t *ascii, uint64_t padded_bases, uint32_t *seq2b, uint32_t *nmask, cudaStream_t s);

// ---- implemented in fl_kmers.cu ----
int fl_kmers_ensure_bitmap(fl_ctx *ctx, KmerSet &s);
// multi (the reference's short-read rule) is only for ctx->ref
int fl_kmers_add_view(fl_ctx *ctx, KmerSet &s, const BatchView &b, int multi);
// FL_EINVAL (with a message) for a multiple-copy add after fl_kmers_release_build_state freed the counts of earlier adds
int fl_kmers_check_multi(fl_ctx *ctx, const char *entry);
int fl_kmers_recount(fl_ctx *ctx, KmerSet &s);
// both sets finalised (counts and probe tables current): every push calls it before it looks at ctx->ref.n
int fl_sets_ready(fl_ctx *ctx);
// FL_EINVAL (with a message) when the contaminant set is added to after reads were pushed
int fl_contam_check_order(fl_ctx *ctx);

// ---- implemented in fl_contam_k.cu (a set with k > 16) ----
int fl_ck_add_view(fl_ctx *ctx, KmerSet &s, const BatchView &b);
int fl_ck_recount(fl_ctx *ctx, KmerSet &s);
// the same mask as fl_probe_paint: 1 bit per padded base of b, the base is covered by a k-mer of s
int fl_ck_paint(fl_ctx *ctx, const KmerSet &s, const BatchView &b, uint32_t *mask, int timer);
int fl_ck_broadcast(fl_ctx *ctx, KmerSet &s, int root);

// ---- implemented in fl_score.cu ----
// defer = the caller will call fl_score_complete() later (fl_reads_push: after the NEXT batch's copy is under way), so
// that the one host round trip of --trim / --split (how many rows did this batch make?) does not stall the copy pipeline
int fl_score_view(fl_ctx *ctx, const BatchView &b, bool defer = false);
int fl_score_complete(fl_ctx *ctx);
// FL_EINVAL (with a message) when --trim_q is set and the k-mer set is not empty, or when the contaminant set is not
// empty and max_contam is outside [0, 100)
int fl_check_trim_q(fl_ctx *ctx);
// the batch's bases are needed as 2-bit codes: k-mer mode, or a contaminant set to probe
static inline bool fl_wants_bases(const fl_ctx *ctx) { return ctx->ref.n > 0 || ctx->contam.n > 0; }
// 1 bit per padded base of b into mask: the base is covered by a 16-mer of s (k_probe_paint, timed as `timer`)
int fl_probe_paint(fl_ctx *ctx, const KmerSet &s, const BatchView &b, uint32_t *mask, int timer);
int fl_reserve_reads(fl_ctx *ctx, size_t n_total);
int fl_reserve_rows(fl_ctx *ctx, size_t n_total);

// ---- implemented in fl_phred.cu ----
int fl_score_phred(fl_ctx *ctx, const BatchView &b);
// Where one Phred pass writes its scores: mean / window / passed per item of the view, which is a batch's reads or its
// rows. whole_reads = the items are the context's next reads: also write the rest of each read's record and its
// identity row (plain Phred mode).
struct PhredOut {
    double *mean, *window;
    uint8_t *passed;
    bool whole_reads;
};
int fl_phred_pass(fl_ctx *ctx, const BatchView &b, const PhredOut &o);

// ---- implemented in fl_qtrim.cu (--trim_q: --trim / --split on Phred qualities) ----
// sc_mask = 1 bit per padded base: the base lies in a run of FL_K bases whose qualities are all >= 33 + trim_q
int fl_qual_mask(fl_ctx *ctx, const BatchView &b);
// the batch's rows [n_rows, n_rows + n_rows_batch) have parent / start / end: score the children on their own quality
// bytes, give every childless read's row its read's scores
int fl_score_qual_rows(fl_ctx *ctx, const BatchView &b, size_t n_rows_batch);

// ---- implemented in fl_comm.cu (no-ops / plain copies on a context without a communicator) ----
int fl_comm_allgather(fl_ctx *ctx, const void *send, void *recv, size_t bytes_per_rank);
int fl_comm_allreduce_u64(fl_ctx *ctx, unsigned long long *buf, size_t n);
int fl_comm_broadcast_bytes(fl_ctx *ctx, void *buf, size_t bytes, int root);

// ---- implemented in fl_select.cu ----
int fl_norm_select_free(fl_ctx *ctx);

// filtlong_b200/csrc/fl_select.cu -- global normalisation, final score and the --target_bases /
// --keep_percent cut, replacing the inline block of the reference's main (src/main.cpp:169-261)
// and Read::set_final_score (src/read.cpp:249-267).
//
// Selection is NOT a sort. The reference sorts descending by final score and keeps passed reads
// while the running total of kept bases is below the target (main.cpp:247-257); a row is therefore
// kept iff  passed && (bases of passed rows ranked strictly before it) < target.  We find the
// cut-off key with a base-WEIGHTED most-significant-digit radix select over the order-preserving
// 64-bit image of the score (a histogram of BASES per digit: 5 levels of 13-bit digits in
// fl_finalize, 8 levels of 8-bit digits in the split-phase fl_select_hist / fl_select_pick), then
// resolve the tie class at the cut-off in (rank, row) order with one prefix scan. The per-level
// histogram is the only thing a sharded run has to all-reduce, which is why the phases are exposed
// separately in the C ABI. A target <= 0 (reachable through the C ABI, or a small keep_percent)
// keeps nothing, as the reference's walk does: no digit is resolved and the cut clears every flag.
//
// Floating point: every per-row expression follows the reference's operation order (no FMA).
// The two global sums (main.cpp:173,183) are fixed-shape tree reductions instead of the
// reference's left-to-right loop, and pow() is CUDA's (<= 2 ulp) instead of glibc's, so
// normalised / final scores agree with the reference to ~1e-15 relative, not bit-for-bit. Given
// the statistics fl_select_summary reports, every row's rescaling is a fixed sequence of IEEE
// operations, and the cut is exactly a stable descending sort plus the prefix walk (DESIGN.md §5).
#include "fl_internal.cuh"

namespace {

constexpr int RED_BLOCKS = 1024;
constexpr int RED_THREADS = 256;

struct RowsView {
    size_t n;
    const int32_t *start, *end;
    const double *mean, *window;
    const uint8_t *passed;
    const uint8_t *excl;             // rows of reads removed by the contaminant set (skipped); null without one
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int d = 16; d; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    return v;
}

// fixed-shape block reduction (same tree every run -> deterministic bits)
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double ws[RED_THREADS / 32];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = 0.0;
    if (threadIdx.x < 32) {
        r = threadIdx.x < RED_THREADS / 32 ? ws[threadIdx.x] : 0.0;
        r = warp_sum(r);
    }
    __syncthreads();
    return r;   // valid in thread 0
}

// partials layout per block b: [b*6 + 0..5] = n, sum_q, passed_bases, rows_bases, min, max
__global__ void __launch_bounds__(RED_THREADS) k_norm_p1(RowsView v, double *__restrict__ partials) {
    const size_t chunk = (v.n + gridDim.x - 1) / gridDim.x;
    const size_t lo = chunk * blockIdx.x, hi = lo + chunk < v.n ? lo + chunk : v.n;
    double s = 0.0, pb = 0.0, rb = 0.0, mn = 100.0, mx = 0.0, cnt = 0.0;   // main.cpp:170-172
    for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        if (v.excl && v.excl[i]) continue;
        const double x = v.mean[i];
        const double len = (double)(v.end[i] - v.start[i]);
        s += x;
        cnt += 1.0;
        rb += len;
        if (v.passed[i]) pb += len;
        if (x > mx) mx = x;                 // main.cpp:175-178 (a NaN never updates either)
        if (x < mn) mn = x;
    }
    __shared__ double smn[RED_THREADS], smx[RED_THREADS];
    smn[threadIdx.x] = mn;
    smx[threadIdx.x] = mx;
    s = block_sum(s);
    cnt = block_sum(cnt);
    pb = block_sum(pb);
    rb = block_sum(rb);
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < RED_THREADS; ++i) {
            if (smn[i] < mn) mn = smn[i];
            if (smx[i] > mx) mx = smx[i];
        }
        double *p = partials + (size_t)blockIdx.x * 6;
        p[0] = cnt; p[1] = s; p[2] = pb; p[3] = rb; p[4] = mn; p[5] = mx;
    }
}

__global__ void __launch_bounds__(RED_THREADS) k_norm_p1_final(const double *__restrict__ partials, int nb,
                                                               double *sums4, double *min1, double *max1) {
    double a[4] = {0, 0, 0, 0}, mn = 100.0, mx = 0.0;
    for (int b = threadIdx.x; b < nb; b += blockDim.x) {
        const double *p = partials + (size_t)b * 6;
#pragma unroll
        for (int k = 0; k < 4; ++k) a[k] += p[k];
        if (p[4] < mn) mn = p[4];
        if (p[5] > mx) mx = p[5];
    }
    __shared__ double smn[RED_THREADS], smx[RED_THREADS];
    smn[threadIdx.x] = mn;
    smx[threadIdx.x] = mx;
    double r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) r[k] = block_sum(a[k]);
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < RED_THREADS; ++i) {
            if (smn[i] < mn) mn = smn[i];
            if (smx[i] > mx) mx = smx[i];
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) sums4[k] = r[k];
        *min1 = mn;
        *max1 = mx;
    }
}

__global__ void __launch_bounds__(RED_THREADS) k_norm_p2(RowsView v, const double *__restrict__ sums4,
                                                         double *__restrict__ partials) {
    const double mean = sums4[1] / sums4[0];                                 // main.cpp:179
    const size_t chunk = (v.n + gridDim.x - 1) / gridDim.x;
    const size_t lo = chunk * blockIdx.x, hi = lo + chunk < v.n ? lo + chunk : v.n;
    double s = 0.0;
    for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        if (v.excl && v.excl[i]) continue;
        const double d = v.mean[i] - mean;                                   // main.cpp:182-183
        s += d * d;
    }
    s = block_sum(s);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(RED_THREADS) k_sum_partials(const double *__restrict__ partials, int nb, double *out) {
    double a = 0.0;
    for (int b = threadIdx.x; b < nb; b += blockDim.x) a += partials[b];
    a = block_sum(a);
    if (threadIdx.x == 0) *out = a;
}

__device__ __forceinline__ double ref_pow(double x, double y) {
    // glibc returns x for y == 1 exactly; sqrt is correctly rounded like glibc's pow(x, 0.5) almost
    // always is. Anything else goes through CUDA's pow (<= 2 ulp).
    if (y == 1.0) return x;
    if (y == 0.5 && x >= 0.0) return sqrt(x);
    return pow(x, y);
}

__device__ __forceinline__ double final_score(double ls, double mq, double wq, double lw, double mw, double ww) {
    const double product = ref_pow(ls, lw) * ref_pow(mq, mw);               // read.cpp:252
    double total = lw + mw;
    const double fs = ref_pow(product, 1.0 / total);                        // read.cpp:254
    double sf;
    if (mq > 0.0) {                                                          // read.cpp:258-261
        const double r = wq / mq;
        sf = (1.0 < r) ? 1.0 : r;       // std::min(r, 1.0): NaN stays NaN (CUDA fmin would not)
    } else sf = 1.0;
    total = lw + mw + ww;
    const double wf = ww / total;
    const double nwf = 1.0 - wf;
    sf = nwf + (sf * wf);
    return fs * sf;
}

__device__ __forceinline__ unsigned long long score_key(double x) {
    // ascending key order == descending score; all NaNs collapse to the best key, so NaN rows rank
    // first, in row order. NaNs occur when every row is NaN (main.cpp:188-207 with stdev == 0), and
    // next to finite rows when invalid quality bytes make a mean negative: an all-'!' read then has
    // a normalised mean > 0 and a window/mean ratio of 0/0.
    if (x != x) return 0ull;
    x = x + 0.0;                                    // -0.0 -> +0.0
    unsigned long long b = (unsigned long long)__double_as_longlong(x);
    unsigned long long u = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
    return ~u;
}

struct ApplyArgs {
    RowsView v;
    const double *sums4, *min1, *max1, *sq1;
    double lw, mw, ww;
    double *nmean, *nwindow, *fscore;
    unsigned long long *key;
    uint8_t *pfinal;
};

__global__ void __launch_bounds__(256) k_norm_apply(ApplyArgs a) {
    const double n = a.sums4[0];
    const double mean = a.sums4[1] / n;
    const double sd = sqrt(a.sq1[0] / n);                                    // main.cpp:187
    double minz, maxz;
    if (sd > 0.0) { minz = (a.min1[0] - mean) / sd; maxz = (a.max1[0] - mean) / sd; }   // main.cpp:189-196
    else { minz = 1.0; maxz = 1.0; }
    const double span = maxz - minz;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.v.n; i += (size_t)gridDim.x * blockDim.x) {
        const double mq = a.v.mean[i], wq = a.v.window[i];
        double ratio = wq / mq;                                              // main.cpp:203-205
        if (ratio > 1.0) ratio = 1.0;
        const double z = (mq - mean) / sd;                                   // main.cpp:206
        const double nm = 100.0 * (z - minz) / span;                         // main.cpp:207
        const double nw = nm * ratio;                                        // main.cpp:208
        const int len = a.v.end[i] - a.v.start[i];
        const double ls = 100.0 * (1.0 + (-5000.0 / ((double)len + 5000.0)));   // read.cpp:241-244
        const double fs = final_score(ls, nm, nw, a.lw, a.mw, a.ww);
        a.nmean[i] = nm;
        a.nwindow[i] = nw;
        a.fscore[i] = fs;
        a.key[i] = score_key(fs);
        a.pfinal[i] = a.v.passed[i];
    }
}

__global__ void k_select_begin(SelectState *st, const double *sums4, long long target, long long total_bases,
                               int any_target) {
    if (threadIdx.x || blockIdx.x) return;
    SelectState s{};
    s.target = target;
    s.total_bases = total_bases;
    s.passed_bases = (long long)sums4[2];
    if (!any_target) s.status = 0;
    else if (target >= total_bases) s.status = 1;                            // main.cpp:239-240
    else if (target >= s.passed_bases) s.status = 2;                         // main.cpp:242-243
    else s.status = 3;
    s.active = s.status == 3 && target > 0;     // target <= 0: nothing to resolve, the cut keeps no row
    *st = s;
}

struct HistArgs {
    size_t n;
    const unsigned long long *key;
    const int32_t *start, *end;
    const uint8_t *passed;
    const SelectState *st;
    int level;
    unsigned long long *hist;   // [256]
};

__global__ void __launch_bounds__(256) k_select_hist(HistArgs a) {
    __shared__ unsigned long long h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    if (a.st->active) {
        const unsigned long long prefix = a.st->prefix;
        const int shift = 56 - 8 * a.level;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x) {
            if (!a.passed[i]) continue;
            const unsigned long long k = a.key[i];
            if (a.level > 0 && (k >> (shift + 8)) != prefix) continue;
            atomicAdd(&h[(k >> shift) & 0xFF], (unsigned long long)(a.end[i] - a.start[i]));
        }
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&a.hist[threadIdx.x], h[threadIdx.x]);
}

__global__ void k_select_pick(SelectState *st, const unsigned long long *hist, int level) {
    if (threadIdx.x || blockIdx.x) return;
    if (!st->active) return;
    unsigned long long cum = st->cum_before;
    const unsigned long long target = (unsigned long long)st->target;
    int pick = -1, last_nonempty = -1;
    unsigned long long before_pick = cum, before_last = cum;
    for (int d = 0; d < 256; ++d) {
        const unsigned long long c = hist[d];
        if (c) { last_nonempty = d; before_last = cum; }
        if (pick < 0 && c && cum + c >= target) { pick = d; before_pick = cum; }
        cum += c;
    }
    if (pick < 0) { pick = last_nonempty < 0 ? 0 : last_nonempty; before_pick = before_last; }   // cannot happen while active
    st->cum_before = before_pick;
    st->prefix = (st->prefix << 8) | (unsigned long long)pick;
    if (level == 7) {
        st->tie_key = st->prefix;
        st->tie_base = target > st->cum_before ? target - st->cum_before : 0ull;
    }
}

struct TieArgs {
    size_t n;
    const unsigned long long *key;
    const int32_t *start, *end;
    const uint8_t *passed;
    const SelectState *st;
    unsigned long long *tie_len;   // [n]: len if row is a passed member of the tie class, else 0
};

__global__ void __launch_bounds__(256) k_tie_len(TieArgs a) {
    const bool active = a.st->active;
    const unsigned long long tk = a.st->tie_key;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x)
        a.tie_len[i] = (active && a.passed[i] && a.key[i] == tk) ? (unsigned long long)(a.end[i] - a.start[i]) : 0ull;
}

__global__ void k_store_tie_total(const unsigned long long *total, unsigned long long *tie_per_rank, int rank, int nranks) {
    if (threadIdx.x || blockIdx.x) return;
    for (int r = 0; r < nranks; ++r) tie_per_rank[r] = (r == rank) ? *total : 0ull;
}

struct CutArgs {
    size_t n;
    const unsigned long long *key;
    const int32_t *start, *end;
    const uint8_t *passed;
    const SelectState *st;
    const unsigned long long *tie_excl;       // exclusive scan of tie_len (local)
    const unsigned long long *tie_per_rank;
    int rank;
    uint8_t *pfinal;
    unsigned long long *keeping;              // [1]
};

__global__ void __launch_bounds__(256) k_select_cut(CutArgs a) {
    unsigned long long kept = 0;
    if (a.st->status == 3) {
        // with a target <= 0 the select is inactive and no row is kept: bases_so_far (0) < target fails
        // for the first row already (main.cpp:252)
        const bool active = a.st->active;
        const unsigned long long tk = a.st->tie_key, room = a.st->tie_base;
        unsigned long long before = 0;
        for (int r = 0; r < a.rank; ++r) before += a.tie_per_rank[r];
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x) {
            uint8_t keep = 0;
            if (active && a.passed[i]) {
                const unsigned long long k = a.key[i];
                if (k < tk) keep = 1;                                          // strictly better than the cut-off key
                else if (k == tk) keep = (before + a.tie_excl[i]) < room;      // main.cpp:252: bases_so_far < target
            }
            a.pfinal[i] = keep;
            if (keep) kept += (unsigned long long)(a.end[i] - a.start[i]);
        }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) kept += __shfl_down_sync(0xffffffffu, kept, d);
    if ((threadIdx.x & 31) == 0 && kept) atomicAdd(a.keeping, kept);
}


// ---------------------------------------------------------------------------------------------
// fl_finalize: the same block with its exchanges behind the C ABI (fl_comm.cu). Scratch in ctx->d_comm:
// ---------------------------------------------------------------------------------------------
struct CommScratch {
    unsigned long long hist[FL_SELECT_BINS];       // base-weighted histogram of one 13-bit digit (all-reduced)
    double stats_send[8];                          // n, sum(mean_q), passed bases, row bases, min, max, input bases, -
    double stats_recv[8 * FL_COMM_MAX_RANKS];
    double sq_send[8];
    double sq_recv[8 * FL_COMM_MAX_RANKS];         // one double per rank (8-byte stride)
    unsigned long long tie_send[8];
    unsigned long long tie_recv[FL_COMM_MAX_RANKS];
    unsigned long long keeping[8];
    long long total_bases[8];                      // [0] global input bases (main.cpp:89 summed over the shards)
};
static_assert(sizeof(CommScratch) <= FL_COMM_SCRATCH_BYTES, "scratch block too small");

__global__ void k_stats_send(const double *sums4, const double *min1, const double *max1, const unsigned long long *dev_bases,
                             long long host_bases, double *send) {
    if (threadIdx.x || blockIdx.x) return;
    send[0] = sums4[0]; send[1] = sums4[1]; send[2] = sums4[2]; send[3] = sums4[3];
    send[4] = *min1; send[5] = *max1;
    send[6] = (double)(host_bases + (dev_bases ? (long long)*dev_bases : 0ll));     // < 2^53: exact
    send[7] = 0.0;
}

// combine the ranks' partials in rank order: every rank computes the same bits, whatever NCCL did inside
__global__ void k_stats_combine(const double *recv, int nranks, double *sums4, double *min1, double *max1, long long *total) {
    if (threadIdx.x || blockIdx.x) return;
    double a[4] = {0, 0, 0, 0}, mn = 100.0, mx = 0.0, tb = 0.0;                     // main.cpp:170-172
    for (int r = 0; r < nranks; ++r) {
        const double *p = recv + 8 * r;
        for (int k = 0; k < 4; ++k) a[k] += p[k];
        if (p[4] < mn) mn = p[4];
        if (p[5] > mx) mx = p[5];
        tb += p[6];
    }
    for (int k = 0; k < 4; ++k) sums4[k] = a[k];
    *min1 = mn;
    *max1 = mx;
    *total = (long long)tb;
}

__global__ void k_sq_combine(const double *recv, int nranks, double *sq1) {
    if (threadIdx.x || blockIdx.x) return;
    double a = 0.0;
    for (int r = 0; r < nranks; ++r) a += recv[r];
    *sq1 = a;
}

__global__ void k_select_begin_dev(SelectState *st, const double *sums4, const long long *total, fl_params p) {
    if (threadIdx.x || blockIdx.x) return;
    SelectState s{};
    const long long total_bases = *total;
    const int any = p.target_bases_set || p.keep_percent_set;
    long long target = 0;
    if (any) {
        target = p.target_bases_set ? (long long)p.target_bases : 0x7FFFFFFFFFFFFFFFll;             // main.cpp:229-232
        if (p.keep_percent_set) {
            const long long keep_target = (long long)((p.keep_percent / 100.0) * (double)total_bases);   // main.cpp:235
            if (keep_target < target) target = keep_target;
        }
    }
    s.target = target;
    s.total_bases = total_bases;
    s.passed_bases = (long long)sums4[2];
    if (!any) s.status = 0;
    else if (target >= total_bases) s.status = 1;                            // main.cpp:239-240
    else if (target >= s.passed_bases) s.status = 2;                         // main.cpp:242-243
    else s.status = 3;
    s.active = s.status == 3 && target > 0;     // target <= 0: nothing to resolve, the cut keeps no row
    *st = s;
}

struct WideHistArgs {
    size_t n;
    const unsigned long long *key;
    const int32_t *start, *end;
    const uint8_t *passed;
    const SelectState *st;
    int shift, width, first;      // digit = (key >> shift) & ((1 << width) - 1); rows must match st->prefix above it
    unsigned long long *hist;     // [FL_SELECT_BINS], zeroed
};

__global__ void __launch_bounds__(256) k_select_hist_wide(WideHistArgs a) {
    extern __shared__ unsigned long long hw[];
    for (int i = threadIdx.x; i < FL_SELECT_BINS; i += blockDim.x) hw[i] = 0ull;
    __syncthreads();
    if (!a.st->active) return;
    const unsigned long long prefix = a.st->prefix;
    const unsigned long long dmask = (1ull << a.width) - 1ull;
    const int up = a.shift + a.width;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x) {
        if (!a.passed[i]) continue;
        const unsigned long long k = a.key[i];
        if (!a.first && (k >> up) != prefix) continue;
        atomicAdd(&hw[(k >> a.shift) & dmask], (unsigned long long)(a.end[i] - a.start[i]));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < FL_SELECT_BINS; i += blockDim.x)
        if (hw[i]) atomicAdd(&a.hist[i], hw[i]);
}

// one block of 1024 threads, 8 bins each: first non-empty bin whose inclusive prefix reaches the target
__global__ void __launch_bounds__(1024) k_select_pick_wide(SelectState *st, const unsigned long long *hist, int width, int last) {
    __shared__ unsigned long long wsum[32];
    __shared__ int s_pick, s_lastne;
    __shared__ unsigned long long s_before_pick;
    if (!st->active) return;
    const int nb = 1 << width;
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long c[8], s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int d = (int)threadIdx.x * 8 + i;
        c[i] = d < nb ? hist[d] : 0ull;
        s += c[i];
    }
    unsigned long long incl = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (unsigned)d) incl += t;
    }
    if (lane == 31) wsum[wid] = incl;
    if (threadIdx.x == 0) { s_pick = 0x7FFFFFFF; s_lastne = -1; }
    __syncthreads();
    if (wid == 0) {
        unsigned long long v = wsum[lane], iv = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, iv, d);
            if (lane >= (unsigned)d) iv += t;
        }
        wsum[lane] = iv - v;
    }
    __syncthreads();
    const unsigned long long base = st->cum_before, target = (unsigned long long)st->target;
    unsigned long long cum = base + wsum[wid] + (incl - s);
    int my_pick = 0x7FFFFFFF, my_last = -1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int d = (int)threadIdx.x * 8 + i;
        if (c[i]) {
            my_last = d;
            if (my_pick == 0x7FFFFFFF && cum + c[i] >= target) my_pick = d;
        }
        cum += c[i];
    }
    if (my_pick != 0x7FFFFFFF) atomicMin(&s_pick, my_pick);
    if (my_last >= 0) atomicMax(&s_lastne, my_last);
    __syncthreads();
    // the owner of the picked (or, if none reaches the target, the last non-empty) bin publishes its prefix
    int pick = s_pick != 0x7FFFFFFF ? s_pick : (s_lastne < 0 ? 0 : s_lastne);
    cum = base + wsum[wid] + (incl - s);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int d = (int)threadIdx.x * 8 + i;
        if (d == pick) { s_before_pick = cum; }
        cum += c[i];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        st->cum_before = s_before_pick;
        st->prefix = (st->prefix << width) | (unsigned long long)pick;
        if (last) {
            st->tie_key = st->prefix;
            st->tie_base = target > st->cum_before ? target - st->cum_before : 0ull;
        }
    }
}

__global__ void k_copy_u64(const unsigned long long *src, unsigned long long *dst) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *dst = *src;
}

}  // namespace

static RowsView rows_view(fl_ctx *c) {
    RowsView v{};
    v.n = c->n_rows;
    v.start = c->w_start.p; v.end = c->w_end.p; v.mean = c->w_mean.p; v.window = c->w_window.p; v.passed = c->w_passed.p;
    v.excl = c->contam.n > 0 ? c->w_excl.p : nullptr;
    return v;
}

static int ensure_final_buffers(fl_ctx *c) {
    size_t n = c->n_rows;
    cudaStream_t s = c->stream;
    FL_CUDA(c, c->w_nmean.reserve(n, 0, s));
    FL_CUDA(c, c->w_nwindow.reserve(n, 0, s));
    FL_CUDA(c, c->w_final.reserve(n, 0, s));
    FL_CUDA(c, c->w_key.reserve(n, 0, s));
    FL_CUDA(c, c->w_pfinal.reserve(n, 0, s));
    FL_CUDA(c, c->sc_f64.reserve((size_t)RED_BLOCKS * 6, 0, s));
    if (!c->d_sel) FL_CUDA(c, cudaMalloc(&c->d_sel, sizeof(SelectState)));
    if (!c->d_norm) FL_CUDA(c, cudaMalloc(&c->d_norm, 16 * sizeof(double)));
    if (!c->d_hist) FL_CUDA(c, cudaMalloc(&c->d_hist, (256 + 64) * sizeof(unsigned long long)));
    return FL_OK;
}

static int red_blocks(fl_ctx *c) {
    size_t nb = (c->n_rows + RED_THREADS * 4 - 1) / (RED_THREADS * 4);
    if (nb < 1) nb = 1;
    if (nb > RED_BLOCKS) nb = RED_BLOCKS;
    return (int)nb;
}

extern "C" int fl_norm_partial1(fl_ctx *ctx, double *dev_sums4, double *dev_min1, double *dev_max1) {
    if (!ctx || !dev_sums4 || !dev_min1 || !dev_max1) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_TRY(ensure_final_buffers(ctx));
    int nb = red_blocks(ctx);
    k_norm_p1<<<nb, RED_THREADS, 0, ctx->stream>>>(rows_view(ctx), ctx->sc_f64.p);
    k_norm_p1_final<<<1, RED_THREADS, 0, ctx->stream>>>(ctx->sc_f64.p, nb, dev_sums4, dev_min1, dev_max1);
    ctx->launches += 2;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

extern "C" int fl_norm_partial2(fl_ctx *ctx, const double *dev_sums4, const double *, const double *, double *dev_sq1) {
    if (!ctx || !dev_sums4 || !dev_sq1) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_TRY(ensure_final_buffers(ctx));
    int nb = red_blocks(ctx);
    k_norm_p2<<<nb, RED_THREADS, 0, ctx->stream>>>(rows_view(ctx), dev_sums4, ctx->sc_f64.p);
    k_sum_partials<<<1, RED_THREADS, 0, ctx->stream>>>(ctx->sc_f64.p, nb, dev_sq1);
    ctx->launches += 2;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

extern "C" int fl_norm_apply(fl_ctx *ctx, const double *dev_sums4, const double *dev_min1, const double *dev_max1,
                             const double *dev_sq1) {
    if (!ctx || !dev_sums4 || !dev_min1 || !dev_max1 || !dev_sq1) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_TRY(ensure_final_buffers(ctx));
    if (ctx->n_rows == 0) return FL_OK;
    ApplyArgs a{};
    a.v = rows_view(ctx);
    a.sums4 = dev_sums4; a.min1 = dev_min1; a.max1 = dev_max1; a.sq1 = dev_sq1;
    a.lw = ctx->p.length_weight; a.mw = ctx->p.mean_q_weight; a.ww = ctx->p.window_q_weight;
    a.nmean = ctx->w_nmean.p; a.nwindow = ctx->w_nwindow.p; a.fscore = ctx->w_final.p; a.key = ctx->w_key.p;
    a.pfinal = ctx->w_pfinal.p;
    unsigned blocks = fl_blocks(ctx->n_rows, 256);
    if (blocks > (unsigned)ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    k_norm_apply<<<blocks, 256, 0, ctx->stream>>>(a);
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

static long long compute_target(const fl_params &p, long long total_bases) {
    long long target = p.target_bases_set ? (long long)p.target_bases : INT64_MAX;     // main.cpp:229-232
    if (p.keep_percent_set) {
        long long keep_target = (long long)((p.keep_percent / 100.0) * (double)total_bases);   // main.cpp:235
        if (keep_target < target) target = keep_target;
    }
    return target;
}

extern "C" int fl_select_begin(fl_ctx *ctx, int64_t total_bases_global, const double *dev_sums4) {
    if (!ctx || !dev_sums4) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_TRY(ensure_final_buffers(ctx));
    const int any = ctx->p.target_bases_set || ctx->p.keep_percent_set;
    long long target = any ? compute_target(ctx->p, total_bases_global) : 0;
    k_select_begin<<<1, 1, 0, ctx->stream>>>(ctx->d_sel, dev_sums4, target, total_bases_global, any);
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

extern "C" int fl_select_hist(fl_ctx *ctx, int level, uint64_t *dev_hist256) {
    if (!ctx || !dev_hist256 || level < 0 || level > 7) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_CUDA(ctx, cudaMemsetAsync(dev_hist256, 0, 256 * sizeof(uint64_t), ctx->stream));
    if (ctx->n_rows == 0) return FL_OK;
    HistArgs a{};
    a.n = ctx->n_rows; a.key = ctx->w_key.p; a.start = ctx->w_start.p; a.end = ctx->w_end.p;
    a.passed = ctx->w_passed.p; a.st = ctx->d_sel; a.level = level;
    a.hist = reinterpret_cast<unsigned long long *>(dev_hist256);
    unsigned blocks = fl_blocks(ctx->n_rows, 256 * 8);
    if (blocks > (unsigned)ctx->sm_count * 4) blocks = ctx->sm_count * 4;
    k_select_hist<<<blocks, 256, 0, ctx->stream>>>(a);
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

extern "C" int fl_select_pick(fl_ctx *ctx, int level, const uint64_t *dev_hist256) {
    if (!ctx || !dev_hist256 || level < 0 || level > 7) return FL_EINVAL;
    FL_ENTER(ctx);
    k_select_pick<<<1, 1, 0, ctx->stream>>>(ctx->d_sel, reinterpret_cast<const unsigned long long *>(dev_hist256), level);
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

extern "C" int fl_select_tie_local(fl_ctx *ctx, uint64_t *dev_tie_per_rank, int rank, int nranks) {
    if (!ctx || !dev_tie_per_rank || rank < 0 || rank >= nranks) return FL_EINVAL;
    FL_ENTER(ctx);
    size_t n = ctx->n_rows;
    FL_CUDA(ctx, ctx->sc_u64a.reserve(n + 1, 0, ctx->stream));
    FL_CUDA(ctx, ctx->sc_u64b.reserve(n + 1, 0, ctx->stream));
    unsigned long long *total = ctx->d_scalars + 8;
    if (n) {
        TieArgs a{};
        a.n = n; a.key = ctx->w_key.p; a.start = ctx->w_start.p; a.end = ctx->w_end.p; a.passed = ctx->w_passed.p;
        a.st = ctx->d_sel; a.tie_len = ctx->sc_u64a.p;
        unsigned blocks = fl_blocks(n, 256);
        if (blocks > (unsigned)ctx->sm_count * 8) blocks = ctx->sm_count * 8;
        k_tie_len<<<blocks, 256, 0, ctx->stream>>>(a);
        ctx->launches++;
    }
    FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64a.p, ctx->sc_u64b.p, n, total));
    k_store_tie_total<<<1, 1, 0, ctx->stream>>>(total, reinterpret_cast<unsigned long long *>(dev_tie_per_rank), rank, nranks);
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

extern "C" int fl_select_apply(fl_ctx *ctx, const uint64_t *dev_tie_per_rank, int rank, uint64_t *dev_keeping1) {
    if (!ctx || !dev_tie_per_rank || !dev_keeping1) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_CUDA(ctx, cudaMemsetAsync(dev_keeping1, 0, sizeof(uint64_t), ctx->stream));
    if (ctx->n_rows) {
        CutArgs a{};
        a.n = ctx->n_rows; a.key = ctx->w_key.p; a.start = ctx->w_start.p; a.end = ctx->w_end.p;
        a.passed = ctx->w_passed.p; a.st = ctx->d_sel; a.tie_excl = ctx->sc_u64b.p;
        a.tie_per_rank = reinterpret_cast<const unsigned long long *>(dev_tie_per_rank); a.rank = rank;
        a.pfinal = ctx->w_pfinal.p; a.keeping = reinterpret_cast<unsigned long long *>(dev_keeping1);
        // rows keep pfinal == passed (written by fl_norm_apply) unless status == 3; the kernel
        // checks st->status itself so that no host round trip is needed
        unsigned blocks = fl_blocks(ctx->n_rows, 256);
        if (blocks > (unsigned)ctx->sm_count * 8) blocks = ctx->sm_count * 8;
        k_select_cut<<<blocks, 256, 0, ctx->stream>>>(a);
        ctx->launches++;
        FL_CUDA(ctx, cudaGetLastError());
    }
    ctx->finalized = true;
    return FL_OK;
}

extern "C" int fl_select_summary(fl_ctx *ctx, const double *dev_sums4, const double *dev_min1, const double *dev_max1,
                                 const double *dev_sq1, const uint64_t *dev_keeping1, int64_t total_bases_global,
                                 fl_summary *out) {
    if (!ctx || !out) return FL_EINVAL;
    FL_ENTER(ctx);
    double h[8] = {0};
    unsigned long long keeping = 0;
    SelectState st{};
    FL_CUDA(ctx, cudaMemcpyAsync(h, dev_sums4, 4 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaMemcpyAsync(h + 4, dev_min1, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaMemcpyAsync(h + 5, dev_max1, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaMemcpyAsync(h + 6, dev_sq1, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaMemcpyAsync(&keeping, dev_keeping1, sizeof(keeping), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaMemcpyAsync(&st, ctx->d_sel, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memset(out, 0, sizeof(*out));
    const double n = h[0], mean = h[1] / n, sd = sqrt(h[6] / n);
    out->min_q = h[4]; out->max_q = h[5]; out->mean_q = mean; out->stdev_q = sd;
    if (sd > 0.0) { out->min_z = (h[4] - mean) / sd; out->max_z = (h[5] - mean) / sd; }
    else { out->min_z = 1.0; out->max_z = 1.0; }
    out->status = st.status;
    out->target = st.target;
    out->passed_bases = (int64_t)h[2];
    out->rows_bases = (int64_t)h[3];
    out->total_bases = total_bases_global;
    out->keeping = st.status == 3 ? (int64_t)keeping : 0;
    return FL_OK;
}

extern "C" int fl_finalize(fl_ctx *ctx, int64_t total_bases, fl_summary *out) {
    FL_ENTER(ctx);
    FL_TRY(ensure_final_buffers(ctx));
    if (ctx->comm_nranks > FL_COMM_MAX_RANKS) { ctx->set_error("fl_finalize: too many ranks"); return FL_ERANGE; }
    if (!ctx->d_comm) FL_CUDA(ctx, cudaMalloc(&ctx->d_comm, FL_COMM_SCRATCH_BYTES));
    if (!ctx->select_attr_set) {
        FL_CUDA(ctx, cudaFuncSetAttribute(k_select_hist_wide, cudaFuncAttributeMaxDynamicSharedMemorySize, FL_SELECT_BINS * 8));
        ctx->select_attr_set = true;
    }
    cudaStream_t st = ctx->stream;
    CommScratch *cs = reinterpret_cast<CommScratch *>(ctx->d_comm);
    double *sums = ctx->d_norm, *mn = ctx->d_norm + 4, *mx = ctx->d_norm + 5, *sq = ctx->d_norm + 6;
    const int nranks = ctx->comm_nranks, rank = ctx->comm_rank;
    const size_t n = ctx->n_rows;
    // ---- statistics (main.cpp:170-196): local partials, one all-gather each, combined in rank order ----
    FL_TRY(fl_norm_partial1(ctx, sums, mn, mx));
    {
        const bool own = total_bases < 0;                 // the context's own count: host pushes + device pushes
        k_stats_send<<<1, 1, 0, st>>>(sums, mn, mx, own ? ctx->d_scalars + 16 : nullptr, own ? (long long)ctx->total_bases : (long long)total_bases,
                                      cs->stats_send);
        ctx->launches++;
    }
    FL_TRY(fl_comm_allgather(ctx, cs->stats_send, cs->stats_recv, 8 * sizeof(double)));
    k_stats_combine<<<1, 1, 0, st>>>(cs->stats_recv, nranks, sums, mn, mx, cs->total_bases);
    ctx->launches++;
    FL_TRY(fl_norm_partial2(ctx, sums, mn, mx, cs->sq_send));
    FL_TRY(fl_comm_allgather(ctx, cs->sq_send, cs->sq_recv, sizeof(double)));
    k_sq_combine<<<1, 1, 0, st>>>(cs->sq_recv, nranks, sq);
    ctx->launches++;
    FL_TRY(fl_norm_apply(ctx, sums, mn, mx, sq));                                   // main.cpp:202-212
    // ---- target + weighted radix select of the cut-off key (main.cpp:218-257) ----
    k_select_begin_dev<<<1, 1, 0, st>>>(ctx->d_sel, sums, cs->total_bases, ctx->p);
    ctx->launches++;
    const bool any_target = ctx->p.target_bases_set || ctx->p.keep_percent_set;
    if (any_target) {
        int done = 0;
        while (done < 64) {
            const int width = 64 - done < FL_SELECT_DIGIT_BITS ? 64 - done : FL_SELECT_DIGIT_BITS;
            const int shift = 64 - done - width;
            FL_CUDA(ctx, cudaMemsetAsync(cs->hist, 0, sizeof(cs->hist), st));
            if (n) {
                WideHistArgs a{};
                a.n = n; a.key = ctx->w_key.p; a.start = ctx->w_start.p; a.end = ctx->w_end.p; a.passed = ctx->w_passed.p;
                a.st = ctx->d_sel; a.shift = shift; a.width = width; a.first = done == 0; a.hist = cs->hist;
                unsigned blocks = fl_blocks(n, 256 * 16);
                if (blocks > (unsigned)ctx->sm_count * 2) blocks = (unsigned)ctx->sm_count * 2;
                if (blocks < 1) blocks = 1;
                k_select_hist_wide<<<blocks, 256, FL_SELECT_BINS * 8, st>>>(a);
                ctx->launches++;
            }
            FL_TRY(fl_comm_allreduce_u64(ctx, cs->hist, (size_t)1 << width));
            k_select_pick_wide<<<1, 1024, 0, st>>>(ctx->d_sel, cs->hist, width, shift == 0);
            ctx->launches++;
            done += width;
        }
        // tie class at the cut-off, in (rank, row) order
        FL_CUDA(ctx, ctx->sc_u64a.reserve(n + 1, 0, st));
        FL_CUDA(ctx, ctx->sc_u64b.reserve(n + 1, 0, st));
        if (n) {
            TieArgs a{};
            a.n = n; a.key = ctx->w_key.p; a.start = ctx->w_start.p; a.end = ctx->w_end.p; a.passed = ctx->w_passed.p;
            a.st = ctx->d_sel; a.tie_len = ctx->sc_u64a.p;
            unsigned blocks = fl_blocks(n, 256);
            if (blocks > (unsigned)ctx->sm_count * 8) blocks = ctx->sm_count * 8;
            k_tie_len<<<blocks, 256, 0, st>>>(a);
            ctx->launches++;
        }
        FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64a.p, ctx->sc_u64b.p, n, cs->tie_send));
        FL_TRY(fl_comm_allgather(ctx, cs->tie_send, cs->tie_recv, sizeof(unsigned long long)));
    } else {
        FL_CUDA(ctx, cudaMemsetAsync(cs->tie_recv, 0, sizeof(cs->tie_recv), st));
    }
    FL_TRY(fl_select_apply(ctx, reinterpret_cast<const uint64_t *>(cs->tie_recv), rank, reinterpret_cast<uint64_t *>(cs->keeping)));
    FL_TRY(fl_comm_allreduce_u64(ctx, cs->keeping, 1));
    FL_CUDA(ctx, cudaGetLastError());
    if (out) {
        long long total = 0;
        FL_CUDA(ctx, cudaMemcpyAsync(&total, cs->total_bases, sizeof(total), cudaMemcpyDeviceToHost, st));
        FL_TRY(fl_select_summary(ctx, sums, mn, mx, sq, reinterpret_cast<const uint64_t *>(cs->keeping), -1, out));
        out->total_bases = total;
    }
    return FL_OK;
}

int fl_norm_select_free(fl_ctx *ctx) {
    if (ctx->d_sel) cudaFree(ctx->d_sel);
    if (ctx->d_norm) cudaFree(ctx->d_norm);
    if (ctx->d_hist) cudaFree(ctx->d_hist);
    ctx->d_sel = nullptr; ctx->d_norm = nullptr; ctx->d_hist = nullptr;
    return FL_OK;
}

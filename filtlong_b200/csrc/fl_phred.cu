// filtlong_b200/csrc/fl_phred.cu -- Phred-mode scoring (reference src/read.cpp:35-39, 208-236, 270-273).
//
// The reference's mean and window quality are defined by strictly sequential double additions:
//     sum += q[c_j]                                   (read.cpp:208-213)
//     w -= a[c_{j-ws}];  w += a[c_j];  min = min(min, w)   (read.cpp:226-232)
// with q[c] = 1 - 10^(-(c-33)/10) and a[c] = q[c] / window_size. Their low-order bits depend on that
// order, and hard thresholds (--min_mean_q / --min_window_q) compare them, so every path in this file
// returns the reference's bits (file built with --fmad=false, q[] / a[] are 256-entry tables evaluated
// with the host libm and replicated in shared memory so that each lane owns its banks).
//
// Two implementations:
//   * DEFAULT (window sizes 16..256): k_phred_first + k_phred_sum + k_phred_win, one warp per read,
//     exact lattice arithmetic inside binades -- see the comment block above k_phred_first.
//   * Work items (FL_PHRED_MODE=0, and every other window size), described next. Also the home of
//     k_phred_fallback, the reference's loop verbatim, which re-scores whatever a fast path rejects.
//
// Work-item decomposition:
//   * reads up to PH_LONG bases: one work item, the fused loop (sum and window together);
//   * longer reads: one item for the mean chain plus one item per PH_SEG-base SEGMENT of the window
//     chain. A segment needs the exact value of w at its first base. It is obtained WITHOUT running
//     the chain: while w stays inside one binade [2^e, 2^(e+1)) every add / subtract of a[c] moves
//     it by exactly rint(a[c] / ulp_e) grid steps (no rounding drift), so
//         w_P = W_0 + ulp_e * (S(P) - S(ws)),   S(x) = sum of rint(a[c]/ulp_e) over the ws bases before x,
//     which costs 2*ws look-ups. This is only a PREDICTION: every segment then runs the true
//     sequential recurrence from its predicted entry, and k_phred_merge accepts a read only if each
//     segment's exit value equals the next segment's predicted entry bit-for-bit (induction from
//     the exact first window). A read that fails the check (binade crossing, round-to-even tie) is
//     re-scored by the plain fused loop;
//   * items are issued in descending cost order over a persistent grid.
#include "fl_device.cuh"

namespace {

#define PH_THREADS 256
#define PH_SMEM (256 * 8 * 16 + 256 * 16 * 8)   // {q,a} x 8 copies + a x 16 copies = 64 KiB
#define PH_SEG 16384
#define PH_LONG (PH_SEG + PH_SEG / 2)

#define ITEM_FUSED 0xFFFFFFFFu
#define ITEM_MEAN 0xFFFFFFFEu

struct Tab {
    const double2 *tqa;   // [c*8]  -> {q[c], a[c]}, lane-private 16-byte bank group
    const double *ta;     // [c*16] -> a[c],         lane-private 8-byte bank pair
};

struct PhredArgs {
    const uint8_t *qual;
    const uint64_t *off;
    const int32_t *len;
    uint32_t n;
    const double *lut;          // [512]
    fl_params p;
    // outputs, already offset to this batch's first read / row (or the view's first item: phred_args_of)
    int32_t *r_len, *r_first, *r_last, *r_nbad, *r_nchild;
    double *r_mean, *r_window;
    uint8_t *r_passed;
    unsigned long long *r_rowstart;
    uint32_t *w_parent;
    int32_t *w_start, *w_end;
    double *w_mean, *w_window;
    uint8_t *w_passed;
    unsigned long long read_base, row_base;
    // work items
    const unsigned long long *item_start;   // [n+1] exclusive scan of items per read
    const uint32_t *order;                  // item indices, descending cost
    const uint2 *items;                     // {read, kind}
    unsigned long long n_items;
    double *it_a, *it_b, *it_c;             // per item: MEAN: sum | SEG: entry, exit, best
    uint32_t *fallback;                     // [0] = count, [1..] = reads to re-score serially
    unsigned long long *work;               // [0], [1]: next read (in `order`) for k_phred_sum / k_phred_win
    unsigned long long *phred_paths;        // k_phred_win's path counters (PW_COUNTERS, accumulated over the context's life)
    int head_len;                          // k_phred_first: bases whose sum the per-read first pass takes
};

__device__ __forceinline__ unsigned byte_of(uint32_t w, int i) { return (w >> (8 * i)) & 0xFFu; }

template <int WI>
__device__ __forceinline__ void out_words(const uint4 &a, const uint4 &b, unsigned sh, uint32_t ow[4]) {
    const uint32_t c[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) ow[k] = __funnelshift_r(c[WI + k], c[WI + k + 1], sh);
}

template <bool DO_SUM, bool DO_WIN>
__device__ __forceinline__ void step(unsigned cin, unsigned cout, const Tab &t, double &sum, double &w, double &best) {
    if (DO_SUM && DO_WIN) {
        const double2 qa = t.tqa[cin * 8];
        const double ao = t.ta[cout * 16];
        sum += qa.x;                 // read.cpp:210-211
        w -= ao;                     // read.cpp:229
        w += qa.y;                   // read.cpp:230
        if (w < best) best = w;      // read.cpp:231-232
    } else if (DO_SUM) {
        sum += t.tqa[cin * 8].x;
    } else {
        const double ai = t.ta[cin * 16];
        const double ao = t.ta[cout * 16];
        w -= ao;
        w += ai;
        if (w < best) best = w;
    }
}

// Walks bases [jlo, jhi) of one read in order. DO_WIN requires jlo >= ws.
template <bool DO_SUM, bool DO_WIN>
__device__ __forceinline__ void chain(const uint8_t *__restrict__ q, int jlo, int jhi, int ws, const Tab &t, double &sum,
                                      double &w, double &best) {
    int j = jlo;
    for (; (j & 15) && j < jhi; ++j) step<DO_SUM, DO_WIN>(q[j], DO_WIN ? q[j - ws] : 0u, t, sum, w, best);
    if (j + 16 <= jhi) {
        const uint4 *qv = reinterpret_cast<const uint4 *>(q);
        const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
        int blk = 0;
        unsigned sh = 0, wi = 0;
        uint4 oa = zero, ob = zero;
        if (DO_WIN) {
            const int i0 = j - ws;                     // >= 0; (i0 & 15) is the same for every 16-byte step
            blk = i0 >> 4;
            sh = ((unsigned)i0 & 3u) * 8u;
            wi = ((unsigned)i0 & 15u) >> 2;
            oa = __ldg(qv + blk);
            ob = __ldg(qv + blk + 1);                  // never beyond the block of base j (see DESIGN.md)
        }
        uint4 in = __ldg(qv + (j >> 4));
        while (j + 16 <= jhi) {
            const bool more = j + 32 <= jhi;
            // next step's loads are issued before this step's dependent chains (software prefetch)
            const uint4 in_next = more ? __ldg(qv + (j >> 4) + 1) : zero;
            const uint4 oc = (DO_WIN && more) ? __ldg(qv + blk + 2) : zero;
            uint32_t ow[4] = {0u, 0u, 0u, 0u};
            if (DO_WIN) {
                switch (wi) {
                    case 0: out_words<0>(oa, ob, sh, ow); break;
                    case 1: out_words<1>(oa, ob, sh, ow); break;
                    case 2: out_words<2>(oa, ob, sh, ow); break;
                    default: out_words<3>(oa, ob, sh, ow); break;
                }
            }
            const uint32_t iw[4] = {in.x, in.y, in.z, in.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int b = 0; b < 4; ++b)
                    step<DO_SUM, DO_WIN>(byte_of(iw[k], b), byte_of(ow[k], b), t, sum, w, best);
            in = in_next;
            oa = ob;
            ob = oc;
            ++blk;
            j += 16;
        }
    }
    for (; j < jhi; ++j) step<DO_SUM, DO_WIN>(q[j], DO_WIN ? q[j - ws] : 0u, t, sum, w, best);
}

__device__ __forceinline__ void write_read(const PhredArgs &a, uint32_t r, int L, double mean, double window) {
    const uint8_t passed = fl_hard_cutoffs(a.p, L, mean, window);
    a.r_len[r] = L;
    a.r_mean[r] = mean;
    a.r_window[r] = window;
    a.r_passed[r] = passed;
    a.r_first[r] = -1;                               // read.cpp:75-76 (only set in k-mer mode)
    a.r_last[r] = -1;
    a.r_nbad[r] = 0;
    a.r_nchild[r] = 0;
    a.r_rowstart[r] = a.row_base + r;
    a.w_parent[r] = (uint32_t)(a.read_base + r);
    a.w_start[r] = 0;
    a.w_end[r] = L;
    a.w_mean[r] = mean;
    a.w_window[r] = window;
    a.w_passed[r] = passed;
}

__device__ __forceinline__ void finish(const PhredArgs &a, uint32_t r, int L, double sum, double best) {
    const double wsd = (double)a.p.window_size;
    if (best < 0.5 / wsd) best = 0.0;                // read.cpp:233-234
    write_read(a, r, L, 100.0 * sum / (double)L, 100.0 * best);
}

// the whole read by one thread: read.cpp:208-236 verbatim
__device__ __forceinline__ void score_fused(const PhredArgs &a, uint32_t r, const Tab &t) {
    const int L = a.len[r], ws = a.p.window_size;
    const uint8_t *q = a.qual + a.off[r];
    double sum = 0.0, w = 0.0, best = 0.0;
    chain<true, false>(q, 0, L < ws ? L : ws, ws, t, sum, w, best);
    if (L <= ws) {                                   // read.cpp:217-218
        const double mean = 100.0 * sum / (double)L;
        write_read(a, r, L, mean, mean);
        return;
    }
    w = sum / (double)ws;                            // read.cpp:223
    best = w;
    chain<true, true>(q, ws, L, ws, t, sum, w, best);
    finish(a, r, L, sum, best);
}

// Window sizes reach 2^31 - 1, so sums like ws + PH_SEG can wrap in int: these are written as differences, which cannot
// (L >= 0, ws > 0). A segmented read has L - ws > PH_SEG.
__device__ __forceinline__ int n_segments(int L, int ws) { return (L - ws - 1) / PH_SEG + 1; }

__device__ __forceinline__ unsigned long long items_of(int L, int ws) {
    if (L <= PH_LONG || L - ws <= PH_SEG) return 1ull;
    return 1ull + (unsigned long long)n_segments(L, ws);
}

// end of the segment that starts at P < L
__device__ __forceinline__ int segment_end(int P, int L) { return (L - P > PH_SEG) ? P + PH_SEG : L; }

// one segment of the window chain of a long read, from a predicted entry value
__device__ __forceinline__ void score_segment(const PhredArgs &a, uint32_t r, int seg, size_t idx, const Tab &t) {
    const int L = a.len[r], ws = a.p.window_size;
    const uint8_t *q = a.qual + a.off[r];
    double sum = 0.0, w = 0.0, best = 0.0;
    chain<true, false>(q, 0, ws, ws, t, sum, w, best);
    const double w0 = sum / (double)ws;              // exact first window (read.cpp:220-223)
    const int P = ws + seg * PH_SEG;                 // < L: no wrap
    const int Pend = segment_end(P, L);
    double entry = w0;
    if (seg > 0) {
        // prediction: grid steps of w inside the binade of w0 (see the file header)
        int e = 0;
        (void)frexp(w0, &e);                         // w0 = m * 2^e, m in [0.5, 1): binade exponent e - 1
        const double scale = ldexp(1.0, 53 - e);     // 1 / ulp of that binade
        long long s0 = 0, sp = 0;
        for (int i = 0; i < ws; ++i) {
            s0 += __double2ll_rn(t.ta[(unsigned)q[i] * 16] * scale);
            sp += __double2ll_rn(t.ta[(unsigned)q[P - ws + i] * 16] * scale);
        }
        entry = w0 + (double)(sp - s0) / scale;
    }
    w = entry;
    best = __longlong_as_double(0x7FF0000000000000ll);   // +inf: only values produced inside the segment count
    chain<false, true>(q, P, Pend, ws, t, sum, w, best);
    a.it_a[idx] = entry;
    a.it_b[idx] = w;
    a.it_c[idx] = best;
}

__device__ __forceinline__ Tab make_tables(const double *lut, unsigned char *smem_raw) {
    double2 *tqa_all = reinterpret_cast<double2 *>(smem_raw);                       // [256][8]
    double *ta_all = reinterpret_cast<double *>(smem_raw + 256 * 8 * 16);           // [256][16]
    for (int i = threadIdx.x; i < 256 * 8; i += blockDim.x) {
        const int c = i >> 3;
        tqa_all[i] = make_double2(lut[c], lut[256 + c]);
    }
    for (int i = threadIdx.x; i < 256 * 16; i += blockDim.x) ta_all[i] = lut[256 + (i >> 4)];
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    Tab t;
    t.tqa = tqa_all + (lane & 7);
    t.ta = ta_all + (lane & 15);
    return t;
}

__global__ void __launch_bounds__(PH_THREADS, 3) k_phred_items(PhredArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const Tab t = make_tables(a.lut, smem_raw);
    const size_t T = (size_t)gridDim.x * blockDim.x;
    for (size_t it = (size_t)blockIdx.x * blockDim.x + threadIdx.x; it < a.n_items; it += T) {
        const size_t idx = a.order[it];
        const uint2 item = a.items[idx];
        const uint32_t r = item.x;
        if (item.y == ITEM_FUSED) {
            score_fused(a, r, t);
        } else if (item.y == ITEM_MEAN) {
            continue;                                // the mean chain of a long read is k_phred_mean_long's job
        } else {
            score_segment(a, r, (int)item.y, idx, t);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Mean chain of a LONG read, one warp per read, exact without walking it serially.
//
// The reference's sum (read.cpp:208-213) is s <- fl(s + q[c_j]) left to right. While s stays in one
// binade [2^e, 2^(e+1)) it is a multiple of ulp_e = 2^(e-52), and for 0 <= q < 1 (IEEE-754 RN)
//     fl(s + q) = s + r(q),   r(q) = q rounded to a multiple of ulp_e,
// unless q sits exactly half way between two multiples (tie: the result then depends on the parity
// of s). r(q) itself is one add and one subtract of the constant C = 2^e (C + q stays in the binade
// for e >= 9), and q - r(q) is exact, so a tie is |q - r(q)| == ulp_e / 2. All r(q) of a tile are
// multiples of ulp_e below 1, their sum D < 2048 <= 2^(e+1) is exact in ANY order, and s + D is exact
// as long as it stays below 2^(e+1). So a warp adds 2048 bases per step -- 64 per lane, one table
// gather and four double ops per base, one shuffle reduction -- and only a step that (a) carries s
// into the next binade, (b) contains a tie or a byte outside the Phred range, or (c) starts below
// 2^11 is redone by lane 0 with the reference's own sequential adds. Those steps are a few dozen per
// read; every other step is exact by the identity above (no speculation involved).
// ---------------------------------------------------------------------------------------------
#define PH_MEAN_SMEM (256 * 16 * 8)
#define PH_MEAN_TILE 2048

__device__ __forceinline__ double serial_tile(const uint8_t *__restrict__ q, int lo, int hi, const double *__restrict__ qtab,
                                              double s) {
    for (int j = lo; j < hi; ++j) s += __ldg(qtab + (unsigned)q[j]);     // true table (global), rare path
    return s;
}

__global__ void __launch_bounds__(256) k_phred_mean_long(PhredArgs a, unsigned long long tie_binades) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *qtab_all = reinterpret_cast<double *>(smem_raw);                               // [256][16]
    // grid-path table: a quality outside [0, 1) becomes NaN, which poisons the tile sum and sends the
    // tile to the serial path without any per-base range test
    for (int i = threadIdx.x; i < 256 * 16; i += blockDim.x) {
        const double v = a.lut[i >> 4];
        qtab_all[i] = (v >= 0.0 && v < 1.0) ? v : __longlong_as_double(0x7FF8000000000000ll);
    }
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const double *qtab = qtab_all + (lane & 15);                 // lane-private bank pair
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t r = warp; r < a.n; r += n_warps) {
        const size_t base = a.item_start[r];
        if (a.item_start[r + 1] - base <= 1) continue;           // short read: the fused item owns it
        const int L = a.len[r];
        const uint8_t *q = a.qual + a.off[r];
        const uint4 *qv = reinterpret_cast<const uint4 *>(q);
        double s = 0.0;
        int j = 0, small_left = 0;
        while (j < L) {
            int e = -2000;
            if (s > 0.0) {
                (void)frexp(s, &e);
                e -= 1;                                          // s in [2^e, 2^(e+1))
            }
            // tile size: the exact-sum argument needs (bases in the tile) <= 2^(e+1); after a failed
            // big tile the next 2048 bases are taken in 128-base pieces so that only the piece that
            // really carries / ties is walked serially
            const bool big = e >= 10 && e <= 1000 && small_left == 0;
            const bool lattice_ok = big || (e >= 6 && e <= 1000);
            const int T = big ? PH_MEAN_TILE : 128;
            const int hi = (j + T < L) ? j + T : L;
            bool done = false;
            if (lattice_ok) {
                const double C = ldexp(1.0, e), half_ulp = ldexp(1.0, e - 53);
                // a rounding tie needs a table value whose dropped bits are exactly 100..0 in this
                // binade; the host lists the binades where ANY Phred value does (none above 2^9 for
                // the default table), everywhere else the per-base tie test is skipped
                const bool check_ties = e < 64 && ((tie_binades >> e) & 1ull);
                double d = 0.0;
                unsigned bad = 0u;
#pragma unroll
                for (int c4 = 0; c4 < 4; ++c4) {                 // up to 4 coalesced 16-byte chunks per lane
                    const int lo = j + 512 * c4 + 16 * (int)lane;
                    if (lo < hi) {
                        const uint4 v = __ldg(qv + (lo >> 4));
                        const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
                        if (lo + 16 <= hi && !check_ties) {
#pragma unroll
                            for (int k = 0; k < 16; ++k) {
                                const double x = qtab[byte_of(wv[k >> 2], k & 3) * 16];
                                d += (C + x) - C;                // x rounded to the grid of the binade
                            }
                        } else {
#pragma unroll
                            for (int k = 0; k < 16; ++k) {
                                const double x = qtab[byte_of(wv[k >> 2], k & 3) * 16];
                                const double rq = (C + x) - C;
                                const bool in = lo + k < hi;
                                bad |= (in && fabs(x - rq) == half_ulp) ? 1u : 0u;   // x - rq is exact
                                d += in ? rq : 0.0;
                            }
                        }
                    }
                }
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    d += __shfl_xor_sync(0xffffffffu, d, o);      // exact: multiples of ulp_e, total < 2^(e+1)
                    bad |= __shfl_xor_sync(0xffffffffu, bad, o);
                }
                if (!bad) {
                    const double s_new = s + d;
                    if (s_new < C + C) { s = s_new; done = true; }
                }
            }
            if (!done) {
                if (big) { small_left = PH_MEAN_TILE / 128; continue; }   // retry this range in small pieces
                if (lane == 0) s = serial_tile(q, j, hi, a.lut, s);        // the reference's own loop
                s = __shfl_sync(0xffffffffu, s, 0);
            }
            if (small_left > 0) --small_left;
            j = hi;
        }
        if (lane == 0) a.it_a[base] = s;
    }
}

// long reads: check the chain of segments and combine (see the file header)
__global__ void __launch_bounds__(256) k_phred_merge(PhredArgs a) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.n) return;
    const size_t base = a.item_start[r];
    const int n_it = (int)(a.item_start[r + 1] - base);
    if (n_it <= 1) return;
    const int L = a.len[r];
    const double sum = a.it_a[base];
    double best = a.it_a[base + 1];                  // entry of segment 0 = exact first window
    bool ok = true;
    for (int k = 0; k < n_it - 1; ++k) {
        const size_t i = base + 1 + k;
        if (k > 0 && __double_as_longlong(a.it_a[i]) != __double_as_longlong(a.it_b[i - 1])) { ok = false; break; }
        const double b = a.it_c[i];
        if (b < best) best = b;
    }
    if (ok) finish(a, r, L, sum, best);
    else a.fallback[1 + atomicAdd(a.fallback, 1u)] = r;
}

__global__ void __launch_bounds__(PH_THREADS, 3) k_phred_fallback(PhredArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const uint32_t n = a.fallback[0];
    if (n == 0) return;
    const Tab t = make_tables(a.lut, smem_raw);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        score_fused(a, a.fallback[1 + i], t);
}

__global__ void k_phred_plan(const int32_t *__restrict__ len, uint32_t n, int ws, unsigned long long *__restrict__ n_items) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) n_items[r] = items_of(len[r], ws);
}

__global__ void k_phred_fill(const int32_t *__restrict__ len, uint32_t n, int ws, const unsigned long long *__restrict__ item_start,
                             uint2 *__restrict__ items, uint32_t *__restrict__ cost) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int L = len[r];
    const size_t base = item_start[r];
    const int cnt = (int)items_of(L, ws);
    if (cnt == 1) {
        items[base] = make_uint2(r, ITEM_FUSED);
        cost[base] = 0 * 256 + fl_length_bucket(L);
        return;
    }
    items[base] = make_uint2(r, ITEM_MEAN);
    cost[base] = 2 * 256 + fl_length_bucket(L);       // kinds are grouped so that warps stay uniform; the long serial chains go first
    for (int k = 0; k < cnt - 1; ++k) {
        items[base + 1 + k] = make_uint2(r, (uint32_t)k);
        const int P = ws + k * PH_SEG;
        const long long work = (long long)(segment_end(P, L) - P) + 2ll * ws;   // 2 * ws alone can pass INT_MAX
        cost[base + 1 + k] = 1 * 256 + fl_length_bucket(work < INT_MAX ? (int)work : INT_MAX);
    }
}

// ---------------------------------------------------------------------------------------------
// Default Phred path: three kernels, all exact, none walks a read base by base in one thread.
//   k_phred_first  one thread per read: the first window (sum, W0 = fl(sum / ws)) and the sum up to the
//                  next 16-byte boundary; reads not longer than the window are finished here.
//   k_phred_sum    one warp per read: the mean's sum, 512 bases per step.
//   k_phred_win    one warp per read: the window chain's minimum, one window length per step.
//
// Lattice identity (as in k_phred_mean_long): while a running double v stays inside one binade
// [C, 2C) it is a multiple of u = ulp(C), and for 0 <= t < C (IEEE RN, t not exactly half way between
// two multiples of u)      fl(v + t) = v + r(t),   fl(v - t) = v - r(t),   r(t) = t rounded to the grid u.
// So a chain is a sum of grid steps, exact in ANY order as long as every partial sum stays inside the
// binade; and inside one binade the BIT PATTERN of a double moves by one unit per grid step, so warp
// scans and reductions of grid steps are 64-bit integer adds.
//
// k_phred_sum: lane l adds its 16 bases to a lane-local acc that starts at C = 2^e, the binade of the
//   running sum s: acc = C + q + q + ... rounds every q to the grid of [C, 2C) exactly as s + q would
//   (the adder does r() for us). The lanes' parts are collected only when the room left in the binade
//   (2C - s; every base adds at most 1) could run out: O(log) warp reductions per binade. The step in
//   which s may cross into the next binade ("careful" step) is resolved exactly: integer scan of the
//   lanes' parts, the first lane whose prefix reaches 2C walks its 16 bases with true adds, the lanes
//   after it redo their parts on the coarser grid. In a binade in which a table value would tie (host
//   mask; only s < 1024 for the Phred table, one value each) a step first looks for that byte; a tie,
//   a NaN (bytes outside the Phred range are NaN in the warp's table) or anything unexpected sends
//   that one step to lane 0 and the reference's own loop.
//
// k_phred_win: step t covers bases [ws + t ws, ws + (t+1) ws); lane l owns K = ceil(ws/32)
//   consecutive bases of it, ALWAYS the same offsets, so the value that leaves the window when lane l
//   adds its k-th base is the value lane l added at its k-th base one step earlier. The whole read is
//   assumed to keep w inside [0.5, 1): upper side by construction (every table value is below
//   (1 - 1e-10)/ws, the first window W0 = fl(sum/ws) is within 1e-13 of the grid sum of its own values,
//   so every later grid value is below 1 - 4e-10), lower side CHECKED at the end: minimum - 2 max table
//   value >= 0.5 (the point after a subtraction is at most one table value below a point after an
//   addition). Inside [0.5, 1) every window value is W0 plus whole grid steps (2^-53):
//       bits(w_j) = bits(W0) + S_A(window j) - S_A(first window),   A_c = a[c] on the grid, as an integer,
//   so the minimum is the window with the least integer sum S_A. Two passes find it:
//   * filter pass, every step: the same lanes and steps on 32-bit filter values F_c = A_c >> 30 (A_c <
//     2^53/ws, so a window of F sums to < 2^23). Per base: byte extract, address, LDS.32 (32 lane-private
//     copies: one wavefront), x += now - old (the old values stay in registers), integer min; per step a
//     32-bit warp scan places the lanes (candidate = W + prefix + the lane's lowest prefix). Since
//     0 <= A_c - 2^30 F_c < 2^30, a window's S_A lies in [2^30 S_F, 2^30 (S_F + ws)): the true minimum can
//     only be at a window with S_F < m + ws, m the least S_F (first window included). Each lane keeps
//     its lowest candidate, the step where it was reached, and the lowest candidate of its other steps.
//   * exact pass: the lanes with a lowest candidate <= m + ws name their steps; each such step is walked
//     with the exact step code, entered at bits(W0) + S_A(the ws bases before it) - S_A(first window)
//     (ws grid look-ups and one warp reduction). If one of those lanes has another step within ws of its
//     lowest, the whole chain is walked exactly instead. Both use the grid table (a[c] rounded to the grid 2^-53 of
//     [0.5, 1)): x += new - old (exact), compare, from the anchor 0.75; a 64-bit warp scan places the
//     lanes. The first window W0 is always a candidate.
//   Table values that tie on the grid, or lie outside [0, 1), have the filter value 2^23: a window holding
//   one sums to >= 2^23 (and every sum stays below 2^32). A byte that enters the window in a step is still
//   in it at the step's last base, so one test of the running filter sum per step (and one of the first
//   window) rejects the read. A rejected read goes to k_phred_fallback (the reference's loop verbatim, one
//   thread). Counters of the paths taken: fl_ctx_phred_paths.
// ---------------------------------------------------------------------------------------------
#define PT_THREADS 256
#define PT_SMEM (256 * 16 * 8)         // one table, 16 lane-private copies = 32 KiB
#define PS_TILE 512
// Blocks per SM of k_phred_sum: four, at 63 registers and no spill. The crossing replay reads its table entries again
// (volatile) instead of reusing the step's 16 gathered doubles; reusing them kept those 32 registers live into the
// replay, and under the 64-register cap of four blocks the compiler then spilled the prefetched uint4, whose store
// waits for the load (every step a full global round trip), or, at three blocks, took 80 registers.
#define PS_OCC 4

struct TieInfo {
    unsigned long long any;            // bit e: some table value q ties when added to a sum in [2^e, 2^(e+1))
    unsigned long long many;           // bit e: more than one does (the step is then walked by lane 0)
    unsigned char ch[64];              // the one that does, when exactly one
};

__device__ __forceinline__ int exponent_of(double v) { return (int)((__double2hiint(v) >> 20) & 0x7FF) - 1023; }
__device__ __forceinline__ double pow2(int e) { return __hiloint2double((e + 1023) << 20, 0); }
__device__ __forceinline__ double shfl_d(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }

__device__ __forceinline__ long long warp_incl_scan_ll(long long v, unsigned lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= (unsigned)d) v += t;
    }
    return v;
}
__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// address of table[c] in this lane's copy (a table of COPIES interleaved copies), c = k-th byte of w
template <int COPIES = 16, typename T>
__device__ __forceinline__ const T *entry_of(const T *tl, uint32_t w, int k) {
    const uint32_t c = __byte_perm(w, 0u, 0x4440u + (unsigned)k);
    return reinterpret_cast<const T *>(reinterpret_cast<const unsigned char *>(tl) + c * (unsigned)(COPIES * sizeof(T)));
}

__global__ void __launch_bounds__(PH_THREADS, 3) k_phred_first(PhredArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const Tab t = make_tables(a.lut, smem_raw);
    const int ws = a.p.window_size;
    for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n; r += (size_t)gridDim.x * blockDim.x) {
        const int L = a.len[r];
        const uint8_t *q = a.qual + a.off[r];
        double sum = 0.0, w = 0.0, best = 0.0;
        chain<true, false>(q, 0, L < ws ? L : ws, ws, t, sum, w, best);
        if (L <= ws) {                                   // read.cpp:217-218
            const double mean = 100.0 * sum / (double)L;
            write_read(a, (uint32_t)r, L, mean, mean);
            continue;
        }
        a.it_b[r] = sum / (double)ws;                    // read.cpp:223
        chain<true, false>(q, ws, L < a.head_len ? L : a.head_len, ws, t, sum, w, best);
        a.it_a[r] = sum;                                 // sum of the first min(L, head_len) bases
    }
}

// does this lane's chunk hold the byte that ties in the current binade?
template <int NW>
__device__ __forceinline__ bool chunk_has(const uint32_t (&cw)[NW], unsigned ch) {
    const uint32_t pat = ch * 0x01010101u;
    uint32_t hit = 0;
#pragma unroll
    for (int i = 0; i < NW; ++i) hit |= __vcmpeq4(cw[i], pat);
    return hit != 0u;
}

__global__ void __launch_bounds__(PT_THREADS, PS_OCC) k_phred_sum(PhredArgs a, TieInfo tie) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *tab = reinterpret_cast<double *>(smem_raw);                // q[256][16]
    __shared__ TieInfo s_tie;
    const double qnan = __longlong_as_double(0x7FF8000000000000ll);
    if (threadIdx.x == 0) s_tie = tie;
    for (int i = threadIdx.x; i < 256 * 16; i += blockDim.x) {
        const double q = a.lut[i >> 4];
        tab[i] = (q >= 0.0 && q < 1.0) ? q : qnan;
    }
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const double *tl = tab + (lane & 15);
    const int H = a.head_len;
    const float inv_tile = 1.0f / (float)PS_TILE;
    // reads are taken longest first from a shared counter: the warps finish together
    for (;;) {
        unsigned long long it = 0;
        if (lane == 0) it = atomicAdd(a.work + 0, 1ull);
        it = __shfl_sync(0xffffffffu, it, 0);
        if (it >= a.n) break;
        const uint32_t r = a.order[it];
        const int L = a.len[r];
        if (L <= H) continue;                                          // k_phred_first has the whole sum
        const uint8_t *q = a.qual + a.off[r];
        const uint4 *qv = reinterpret_cast<const uint4 *>(q);
        double s0 = a.it_a[r];
        long long sb = __double_as_longlong(s0);                       // bit pattern of the collected part of the sum
        int e = exponent_of(s0);
        double Cs = pow2(e), acc = Cs;
        int budget = 0;
        bool tieflag = e >= 0 && e < 64 && ((s_tie.any >> e) & 1ull);
        bool nanf = false;
        uint4 pre = make_uint4(0x21212121u, 0x21212121u, 0x21212121u, 0x21212121u);
        if (H + 16 * (int)lane < L) pre = __ldg(qv + ((H >> 4) + (int)lane));
        for (int j = H; j < L; j += PS_TILE) {
            uint32_t cw[4] = {pre.x, pre.y, pre.z, pre.w};
            {
                const int pn = j + PS_TILE + 16 * (int)lane;
                if (pn < L) pre = __ldg(qv + (pn >> 4));
            }
            const int n = (L - j < PS_TILE) ? L - j : PS_TILE;
            if (n < PS_TILE) {                                         // bytes beyond the read become '!' (q = 0: adds nothing)
                const int nv = n - 16 * (int)lane;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int vb = nv - 4 * i;
                    const uint32_t m = vb >= 4 ? 0xFFFFFFFFu : (vb <= 0 ? 0u : (0xFFFFFFFFu >> (32 - 8 * vb)));
                    cw[i] = (cw[i] & m) | (0x21212121u & ~m);
                }
            }
            const bool in_range = e >= 5 && e < 52;
            int mode = 0;                                              // 0: lane-local grid, 1: careful, 2: lane 0 walks the step
            if (budget == 0 || tieflag) {
                if (budget == 0) {
                    nanf |= (acc != acc);
                    sb += warp_sum_ll(__double_as_longlong(acc) - __double_as_longlong(Cs));   // grid units, still below 2 Cs
                    acc = Cs;
                    if (in_range) {
                        // every base adds at most 1.0: budget * 512 <= floor(room) - 1 keeps the sum strictly inside the binade
                        long long room = ((__double_as_longlong(Cs) + (1ll << 52)) - sb) >> (52 - e);
                        if (room > (1ll << 30)) room = 1ll << 30;
                        budget = room >= 1 ? (int)((room - 1) >> 9) : 0;
                    }
                }
                if (!in_range || sb <= 0) {
                    mode = 2;
                } else {
                    if (tieflag && (((s_tie.many >> e) & 1ull) || __any_sync(0xffffffffu, chunk_has<4>(cw, s_tie.ch[e])))) mode = 2;
                    if (mode == 2 && budget > 0) {
                        sb += warp_sum_ll(__double_as_longlong(acc) - __double_as_longlong(Cs));
                        acc = Cs;
                        budget = 0;
                    }
                    if (mode == 0 && budget == 0) mode = 1;
                }
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) acc += *entry_of(tl, cw[k >> 2], k & 3);       // read.cpp:210-211 on the grid of [Cs, 2 Cs)
            if (mode == 0) {
                --budget;
                continue;
            }
            // acc = Cs + this lane's part, the collected sum is in sb
            bool serial = mode == 2 || __any_sync(0xffffffffu, acc != acc);
            if (!serial) {
                // the step may cross into the next binade, several times while the sum is still small:
                // resolve one crossing per round, the lanes after the crossing lane redo their parts on
                // the coarser grid
                long long cur = sb;                                    // pattern of the exact sum before lane `lo`
                int ce = e, lo = 0;
                double C = Cs, part = acc;
                for (int round = 0; round < 6; ++round) {
                    const long long top = __double_as_longlong(C) + (1ll << 52);       // pattern of 2 C
                    const long long u = (int)lane >= lo ? __double_as_longlong(part) - __double_as_longlong(C) : 0ll;
                    const long long P = warp_incl_scan_ll(u, lane);
                    const unsigned cross = __ballot_sync(0xffffffffu, cur + P >= top);
                    if (cross == 0u) {
                        sb = cur + __shfl_sync(0xffffffffu, P, 31);
                        e = ce;
                        Cs = C;
                        break;
                    }
                    const int lx = __ffs(cross) - 1;
                    // one pass over the 16 bases for both jobs: lane lx continues from the exact sum before
                    // its part with TRUE adds (read.cpp:210-211: this is where the sum leaves the binade),
                    // the lanes after it redo their parts on the next binade's grid, anchored at 2 C
                    const double t0 = __longlong_as_double(cur + __shfl_sync(0xffffffffu, P - u, lx));
                    C = C + C;
                    ce += 1;
                    double v = (int)lane == lx ? t0 : C;
                    if ((int)lane >= lx) {
#pragma unroll
                        for (int k = 0; k < 16; ++k) v += *(const volatile double *)entry_of(tl, cw[k >> 2], k & 3);   // (see PS_OCC)
                    }
                    const double t = shfl_d(v, lx);
                    bool hit = false;
                    if ((s_tie.any >> ce) & 1ull) hit = ((s_tie.many >> ce) & 1ull) || __any_sync(0xffffffffu, chunk_has<4>(cw, s_tie.ch[ce]));
                    if (hit || exponent_of(t) != ce || !(t == t) || round == 5) {
                        serial = true;
                        break;
                    }
                    cur = __double_as_longlong(t);
                    lo = lx + 1;
                    part = v;                                          // (only lanes >= lo are read)
                }
                if (!serial) tieflag = (s_tie.any >> e) & 1ull;
            }
            if (serial) {                                              // the reference's own loop for this step
                double v = __longlong_as_double(sb);
                if (lane == 0)
                    for (int p = 0; p < n; ++p) v += __ldg(a.lut + (unsigned)q[j + p]);
                v = shfl_d(v, 0);
                sb = __double_as_longlong(v);
                e = exponent_of(v);
                Cs = pow2(e);
                tieflag = e >= 0 && e < 64 && ((s_tie.any >> e) & 1ull);
            }
            acc = Cs;
            budget = 0;
        }
        nanf |= (acc != acc);
        sb += warp_sum_ll(__double_as_longlong(acc) - __double_as_longlong(Cs));
        const bool any_nan = __any_sync(0xffffffffu, nanf);
        if (lane == 0) a.it_a[r] = any_nan ? qnan : __longlong_as_double(sb);
    }
}

// raw words holding the K bytes at byte position pos of a read (any alignment)
template <int NW>
__device__ __forceinline__ void load_raw(const uint32_t *__restrict__ q32, int pos, int maxword, uint32_t (&w)[NW + 1]) {
    const int wi = pos >> 2;
#pragma unroll
    for (int i = 0; i <= NW; ++i) {
        const int x = wi + i;
        w[i] = __ldg(q32 + (x < maxword ? x : maxword));
    }
}
template <int NW>
__device__ __forceinline__ void align_raw(const uint32_t (&w)[NW + 1], int pos, uint32_t (&o)[NW]) {
    const unsigned bs = ((unsigned)pos & 3u) * 8u;
#pragma unroll
    for (int i = 0; i < NW; ++i) o[i] = __funnelshift_r(w[i], w[i + 1], bs);
}

#define PT_ANCHOR 0.75
#define PT_ANCHOR_BITS 0x3FE8000000000000ll
#define PW_SHIFT 30                    // filter value of c: A_c >> 30 (A_c < 2^53 / ws, so a window sums to < 2^23)
#define PW_BAD 0x800000u               // 2^23: filter value of a byte the lattice cannot take
#define PW_NONE 0xFFFFFFFFu
#define PW_CHUNK 2048                  // k_phred_win asks L2 for a read's bytes in chunks of this size, one chunk ahead
#define PW_SMEM (256 * 32 * 4 + 256 * 8 * 8)   // filter table, 32 copies (32 KiB) + grid table, 8 copies (16 KiB)
// paths a read takes through k_phred_win, counted per read and per base; counter 8 is the exact steps walked
enum { PW_CAND = 0, PW_FULL = 1, PW_BAD_BYTE = 2, PW_LOW = 3, PW_COUNTERS = 9 };

// asks L2 for bytes [pos, pos + PW_CHUNK) of a read, clamped to its padded extent. Reads start on 64-byte boundaries and
// own whole 64-byte lines (the clamped word loads rely on the same), so the range is 16-byte aligned, a multiple of 16
// long, and never leaves the arena. The filter pass has one step of loads in flight per warp; with the next chunk
// already on its way to L2 those loads wait for L2, not for HBM.
__device__ __forceinline__ void prefetch_chunk(const uint8_t *q, int pos, int padded) {
    if (pos >= padded) return;
    const int end = pos + PW_CHUNK < padded ? pos + PW_CHUNK : padded;
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(q + pos), "r"((uint32_t)(end - pos)) : "memory");
}

// inclusive warp scan; the shuffle's own predicate says whether the source lane exists (no lane tests)
__device__ __forceinline__ uint32_t warp_incl_scan_u32(uint32_t v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1)
        asm("{\n\t.reg .u32 t;\n\t.reg .pred p;\n\t"
            "shfl.sync.up.b32 t|p, %0, %1, 0, 0xffffffff;\n\t"
            "@p add.u32 %0, %0, t;\n\t}"
            : "+r"(v) : "r"(d));
    return v;
}

// one exact step of one lane: K bases; TAIL: only the first nvalid bases exist. x ends at anchor + (sum of
// the lane's grid steps), m is its lowest point (the anchor itself if the lane owns nothing). The bases
// that leave the window are the ones this lane added one step earlier (cwas: that step's bytes).
template <int K, bool TAIL>
__device__ __forceinline__ void win_core(const uint32_t (&cw)[(K + 3) / 4], const uint32_t (&cwas)[(K + 3) / 4],
                                         const double *__restrict__ tl, int nvalid, double &x, double &m) {
    x = PT_ANCHOR;
    m = PT_ANCHOR;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        if (!TAIL || k < nvalid) {
            const double now = *entry_of<8>(tl, cw[k >> 2], k & 3), was = *entry_of<8>(tl, cwas[k >> 2], k & 3);
            x += now - was;                // read.cpp:229-230: both are grid multiples, the difference is exact
            m = x < m ? x : m;             // read.cpp:231-232
        }
    }
}

// the same step on the filter values: x ends at the sum of the lane's (now - was), m is its lowest prefix
// (0, the value before the lane's first base, included). fbase: shared address of this lane's copy, so
// that a look-up is one address op (fbase + c * 128) and one LDS.32.
template <int K, bool TAIL>
__device__ __forceinline__ void filter_core(const uint32_t (&cw)[(K + 3) / 4], uint32_t fbase, int nvalid,
                                            const uint32_t (&was)[K], uint32_t (&now)[K], int &x, int &m) {
    x = 0;
    m = 0;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const uint32_t c = __byte_perm(cw[k >> 2], 0u, 0x4440u + (unsigned)(k & 3));
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(now[k]) : "r"(fbase + (c << 7)));
        if (!TAIL || k < nvalid) {
            x += (int)(now[k] - was[k]);
            m = min(m, x);
        }
    }
}

// this lane's bytes of the window [pos - lpos, pos - lpos + ws) ('!' beyond its share), and the warp's
// exact grid sum of the window in units of 2^-53 (multiples of 2^-53 below 1: every partial sum is exact)
template <int K>
__device__ __forceinline__ long long window_grid(const uint32_t *__restrict__ q32, int pos, int maxword, const double *__restrict__ tg,
                                                 const uint32_t (&keep)[(K + 3) / 4], const uint32_t (&fill)[(K + 3) / 4],
                                                 uint32_t (&cw)[(K + 3) / 4]) {
    constexpr int NW = (K + 3) / 4;
    uint32_t raw[NW + 1];
    load_raw<NW>(q32, pos, maxword, raw);
    align_raw<NW>(raw, pos, cw);
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < NW; ++i) cw[i] = (cw[i] & keep[i]) | fill[i];
#pragma unroll
    for (int k = 0; k < K; ++k) s += *entry_of<8>(tg, cw[k >> 2], k & 3);
    return warp_sum_ll(__double2ll_rn(s * 9007199254740992.0));
}

// the exact chain over steps [t0, t1), entered with the exact value of the window that ends just before
// step t0: bits(W0) + S(t0) - S(0), S(t) = grid sum of bases [t ws, t ws + ws). Returns this lane's lowest
// window value (bit pattern).
template <int K>
__device__ __forceinline__ long long win_exact(const uint32_t *__restrict__ q32, int maxword, int L, int ws, int t0, int t1,
                                               long long W0b, const double *__restrict__ tg, int lpos, int nb_lane,
                                               const uint32_t (&keep)[(K + 3) / 4], const uint32_t (&fill)[(K + 3) / 4],
                                               unsigned lane) {
    constexpr int NW = (K + 3) / 4;
    uint32_t cwas[NW];
    const long long S0 = window_grid<K>(q32, lpos, maxword, tg, keep, fill, cwas);
    long long Wb = W0b + (window_grid<K>(q32, t0 * ws + lpos, maxword, tg, keep, fill, cwas) - S0);
    long long mnb = 0x7FFFFFFFFFFFFFFFll;
    const int jend = min(L, ws + t1 * ws);
    uint32_t pre[NW + 1];
    load_raw<NW>(q32, ws + t0 * ws + lpos, maxword, pre);
    // one step: bases [j, j + ws) (fewer in the last one)
    for (int j = ws + t0 * ws; j < jend; j += ws) {
        uint32_t cw[NW];
        align_raw<NW>(pre, j + lpos, cw);
        if (j + ws < jend) load_raw<NW>(q32, j + ws + lpos, maxword, pre);
        const int n = L - j;
        double x, m;
        if (n >= ws) {
#pragma unroll
            for (int i = 0; i < NW; ++i) cw[i] = (cw[i] & keep[i]) | fill[i];
            win_core<K, false>(cw, cwas, tg, K, x, m);
        } else {
            win_core<K, true>(cw, cwas, tg, max(0, min(nb_lane, n - lpos)), x, m);
        }
        const long long nx = __double_as_longlong(x) - PT_ANCHOR_BITS;
        const long long inc = warp_incl_scan_ll(nx, lane);
        const long long cand = Wb + (inc - nx) + (__double_as_longlong(m) - PT_ANCHOR_BITS);
        mnb = cand < mnb ? cand : mnb;
        Wb += __shfl_sync(0xffffffffu, inc, 31);
#pragma unroll
        for (int i = 0; i < NW; ++i) cwas[i] = cw[i];
    }
    return mnb;
}

template <int K>
__global__ void __launch_bounds__(PT_THREADS, 4) k_phred_win(PhredArgs a) {
    constexpr int NW = (K + 3) / 4;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t *ftab = reinterpret_cast<uint32_t *>(smem_raw);                       // filter values [256][32]
    double *gtab = reinterpret_cast<double *>(smem_raw + 256 * 32 * 4);            // a[256][8] on the grid 2^-53
    __shared__ double s_amax;
    __shared__ uint32_t s_mask[32][4];
    const int ws = a.p.window_size;
    const double qnan = __longlong_as_double(0x7FF8000000000000ll);
    if (threadIdx.x == 0) {
        double mx = 0.0;
        for (int c = 0; c < 256; ++c) {
            const double v = a.lut[256 + c];
            if (v >= 0.0 && v > mx && v * (double)ws <= 1.0 - 1e-10) mx = v;
        }
        s_amax = (0.5 + mx) - 0.5;                                     // on the grid
    }
    if (threadIdx.x < 32) {
        // bytes beyond the lane's share read as '!' (a = 0: no effect on the chain)
        const int nb = max(0, min(K, ws - K * (int)threadIdx.x));
        for (int i = 0; i < 2; ++i) {
            uint32_t m = 0;
            for (int b = 0; b < 4; ++b)
                if (4 * i + b < nb) m |= 0xFFu << (8 * b);
            s_mask[threadIdx.x][i] = m;
            s_mask[threadIdx.x][2 + i] = 0x21212121u & ~m;
        }
    }
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) {
        const double v = a.lut[256 + (i >> 5)];
        bool ok = v >= 0.0 && v * (double)ws <= 1.0 - 1e-10;
        if (ok && v > 0.0) {
            const double sc = ldexp(v, 53);                           // exact; v < 1 so sc < 2^53
            ok = (sc - floor(sc)) != 0.5;                              // would tie on the grid of [0.5, 1)
        }
        const double g = (0.5 + v) - 0.5;                              // a[c] rounded to the grid 2^-53 of [0.5, 1)
        ftab[i] = ok ? (uint32_t)(__double2ull_rn(ldexp(g, 53)) >> PW_SHIFT) : PW_BAD;
        if ((i & 31) < 8) gtab[(i >> 5) * 8 + (i & 31)] = ok ? g : qnan;
    }
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const uint32_t fbase = (uint32_t)__cvta_generic_to_shared(ftab + lane);
    const double *tg = gtab + (lane & 7);
    const double thr = 0.5 + 2.0 * s_amax;
    const int nb_lane = max(0, min(K, ws - K * (int)lane));           // bases of a full step owned by this lane
    const int lpos = K * (int)lane;
    uint32_t keep[NW], fill[NW];
#pragma unroll
    for (int i = 0; i < NW; ++i) {
        keep[i] = s_mask[lane][i];
        fill[i] = s_mask[lane][2 + i];
    }
    unsigned long long paths = 0;                                      // lane i < PW_COUNTERS: counter i of a.phred_paths
    for (;;) {
        unsigned long long it = 0;
        if (lane == 0) it = atomicAdd(a.work + 1, 1ull);
        it = __shfl_sync(0xffffffffu, it, 0);
        if (it >= a.n) break;
        const uint32_t r = a.order[it];
        const int L = a.len[r];
        if (L <= ws) continue;                                         // finished by k_phred_first
        const uint8_t *q = a.qual + a.off[r];
        const uint32_t *q32 = reinterpret_cast<const uint32_t *>(q);
        const int padded = (L + 63) & ~63;
        const int maxword = (padded >> 2) - 1;
        const int nsteps = (L - 1) / ws;
        const double W0 = a.it_b[r];                                   // fl(sum of the first window / ws), read.cpp:223
        bool reject = !(W0 >= thr && W0 < 1.0);
        // ---- filter pass: the window sums of the filter values, every step ----
        uint32_t best = PW_NONE, other = PW_NONE, S0f = 0;             // this lane's lowest candidate, the lowest of its
        int bstep = 0;                                                 // other steps, the first window's sum
        if (!reject) {
            uint32_t va[K], vb[K];
            {
                uint32_t raw[NW + 1], cw[NW];
                load_raw<NW>(q32, lpos, maxword, raw);
                align_raw<NW>(raw, lpos, cw);
#pragma unroll
                for (int k = 0; k < K; ++k) {
                    va[k] = (k < nb_lane) ? ftab[__byte_perm(cw[k >> 2], 0u, 0x4440u + (unsigned)(k & 3)) * 32 + lane] : 0u;
                    S0f += va[k];
                }
            }
            S0f = __reduce_add_sync(0xffffffffu, S0f);
            uint32_t W = S0f;                                          // sum of the window ending at base j - 1
            reject = W >= PW_BAD;
            uint32_t pre[NW + 1];
            if (lane == 0) {
                prefetch_chunk(q, 0, padded);
                prefetch_chunk(q, PW_CHUNK, padded);
            }
            int pf = 2 * PW_CHUNK;                                     // the next chunk to ask L2 for
            load_raw<NW>(q32, ws + lpos, maxword, pre);
            int j = ws, t = 0;
            // one step: bases [j, j + ws) (fewer in the last one). A byte that enters the window in this step is
            // still inside it at the step's last base, so one test of W per step sees every PW_BAD.
#define PW_STEP(WAS, NOW)                                                                                     \
            {                                                                                                 \
                uint32_t cw[NW];                                                                              \
                if (j + ws > pf - PW_CHUNK) {       /* the step reaches the chunk before pf: ask for pf's */  \
                    if (lane == 0) prefetch_chunk(q, pf, padded);                                             \
                    pf += PW_CHUNK;                                                                           \
                }                                                                                             \
                align_raw<NW>(pre, j + lpos, cw);                                                             \
                if (j + ws < L) load_raw<NW>(q32, j + ws + lpos, maxword, pre);                               \
                const int n = L - j;                                                                          \
                int x, m;                                                                                     \
                if (n >= ws) {                                                                                \
                    _Pragma("unroll") for (int i = 0; i < NW; ++i) cw[i] = (cw[i] & keep[i]) | fill[i];       \
                    filter_core<K, false>(cw, fbase, K, WAS, NOW, x, m);                                      \
                } else {                                                                                      \
                    filter_core<K, true>(cw, fbase, max(0, min(nb_lane, n - lpos)), WAS, NOW, x, m);          \
                }                                                                                             \
                const uint32_t inc = warp_incl_scan_u32((uint32_t)x);                                         \
                const uint32_t cand = W + (inc - (uint32_t)x) + (uint32_t)m;                                  \
                other = min(other, max(cand, best));                                                          \
                bstep = cand < best ? t : bstep;                                                              \
                best = min(best, cand);                                                                       \
                W += __shfl_sync(0xffffffffu, inc, 31);                                                       \
                reject |= W >= PW_BAD;                                                                        \
                j += ws;                                                                                      \
                ++t;                                                                                          \
            }
            while (!reject) {
                PW_STEP(va, vb)
                if (j >= L || reject) break;
                PW_STEP(vb, va)
                if (j >= L) break;
            }
#undef PW_STEP
        }
        // ---- exact pass: only the steps that can hold the minimum ----
        const double s = a.it_a[r];                                    // the mean's sum (k_phred_first / k_phred_sum)
        double mn = 0.0;
        int path = PW_BAD_BYTE, exact_steps = 0;                       // (or W0 outside [thr, 1))
        if (!reject) {
            // a window's exact grid sum lies in [2^30 S~, 2^30 (S~ + ws)): the minimum has S~ < mt + ws
            const uint32_t mt = min(__reduce_min_sync(0xffffffffu, best), S0f);
            const bool rel = best <= mt + (uint32_t)ws;
            const bool ambiguous = __any_sync(0xffffffffu, rel && other <= best + (uint32_t)ws);
            // candidate steps (one per relevant lane), or one walk over every step when a relevant lane has
            // another step within ws of its lowest
            uint32_t pend = ambiguous ? (lane == 0 ? 0u : PW_NONE) : (rel ? (uint32_t)bstep : PW_NONE);
            long long mnb = __double_as_longlong(W0);                  // the first window is always a candidate
            for (;;) {
                const uint32_t t = __reduce_min_sync(0xffffffffu, pend);
                if (t == PW_NONE) break;
                const int t1 = ambiguous ? nsteps : (int)t + 1;
                const long long c = win_exact<K>(q32, maxword, L, ws, (int)t, t1, __double_as_longlong(W0), tg, lpos, nb_lane, keep, fill, lane);
                mnb = c < mnb ? c : mnb;
                exact_steps += t1 - (int)t;
                if (pend == t) pend = PW_NONE;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                const long long v = __shfl_xor_sync(0xffffffffu, mnb, o);
                mnb = v < mnb ? v : mnb;
            }
            mn = __longlong_as_double(mnb);
            reject = !(mn >= thr) || !(s == s);
            path = reject ? PW_LOW : ambiguous ? PW_FULL : PW_CAND;
        }
        if (lane == 0) {
            if (reject) a.fallback[1 + atomicAdd(a.fallback, 1u)] = r;
            else finish(a, r, L, s, mn);
        }
        if (lane == 2u * path) paths += 1;
        else if (lane == 2u * path + 1) paths += (unsigned long long)L;
        else if (lane == 8) paths += (unsigned long long)exact_steps;
    }
    if (lane < PW_COUNTERS && paths) atomicAdd(a.phred_paths + lane, paths);
}

}  // namespace

static int ensure_lut(fl_ctx *ctx) {
    if (ctx->d_lut && ctx->lut_window == ctx->p.window_size) return FL_OK;
    double h[512];
    fl_phred_luts(ctx->p.window_size, h, h + 256);
    if (!ctx->d_lut) FL_CUDA(ctx, cudaMalloc(&ctx->d_lut, sizeof(h)));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->d_lut, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
    // binades [2^e, 2^(e+1)) of the running sum in which some table value in [0,1) would sit exactly
    // on a rounding tie (its bits below 2^(e-52) are 100..0): only there k_phred_mean_long tests ties
    ctx->tie_binades = 0;
    ctx->tie_many = 0;
    memset(ctx->tie_char, 0, sizeof(ctx->tie_char));
    for (int e = 0; e < 64; ++e)
        for (int c = 0; c < 256; ++c) {
            const double q = h[c];
            if (!(q > 0.0 && q < 1.0)) continue;
            const double scaled = ldexp(q, 52 - e);          // exact
            if (scaled - floor(scaled) == 0.5) {
                if (ctx->tie_binades & (1ull << e)) ctx->tie_many |= 1ull << e;
                ctx->tie_binades |= 1ull << e;
                ctx->tie_char[e] = (unsigned char)c;
            }
        }
    // same for the window table a[] and the binades [2^-e, 2^(1-e)) of w (bit e), (kept for diagnostics)
    ctx->tie_binades_a = 0;
    for (int e = 0; e < 64; ++e)
        for (int c = 0; c < 256; ++c) {
            const double v = h[256 + c];
            if (!(v > 0.0 && v < 1.0)) continue;
            const double scaled = ldexp(v, 52 + e);          // exact (power-of-two scaling)
            if (scaled < 9007199254740992.0 && scaled - floor(scaled) == 0.5) ctx->tie_binades_a |= 1ull << e;
        }
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->lut_window = ctx->p.window_size;
    return FL_OK;
}

// The arguments every Phred kernel shares: the view, the tables and where the scores go. A pass that is not over whole
// reads sends everything but mean / window / passed to sc_sink, which nothing reads: the kernels stay exactly as they
// are (a test for the case inside write_read cost k_phred_win<8> a register spill).
static int phred_args_of(fl_ctx *ctx, const BatchView &b, const PhredOut &o, PhredArgs *out) {
    PhredArgs a{};
    a.qual = b.qual; a.off = b.off; a.len = b.len; a.n = b.n;
    a.lut = ctx->d_lut; a.p = ctx->p;
    a.r_mean = o.mean; a.r_window = o.window; a.r_passed = o.passed;
    if (o.whole_reads) {
        const size_t rb = ctx->n_reads, wb = ctx->n_rows;
        a.r_len = ctx->r_len.p + rb; a.r_first = ctx->r_first.p + rb; a.r_last = ctx->r_last.p + rb;
        a.r_nbad = ctx->r_nbad.p + rb; a.r_nchild = ctx->r_nchild.p + rb;
        a.r_rowstart = ctx->r_rowstart.p + rb;
        a.w_parent = ctx->w_parent.p + wb; a.w_start = ctx->w_start.p + wb; a.w_end = ctx->w_end.p + wb;
        a.w_mean = ctx->w_mean.p + wb; a.w_window = ctx->w_window.p + wb; a.w_passed = ctx->w_passed.p + wb;
        a.read_base = rb; a.row_base = wb;
    } else {
        FL_CUDA(ctx, ctx->sc_sink.reserve((size_t)b.n + 1, 0, ctx->stream));   // 8 bytes per item: room for any field
        unsigned long long *s = ctx->sc_sink.p;
        int32_t *s32 = reinterpret_cast<int32_t *>(s);
        a.r_len = a.r_first = a.r_last = a.r_nbad = a.r_nchild = a.w_start = a.w_end = s32;
        a.r_rowstart = s;
        a.w_parent = reinterpret_cast<uint32_t *>(s);
        a.w_mean = a.w_window = reinterpret_cast<double *>(s);
        a.w_passed = reinterpret_cast<uint8_t *>(s);
    }
    *out = a;
    return FL_OK;
}

int fl_score_phred(fl_ctx *ctx, const BatchView &b) {
    if (!b.qual) {
        ctx->set_error("FASTA input not supported without an external reference (no quality string and the k-mer set is empty)");
        return FL_EINVAL;                                   // main.cpp:103-106
    }
    const size_t n = b.n;
    FL_TRY(fl_reserve_reads(ctx, ctx->n_reads + n));
    FL_TRY(fl_reserve_rows(ctx, ctx->n_rows + n));
    const size_t rb = ctx->n_reads;
    FL_TRY(fl_phred_pass(ctx, b, PhredOut{ctx->r_mean.p + rb, ctx->r_window.p + rb, ctx->r_passed.p + rb, true}));
    ctx->n_reads += n;
    ctx->n_rows += n;
    return FL_OK;
}

int fl_phred_pass(fl_ctx *ctx, const BatchView &b, const PhredOut &o) {
    FL_TRY(ensure_lut(ctx));
    const size_t n = b.n;
    cudaStream_t st = ctx->stream;
    const int ws = ctx->p.window_size;
    if (ctx->phred_mode != 0 && ws >= 16 && ws <= 256) {
        // default: one warp per read, both chains by exact grid arithmetic (k_phred_sum, k_phred_win)
        FL_CUDA(ctx, ctx->sc_order.reserve(n, 0, st));
        FL_TRY(fl_order_by_length(ctx, b.len, n, ctx->sc_order.p));
        PhredArgs a;
        FL_TRY(phred_args_of(ctx, b, o, &a));
        a.order = ctx->sc_order.p;
        a.head_len = (ws + 15) & ~15;                     // k_phred_first sums up to here; k_phred_sum takes over (16-byte loads)
        FL_CUDA(ctx, ctx->sc_f64.reserve(3 * n + 8, 0, st));
        a.it_a = ctx->sc_f64.p; a.it_b = ctx->sc_f64.p + n; a.it_c = ctx->sc_f64.p + 2 * n;
        FL_CUDA(ctx, ctx->sc_u32a.reserve(n + 2, 0, st));
        a.fallback = ctx->sc_u32a.p;
        FL_CUDA(ctx, cudaMemsetAsync(a.fallback, 0, sizeof(uint32_t), st));
        a.work = ctx->d_scalars + 24;
        FL_CUDA(ctx, cudaMemsetAsync(a.work, 0, 2 * sizeof(unsigned long long), st));
        a.phred_paths = ctx->d_scalars + FL_SCALAR_PHRED_PATHS;
        if (!ctx->phred_attr_set) {
            FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_sum, cudaFuncAttributeMaxDynamicSharedMemorySize, PT_SMEM));
            FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_win<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM));
            FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_win<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM));
            FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_win<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, PW_SMEM));
            FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_first, cudaFuncAttributeMaxDynamicSharedMemorySize, PH_SMEM));
            FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_fallback, cudaFuncAttributeMaxDynamicSharedMemorySize, PH_SMEM));
            ctx->phred_attr_set = true;
        }
        {
            unsigned hb = fl_blocks(n, PH_THREADS);
            if (hb > (unsigned)ctx->sm_count * 3) hb = (unsigned)ctx->sm_count * 3;
            k_phred_first<<<hb, PH_THREADS, PH_SMEM, st>>>(a);
            ctx->launches++;
        }
        // persistent grids, as many blocks as stay resident: k_phred_sum PS_OCC per SM, k_phred_win 4
        const bool occ_set = ctx->phred_occupancy >= 1 && ctx->phred_occupancy <= 6;
        const unsigned want = fl_blocks(n * 32, PT_THREADS);
        const unsigned sblocks = min(want, (unsigned)ctx->sm_count * (unsigned)(occ_set ? ctx->phred_occupancy : PS_OCC));
        const unsigned blocks = min(want, (unsigned)ctx->sm_count * (unsigned)(occ_set ? ctx->phred_occupancy : 4));
        {
            // timed as one scoring pass: the sum kernel and the window kernel
            KernelTimer kt(ctx, FL_KERNEL_SCORE_PHRED);
            TieInfo ti;
            ti.any = ctx->tie_binades;
            ti.many = ctx->tie_many;
            memcpy(ti.ch, ctx->tie_char, 64);
            // (One fused pass -- a 16-byte {q, a} gather per base feeding both chains, the step one window long -- was
            // built and measured slower: 14 % MORE instructions, because the sum's bookkeeping then runs once per 250 bases
            // instead of once per 512, and 80 registers cost a quarter of the warps; the code is gone.)
            k_phred_sum<<<sblocks, PT_THREADS, PT_SMEM, st>>>(a, ti);
            if (ws <= 64) k_phred_win<2><<<blocks, PT_THREADS, PW_SMEM, st>>>(a);
            else if (ws <= 128) k_phred_win<4><<<blocks, PT_THREADS, PW_SMEM, st>>>(a);
            else k_phred_win<8><<<blocks, PT_THREADS, PW_SMEM, st>>>(a);
            ctx->launches += 2;
        }
        k_phred_fallback<<<ctx->sm_count, PH_THREADS, PH_SMEM, st>>>(a);   // reads the window kernel rejected (normally none)
        ctx->launches++;
        FL_CUDA(ctx, cudaGetLastError());
        return FL_OK;
    }
    // ---- phred_mode 0 (kept for comparison): work items, one thread per chain ----
    // ---- plan: items per read -> exclusive scan -> item table ----
    FL_CUDA(ctx, ctx->sc_u64a.reserve(n + 1, 0, st));
    k_phred_plan<<<fl_blocks(n, 256), 256, 0, st>>>(b.len, b.n, ws, ctx->sc_u64a.p);
    ctx->launches++;
    FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64a.p, ctx->sc_u64a.p, n, ctx->d_scalars));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->sc_u64a.p + n, ctx->d_scalars, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars, ctx->d_scalars, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(ctx, cudaStreamSynchronize(st));
    const size_t n_items = (size_t)ctx->h_scalars[0];
    FL_CUDA(ctx, ctx->sc_u64b.reserve(n_items + 1, 0, st));                 // items (uint2 = 8 bytes)
    FL_CUDA(ctx, ctx->sc_u32a.reserve(n_items + n + 2, 0, st));             // cost [n_items] | fallback [1 + n]
    FL_CUDA(ctx, ctx->sc_order.reserve(n_items, 0, st));
    FL_CUDA(ctx, ctx->sc_f64.reserve(3 * n_items + 8, 0, st));
    uint2 *items = reinterpret_cast<uint2 *>(ctx->sc_u64b.p);
    uint32_t *cost = ctx->sc_u32a.p;                     // bucket key = kind * 256 + length bucket
    uint32_t *fallback = ctx->sc_u32a.p + n_items;
    k_phred_fill<<<fl_blocks(n, 256), 256, 0, st>>>(b.len, b.n, ws, ctx->sc_u64a.p, items, cost);
    ctx->launches++;
    FL_CUDA(ctx, cudaMemsetAsync(fallback, 0, sizeof(uint32_t), st));
    FL_TRY(fl_order_by_key(ctx, cost, n_items, ctx->sc_order.p));

    PhredArgs a;
    FL_TRY(phred_args_of(ctx, b, o, &a));
    a.item_start = ctx->sc_u64a.p; a.order = ctx->sc_order.p; a.items = items; a.n_items = n_items;
    a.it_a = ctx->sc_f64.p; a.it_b = ctx->sc_f64.p + n_items; a.it_c = ctx->sc_f64.p + 2 * n_items;
    a.fallback = fallback;
    if (!ctx->phred_items_attr_set) {
        FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_items, cudaFuncAttributeMaxDynamicSharedMemorySize, PH_SMEM));
        FL_CUDA(ctx, cudaFuncSetAttribute(k_phred_fallback, cudaFuncAttributeMaxDynamicSharedMemorySize, PH_SMEM));
        ctx->phred_items_attr_set = true;
    }
    unsigned blocks = fl_blocks(n_items, PH_THREADS);
    const unsigned max_blocks = (unsigned)ctx->sm_count * 3;
    if (blocks > max_blocks) blocks = max_blocks;
    {
        KernelTimer kt(ctx, FL_KERNEL_SCORE_PHRED);
        k_phred_items<<<blocks, PH_THREADS, PH_SMEM, st>>>(a);
    }
    ctx->launches++;
    if (n_items > n) {
        k_phred_mean_long<<<ctx->sm_count * 6, 256, PH_MEAN_SMEM, st>>>(a, ctx->tie_binades);
        ctx->launches++;
        k_phred_merge<<<fl_blocks(n, 256), 256, 0, st>>>(a);
        k_phred_fallback<<<ctx->sm_count, PH_THREADS, PH_SMEM, st>>>(a);
        ctx->launches += 2;
    }
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

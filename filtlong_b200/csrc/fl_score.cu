// filtlong_b200/csrc/fl_score.cu -- per-read scoring, replaces Read::Read (reference src/read.cpp:25-144).
//
// Two modes, chosen by the state of the k-mer set exactly like read.cpp:35 (`kmers->empty()`):
//
//  Phred mode (read.cpp:35-39) lives in fl_phred.cu: one THREAD per work item walks the quality string in the reference's
//    own operation order -- sum += q[c] for the mean (read.cpp:208-213), and the incremental
//    window recurrence w -= a[c_out]; w += a[c_in] (read.cpp:216-236) -- so mean and window
//    quality come out bit-identical to the reference (their rounding depends on the order of
//    the additions). q[] and a[] = q[]/window_size are 256-entry tables evaluated with the host
//    libm (read.cpp:270-273) and replicated in shared memory so that every lane owns its banks.
//    Rows are issued longest-first (length buckets) so lanes of a warp carry similar work.
//
//  k-mer mode (read.cpp:43-58): kernel A is the HBM-bound hot loop -- a warp streams 1024 bases
//    per step (coalesced 8-byte loads of 2-bit codes), forms the 32 forward 16-mers of each lane
//    with funnel shifts, probes the 512 MiB direct-address bitmap (one 32-byte sector per base
//    when the set exceeds L2), and paints 16-base hits into a 1-bit-per-base mask with shuffles.
//    Kernels B then work on that mask only (L/8 bytes per read): popcount -> mean (exact: the
//    reference sums 1.0s), first/last base in a k-mer (read.cpp:75-84), bad ranges and child
//    ranges (read.cpp:89-130), and the serial window recurrence on {0, 1/ws} per row. Children
//    are NOT re-probed: a matching 16-mer never overlaps a bad range, so a child's mask is the
//    parent's mask restricted to the child range (SURVEY 8a-R7); the reference re-runs the whole
//    constructor instead (read.cpp:137).
#include <cmath>

#include "fl_device.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// shared scalar helpers (double arithmetic in exactly the reference's order; file is compiled
// with --fmad=false so nothing is contracted)
// ---------------------------------------------------------------------------------------------


// ---------------------------------------------------------------------------------------------
// k-mer mode, kernel A: probe + paint
// ---------------------------------------------------------------------------------------------
struct ProbeArgs {
    const uint32_t *seq2b;
    const uint64_t *off;
    const int32_t *len;
    const unsigned long long *tile_start;   // [n+1]; [n] = number of tiles
    uint32_t n;
    const uint32_t *bitmap;
    const uint32_t *anchor;                  // position-anchored table (fl_anchor_slot), used when ANCH
    const unsigned long long *filter;        // L2-resident pre-filter (fl_kmers.cu), used when FILT
    unsigned filter_log2_words;
    int filter_kind;
    uint32_t *mask;                          // 1 bit per padded base, same coordinates as the arena
};

// Single-word loads of the membership tables are ld.global.nc.L1::no_allocate (no L1 line fill for a random probe).
// Measured and dropped: ld.global.cg, L2 eviction-priority hints on filter / table / mask traffic, the persisting-L2
// window, and .L2::64B on the table sectors (it halves the DRAM bytes, not the time: the ceiling is L2-missing
// REQUESTS per second).
// word holding the membership bit of `kmer`, and the bit's index, for the k-mer that starts at a read
// position whose low two bits are pos_lo2
template <bool ANCH>
__device__ __forceinline__ void probe_slot(uint32_t kmer, unsigned pos_lo2, uint32_t &word, uint32_t &bit) {
    if (ANCH) fl_anchor_slot(kmer, 3u - pos_lo2, word, bit);
    else { word = kmer >> 5; bit = kmer & 31u; }
}

__device__ __forceinline__ uint32_t probe(const uint32_t *__restrict__ bitmap, uint32_t word_index) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(bitmap + word_index));
    return v;
}

// (compiled for 5 / 6 blocks per SM the pair-keyed variant spills and runs slower)
template <int FILT, bool ANCH>
__global__ void __launch_bounds__(256, 4) k_probe_paint(ProbeArgs a) {
    const unsigned lane = threadIdx.x & 31;
    const uint32_t *__restrict__ table = ANCH ? a.anchor : a.bitmap;
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long n_tiles = a.tile_start[a.n];      // read on the device: no host round trip between the scan and the launch
    for (unsigned long long tile = warp; tile < n_tiles; tile += n_warps) {
        const uint32_t s = fl_find_seq(a.tile_start, a.n, tile);
        const int L = a.len[s];
        const unsigned long long off = a.off[s];
        const uint32_t *seqw = a.seq2b + (off >> 4);
        uint32_t *maskw = a.mask + (off >> 5);
        const unsigned long long padded = ((unsigned long long)L + FL_ALIGN_BASES - 1) & ~(unsigned long long)(FL_ALIGN_BASES - 1);
        const unsigned long long tile_base = (tile - a.tile_start[s]) * FL_TILE_BASES;

        // hits of the 16 k-mer starts just before the tile (they paint into the tile's first bases)
        uint32_t carry = 0;   // bit k = hit of the k-mer starting at base (run_start - 32 + k)
        if (tile_base > 0) {
            uint32_t wa = __ldg(seqw + (tile_base >> 4) - 1), wb = __ldg(seqw + (tile_base >> 4));
            uint32_t hit = 0;
            if (lane < 16) {
                unsigned long long b = tile_base - 16 + lane;
                if (b + (FL_K - 1) < (unsigned long long)L) {
                    uint32_t k = __funnelshift_l(wb, wa, 2 * lane);
                    uint32_t word, bit;
                    probe_slot<ANCH>(k, lane & 3u, word, bit);         // tile_base is a multiple of 4
                    hit = (probe(table, word) >> bit) & 1u;
                }
            }
            carry = __ballot_sync(0xffffffffu, hit) << 16;
        }
        for (int step = 0; step < FL_TILE_STEPS; ++step) {
            const unsigned long long sb = tile_base + (unsigned long long)step * FL_STEP_BASES;
            if (sb >= padded) break;
            const LaneWords w = fl_load_lane_words(seqw, sb, padded, lane);
            const unsigned long long lb = sb + 32ull * lane;
            // number of valid k-mer starts in this lane's run: starts b with b + 15 < L
            long long nv = (long long)L - (FL_K - 1) - (long long)lb;
            const int nvalid = nv <= 0 ? 0 : (nv >= 32 ? 32 : (int)nv);
            uint32_t h = 0;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                uint32_t words[16];
                uint32_t go = 0xFFFFu;                // which of the 16 k-mers still need the exact bitmap
                if (FILT == 1) {
                    // 16 independent loads from the 32 MiB pre-filter (kept in L2): most k-mers of a
                    // noisy read are absent and stop here, without touching HBM
                    unsigned long long f[16];
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        uint32_t word;
                        unsigned long long fb;
                        fl_filter_slot(fl_kmer_at(w, half * 16 + i), a.filter_log2_words, a.filter_kind, word, fb);
                        if (half * 16 + i < nvalid) {
                            f[i] = __ldcg(a.filter + word);   // L2 only (no L1 line fill)
                        } else f[i] = 0ull;
                    }
                    go = 0;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        uint32_t word;
                        unsigned long long fb;
                        fl_filter_slot(fl_kmer_at(w, half * 16 + i), a.filter_log2_words, a.filter_kind, word, fb);
                        go |= ((f[i] & fb) == fb ? 1u : 0u) << i;
                    }
                }
                if (FILT == 2) {
                    // group-keyed pre-filter: the four 16-mers of a table group share ONE filter word (4 loads per half, not 16)
                    unsigned long long f[4];
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const int p0 = half * 16 + 4 * g;
                        const uint32_t word = fl_filter_word_group4(fl_kmer_at(w, p0 + 3), 0u, a.filter_log2_words);
                        f[g] = p0 < nvalid ? __ldcg(a.filter + word) : 0ull;
                    }
                    go = 0;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const unsigned long long fb = fl_filter_bits_role(fl_kmer_at(w, half * 16 + i), 3u - (unsigned)(i & 3), a.filter_kind);
                        go |= ((f[i >> 2] & fb) == fb ? 1u : 0u) << i;
                    }
                }
                if (FILT == 3) {
                    // pair-keyed pre-filter: two neighbouring 16-mers share a word (8 loads per half)
                    unsigned long long f[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        const int p0 = half * 16 + 2 * q;
                        const uint32_t word = fl_filter_word_pair(fl_kmer_at(w, p0), 0u, a.filter_log2_words);
                        f[q] = p0 < nvalid ? __ldcg(a.filter + word) : 0ull;
                    }
                    go = 0;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const unsigned long long fb = fl_filter_bits_role(fl_kmer_at(w, half * 16 + i), (unsigned)(i & 1), a.filter_kind);
                        go |= ((f[i >> 1] & fb) == fb ? 1u : 0u) << i;
                    }
                }
                if (ANCH) {
                    // the four 16-mers starting at 4g .. 4g+3 of the lane's run (a multiple of 32, so of 4)
                    // share one 32-byte sector of the anchored table, read as its two 128-bit halves (sm_90 has no
                    // 256-bit load). Lane pairs loading the two halves of one sector in one instruction and trading them
                    // by shuffles were measured slower on an H100 (400 W): config 3 probe 137 against 116 ms, config 5 equal.
                    uint32_t sec[4][8];
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const int p0 = half * 16 + 4 * g;
                        const uint32_t key = (fl_kmer_at(w, p0 + 3) >> 6) & 0x3FFFFFFu;   // bases p0+3 .. p0+15
                        const bool need = p0 < nvalid && ((go >> (4 * g)) & 0xFu);
                        if (need) {
                            const uint32_t *s = table + (size_t)key * 8u;
                            asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];"
                                         : "=r"(sec[g][0]), "=r"(sec[g][1]), "=r"(sec[g][2]), "=r"(sec[g][3]) : "l"(s));
                            asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];"
                                         : "=r"(sec[g][4]), "=r"(sec[g][5]), "=r"(sec[g][6]), "=r"(sec[g][7]) : "l"(s + 4));
                        } else {
#pragma unroll
                            for (int q = 0; q < 8; ++q) sec[g][q] = 0u;
                        }
                    }
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int p = half * 16 + 4 * g + j;
                            uint32_t word, bit;
                            fl_anchor_slot(fl_kmer_at(w, p), 3u - (unsigned)j, word, bit);
                            const uint32_t v = (word & 1u) ? sec[g][2 * (3 - j) + 1] : sec[g][2 * (3 - j)];
                            const uint32_t ok = (p < nvalid && ((go >> (4 * g + j)) & 1u)) ? 1u : 0u;
                            h |= (((v >> bit) & 1u) & ok) << p;
                        }
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int p = half * 16 + i;
                        const uint32_t k = fl_kmer_at(w, p);
                        words[i] = (p < nvalid && ((go >> i) & 1u)) ? probe(table, k >> 5) : 0u;     // read.cpp:52
                    }
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int p = half * 16 + i;
                        const uint32_t k = fl_kmer_at(w, p);
                        h |= ((words[i] >> (k & 31)) & 1u) << p;
                    }
                }
            }
            // paint: base covered if any of the 16 k-mers ending at or after it hit (read.cpp:53-54)
            uint32_t prev = __shfl_up_sync(0xffffffffu, h, 1);
            if (lane == 0) prev = carry;
            unsigned long long y = ((unsigned long long)h << 32) | prev;
            y |= y << 1;
            y |= y << 2;
            y |= y << 4;
            y |= y << 8;
            if (lb < padded) {
                maskw[lb >> 5] = (uint32_t)(y >> 32);
            }
            carry = __shfl_sync(0xffffffffu, h, 31);
        }
    }
}

__global__ void k_tiles_of(const int32_t *__restrict__ len, uint32_t n, unsigned long long *__restrict__ tiles) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) tiles[i] = fl_tiles_of(len[i] > 0 ? (int)(((unsigned)len[i] + FL_ALIGN_BASES - 1) & ~(FL_ALIGN_BASES - 1)) : 0);
}

// ---------------------------------------------------------------------------------------------
// k-mer mode, kernels B: everything else from the 1-bit mask, one WARP per read / per row.
//
//   k_kmer_scan<EMIT>  one warp per read streams the mask (32 words = 1024 bases per step, coalesced):
//                      first / last base in a k-mer (read.cpp:75-84), the zero runs that become bad ranges
//                      (read.cpp:89-117) found with ballots and shuffles (a run that crosses word boundaries
//                      is closed by the lane holding its terminating one-bit), child ranges (read.cpp:119-130).
//                      Pass 1 counts, an exclusive scan places the rows, pass 2 (EMIT) writes them.
//   k_kmer_window      one warp per row: mean = 100 * popcount / len (the reference sums exact 1.0s), and the
//                      window quality of read.cpp:216-236 bit for bit without walking the row (see below).
// ---------------------------------------------------------------------------------------------
struct ScanArgs {
    const uint32_t *mask;
    const uint64_t *off;
    const int32_t *len;
    uint32_t n;
    fl_params p;
    int32_t *r_len, *r_first, *r_last, *r_nbad, *r_nchild;
    unsigned long long *r_rowstart;       // COUNT: row_base + r (final when nothing can have children). EMIT: in = batch-local exclusive scan, out = + row_base
    unsigned long long *rows_per_read;    // COUNT out [n]
    int32_t *item_len;                    // COUNT: [r] = L (the parent item). EMIT: [n + row] = child length, 0 for the row of a childless read
    uint32_t *w_parent;                   // EMIT out, offset to this batch's first row
    int32_t *w_start, *w_end;
    unsigned long long read_base, row_base;
};

template <bool EMIT>
__global__ void __launch_bounds__(256) k_kmer_scan(ScanArgs a) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned lower = (1u << lane) - 1u;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    const bool split_set = a.p.split_set != 0, trim = a.p.trim != 0;
    const int split = a.p.split;
    for (size_t r = warp; r < a.n; r += n_warps) {
        const int L = a.len[r];
        const uint32_t *m = a.mask + (a.off[r] >> 5);
        const int n_words = (L + 31) >> 5;
        unsigned long long rs_row = 0;
        if (EMIT) {
            rs_row = a.r_rowstart[r];
            if (lane == 0) a.r_rowstart[r] = rs_row + a.row_base;
            if (a.r_nchild[r] == 0) {                            // the read is its own row (main.cpp:140)
                if (lane == 0) {
                    a.w_parent[rs_row] = (uint32_t)(a.read_base + r);
                    a.w_start[rs_row] = 0;
                    a.w_end[rs_row] = L;
                    a.item_len[a.n + rs_row] = 0;                // scored by the parent's item
                }
                continue;
            }
        }
        int first = -1, last = -1, n_bad = 0, n_child = 0, rs = 0;
        int carry_open = 0;                                      // length of the zero run that ends at the end of the previous step
        bool seen_one = false;
        auto child = [&](int s, int e, int idx) {
            if (EMIT) {
                a.w_parent[rs_row + idx] = (uint32_t)(a.read_base + r);
                a.w_start[rs_row + idx] = s;
                a.w_end[rs_row + idx] = e;
                a.item_len[a.n + rs_row + idx] = e - s;
            }
        };
        uint32_t x_next = (int)lane < n_words ? __ldg(m + lane) : 0u;      // one step ahead: the loop body is a dependent chain
        for (int wb = 0; wb < n_words; wb += 32) {
            const int wi = wb + (int)lane;
            const uint32_t x = x_next;
            x_next = wi + 32 < n_words ? __ldg(m + wi + 32) : 0u;
            const unsigned nz = __ballot_sync(0xffffffffu, x != 0u);
            const int tzc = x ? __clz(x) : 32, lzc = x ? __ffs(x) - 1 : 32;
            // common case: every word of the step has a hit, nothing open from before can reach --split, and this is
            // not the step that holds the read's first hit: no bad range can start or end here
            if (seen_one && nz == 0xffffffffu && (!split_set || (split >= 64 && carry_open + 32 < split))) {
                carry_open = __shfl_sync(0xffffffffu, tzc, 31);
                last = (wb + 31) * 32 + 32 - carry_open;
                continue;
            }
            if (nz == 0u) {                                      // 1024 uncovered bases: the open run just grows
                carry_open += 1024;
                continue;
            }
            const unsigned lo_nz = nz & lower;
            const int j = lo_nz ? 31 - __clz(lo_nz) : 0;
            const int tz_j = __shfl_sync(0xffffffffu, tzc, j);
            const int open_prev = lo_nz ? tz_j + 32 * ((int)lane - j - 1) : carry_open + 32 * (int)lane;
            const int o = (wb + (int)lane) * 32 + lzc;           // position of this word's lowest one-bit
            const int runlen = open_prev + lzc, z = o - runlen;
            const bool is_first = x && !seen_one && !lo_nz;      // the run is [0, first): read.cpp:106-111 decides
            const bool b_emit = x && (is_first ? ((split_set && o >= split && o > 0) || (trim && o > 0))
                                               : (split_set && runlen >= split));
            if (!(split_set && split < 32)) {
                // bad ranges end only where a word has its lowest one-bit: at most one per lane, counted with ballots
                const unsigned em = __ballot_sync(0xffffffffu, b_emit);
                if (em) {
                    const unsigned lo_em = em & lower;
                    const int prev_e = __shfl_sync(0xffffffffu, o, lo_em ? 31 - __clz(lo_em) : 0);
                    const int rs_mine = lo_em ? prev_e : rs;
                    const bool b_child = b_emit && z - rs_mine > 0;
                    const unsigned cm = __ballot_sync(0xffffffffu, b_child);
                    if (EMIT && b_child) child(rs_mine, z, n_child + __popc(cm & lower));
                    n_bad += __popc(em);
                    n_child += __popc(cm);
                    rs = __shfl_sync(0xffffffffu, o, 31 - __clz(em));
                }
            } else {
                // zero runs strictly inside the word (shorter than 32: only a --split below 32 can want them)
                int n_in = 0, in_last_e = 0;
                if (split_set && split < 32 && x) {
                    uint32_t y = ~x & (0xFFFFFFFFu << lzc) & (0xFFFFFFFFu >> tzc);
                    while (y) {
                        const int s0 = __ffs(y) - 1;
                        const uint32_t rest = ~(y >> s0);
                        const int ln = __ffs(rest) - 1;              // run length (a one-bit follows inside the word)
                        if (ln >= split) { ++n_in; in_last_e = wi * 32 + s0 + ln; }
                        y &= ~(((1u << ln) - 1u) << s0);
                    }
                }
                const bool emits = b_emit || n_in > 0;
                const int my_last_e = n_in > 0 ? in_last_e : o;
                const unsigned em = __ballot_sync(0xffffffffu, emits);
                const unsigned lo_em = em & lower;
                const int pe = lo_em ? 31 - __clz(lo_em) : 0;
                const int prev_e = __shfl_sync(0xffffffffu, my_last_e, pe);
                const int rs_mine = lo_em ? prev_e : rs;
                const int b_child = (b_emit && z - rs_mine > 0) ? 1 : 0;
                const int my_children = b_child + n_in;              // every in-word run is preceded by a one-bit: a child always
                int incl = my_children;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= (unsigned)d) incl += t;
                }
                if (EMIT && emits) {
                    int idx = n_child + incl - my_children, prev = rs_mine;
                    if (b_emit) {
                        if (b_child) child(prev, z, idx++);
                        prev = o;
                    }
                    if (n_in > 0) {
                        uint32_t y = ~x & (0xFFFFFFFFu << lzc) & (0xFFFFFFFFu >> tzc);
                        while (y) {
                            const int s0 = __ffs(y) - 1;
                            const uint32_t rest = ~(y >> s0);
                            const int ln = __ffs(rest) - 1;
                            if (ln >= split) {
                                child(prev, wi * 32 + s0, idx++);
                                prev = wi * 32 + s0 + ln;
                            }
                            y &= ~(((1u << ln) - 1u) << s0);
                        }
                    }
                }
                int my_bad = (b_emit ? 1 : 0) + n_in;
#pragma unroll
                for (int d = 16; d; d >>= 1) my_bad += __shfl_xor_sync(0xffffffffu, my_bad, d);
                n_bad += my_bad;
                n_child += __shfl_sync(0xffffffffu, incl, 31);
                if (em) rs = __shfl_sync(0xffffffffu, my_last_e, 31 - __clz(em));
            }
            {
                const int top = 31 - __clz(nz);
                const int tz_top = __shfl_sync(0xffffffffu, tzc, top);
                carry_open = tz_top + 32 * (31 - top);
                last = (wb + top) * 32 + 32 - tz_top;                                       // read.cpp:81-84
                if (!seen_one) first = __shfl_sync(0xffffffffu, o, __ffs(nz) - 1);          // read.cpp:77-80
                seen_one = true;
            }
        }
        // the tail [last, L) and the closing child (read.cpp:112-116, 127-129)
        if (first < 0) {
            if (split_set && L > 0 && L >= split) n_bad = 1;     // one zero run [0, L): a bad range without children
        } else {
            const bool tail_bad = last < L && ((split_set && (L - last) >= split) || trim);
            if (tail_bad) {
                ++n_bad;
                if (last - rs > 0) { if (lane == 0) child(rs, last, n_child); ++n_child; }
                rs = L;
            }
            if (n_bad > 0 && L - rs > 0) { if (lane == 0) child(rs, L, n_child); ++n_child; }
        }
        if (!EMIT && lane == 0) {
            a.r_len[r] = L;
            a.r_first[r] = first;
            a.r_last[r] = last;
            a.r_nbad[r] = n_bad;
            a.r_nchild[r] = n_child;
            a.rows_per_read[r] = n_child > 0 ? (unsigned long long)n_child : 1ull;
            a.r_rowstart[r] = a.row_base + r;
            a.item_len[r] = L;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Window quality in k-mer mode (read.cpp:216-236 on qualities in {0, 1}) WITHOUT walking the row.
//
// The reference's chain:  w0 = fl(c0 / ws);  per step  w -= out ? rq : 0;  w += in ? rq : 0;  best = min(best, w),
// rq = fl(1 / ws). With c the window's hit count (an integer prefix sum of the mask: parallel):
//  (1) inside one binade adding / subtracting rq moves w by exactly R = rq rounded to the binade's grid -- inverse
//      operations. Also in a "tie binade" (rq = (n + 1/2) grid units exactly): round-half-even makes every result
//      of an operation there EVEN, and from an even value the step is the even one of n, n + 1;
//  (2) subtracting rq across a binade's floor (onto the finer grid) and adding it back returns to the same value;
//  (3) hence from an ANCHOR (w_a, c_a) every value the chain takes at a level c it reaches by moves below the
//      highest level visited so far is one function F(c): walk down from the anchor (or up,
//      on the anchor's grid). The chain's minimum over such an EPOCH is F(min c): one integer reduction, one
//      short walk (grid jumps inside a binade, one true subtraction per binade floor);
//  (4) not reversible: an addition that reaches a level not visited since the anchor AND next to a binade edge
//      (it enters the coarser grid above, or leaves the binade's lowest level), and an ODD value inside a tie
//      binade (the first after entering from the finer grid below, or w0 itself) until an operation made it even.
//      Only THAT step is done with the reference's own double operations (its word is spread over the warp, one lane
//      per step, to find it); a new epoch starts from the value it produced. Rare: a few record levels per row.
// tests/models/kmer_window_model.c is the scalar model of exactly this procedure (fuzzed against the reference
// recurrence: tests/test_kmer_window_model.py); the kernel below is its transcription, 32 words per iteration.
// ---------------------------------------------------------------------------------------------
// one edge for every binade from rq's own up to 2^1: at most 33 for an int window size (rq >= 2^-31). Dropping one lets the
// chain cross that edge as if it were inside a binade: at ws >= 2^15 (more than 16 binades) the window quality of a row
// hovering at half coverage came out one ulp off (tests/test_gpu_kmer_masks.py).
#define KW_MAX_EDGES 34

struct KwConsts {
    double rq;
    unsigned long long mant_rq;               // 53-bit significand of rq
    int e_rq;                                 // rq in [2^e_rq, 2^(e_rq+1))
    int n_edges;
    int elo[KW_MAX_EDGES], ehi[KW_MAX_EDGES]; // count intervals around the binade edges 2^e / rq (+- two levels)
};

struct KwAnchor {
    double w;
    long long wb, rint, lo, hi;
    int c, c_edge;
    bool lattice;
    bool unsafe;                              // odd value inside a tie binade: every differing step is walked until it is even
};

// grid parameters of the binade of w; false if it has none (rq's own binade and below -- arithmetic there is exact -- or
// an odd value in a tie binade; *tie_odd tells the latter)
__device__ __forceinline__ bool kw_binade(const KwConsts &k, double w, long long &wb, long long &rint, long long &lo, long long &hi,
                                          bool *tie_odd = nullptr) {
    if (tie_odd) *tie_odd = false;
    if (!(w > 0.0)) return false;
    const long long b = __double_as_longlong(w);
    const int e = (int)((b >> 52) & 0x7FF) - 1023;
    const int s = e - k.e_rq;
    if (s < 1 || s > 52) return false;
    const unsigned long long half = 1ull << (s - 1);
    long long r = (long long)((k.mant_rq + half) >> s);
    if ((k.mant_rq & ((1ull << s) - 1ull)) == half) {
        // tie binade: rq = (n + 1/2) grid units; results of operations inside it are even, and from an even value the
        // step is the even one of n, n + 1
        if (b & 1) {
            if (tie_odd) *tie_odd = true;
            return false;
        }
        const long long n = (long long)(k.mant_rq >> s);
        r = (n & 1) ? n + 1 : n;
    }
    wb = b;
    rint = r;
    lo = (long long)(e + 1023) << 52;
    hi = lo + (1ll << 52);
    return true;
}

// floor(x / y) for 0 <= x < 2^53, 0 < y < 2^53 without a 64-bit integer division
__device__ __forceinline__ long long kw_floor_div(long long x, long long y) {
    long long q = (long long)((double)x / (double)y);
    if (q * y > x) --q;
    else if ((q + 1) * y <= x) ++q;
    return q;
}

__device__ __forceinline__ void kw_set_anchor(KwAnchor &a, const KwConsts &k, double w, int c) {
    a.w = w;
    a.c = c;
    a.lattice = kw_binade(k, w, a.wb, a.rint, a.lo, a.hi, &a.unsafe);
    a.c_edge = c;                                              // no usable grid: any level above the anchor ends the epoch
    if (a.lattice) a.c_edge = c + (int)kw_floor_div(a.hi - 2 - a.wb, a.rint);
}

// F(c) for c <= a.c_edge: the chain's value at level c inside the anchor's epoch
__device__ __forceinline__ double kw_eval(const KwAnchor &a, const KwConsts &k, int c) {
    if (c >= a.c) return a.lattice ? __longlong_as_double(a.wb + a.rint * (long long)(c - a.c)) : a.w;
    double w = a.w;
    int cur = a.c;
    while (cur > c) {
        long long wb, rint, lo, hi;
        if (kw_binade(k, w, wb, rint, lo, hi)) {
            long long room = kw_floor_div(wb - (lo + 1), rint);      // levels that can be descended on the grid (value stays >= 2^e + ulp)
            if (room > (long long)(cur - c)) room = cur - c;
            if (room > 0) {
                w = __longlong_as_double(wb - rint * room);
                cur -= (int)room;
                continue;
            }
        }
        w = w - k.rq;                                                // read.cpp:229: across the binade floor
        --cur;
    }
    return w;
}

struct WinArgs {
    const uint32_t *mask;
    const uint64_t *off;                    // per batch read
    const int32_t *len;
    const uint32_t *order;                  // items in descending length order
    uint32_t n_items, n_reads;              // items [0, n_reads): the reads themselves; [n_reads, n_items): rows (batch-local)
    fl_params p;
    KwConsts k;
    const int32_t *r_nchild;
    const unsigned long long *r_rowstart;   // global row index of a read's first row
    unsigned long long row_base, read_base;
    const uint32_t *w_parent;               // batch-local row arrays
    const int32_t *w_start, *w_end;
    double *r_mean, *r_window;              // batch-local outputs per read / per row
    uint8_t *r_passed;
    double *w_mean, *w_window;
    uint8_t *w_passed;
    unsigned long long *work;               // shared item counter
};

// the two mask words that hold bits [pos, pos + 32) (last valid word: m[last_word]); kw_bits = their funnel shift
__device__ __forceinline__ uint2 kw_raw(const uint32_t *__restrict__ m, long long pos, int last_word) {
    const int wi = (int)(pos >> 5);
    return make_uint2(__ldg(m + (wi <= last_word ? wi : last_word)), __ldg(m + (wi + 1 <= last_word ? wi + 1 : last_word)));
}
__device__ __forceinline__ uint32_t kw_bits(const uint32_t *__restrict__ m, long long pos, int last_word) {
    const uint2 r = kw_raw(m, pos, last_word);
    return __funnelshift_r(r.x, r.y, (unsigned)pos & 31u);
}

// popcount of bits [S, S + n) of the mask, by the whole warp
__device__ __forceinline__ int kw_popcount(const uint32_t *__restrict__ m, int S, int n, int last_word, unsigned lane) {
    int cnt = 0;
    for (int j = (int)lane * 32; j < n; j += 1024) {
        uint32_t v = kw_bits(m, (long long)S + j, last_word);
        if (n - j < 32) v &= (1u << (n - j)) - 1u;
        cnt += __popc(v);
    }
    return __reduce_add_sync(0xffffffffu, cnt);
}

__global__ void __launch_bounds__(256, 4) k_kmer_window(WinArgs a) {
    // nibble table: 4 steps with pure-plus bits p and pure-minus bits q (p & q == 0) ->
    // (delta + 4) | (lowest after-step partial sum + 4) << 4 | (highest + 4) << 8
    __shared__ unsigned short lut[256];
    {
        const int p = threadIdx.x & 15, q = threadIdx.x >> 4;
        int d = 0, mn = 99, mx = -99;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            d += ((p >> t) & 1) - ((q >> t) & 1);
            mn = d < mn ? d : mn;
            mx = d > mx ? d : mx;
        }
        lut[threadIdx.x & 255] = (unsigned short)((d + 4) | ((mn + 4) << 4) | ((mx + 4) << 8));
    }
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const KwConsts &k = a.k;
    const int ws = a.p.window_size;
    const double wsd = (double)ws;
    // items come from a shared counter (longest first); a warp holds its NEXT item's index one row ahead, so that the
    // dependent loads atomicAdd -> order[it] -> descriptors are not all paid at the start of every row
    unsigned long long it_next = 0;
    if (lane == 0) it_next = atomicAdd(a.work, 1ull);
    it_next = __shfl_sync(0xffffffffu, it_next, 0);
    uint32_t idx_next = it_next < a.n_items ? __ldg(a.order + it_next) : 0u;
    for (;;) {
        const unsigned long long it = it_next;
        if (it >= a.n_items) break;
        const uint32_t idx = idx_next;
        if (lane == 0) it_next = atomicAdd(a.work, 1ull);
        it_next = __shfl_sync(0xffffffffu, it_next, 0);
        idx_next = it_next < a.n_items ? __ldg(a.order + it_next) : 0u;
        uint32_t r;
        int S, E;
        long long row = -1;                                        // batch-local row this item writes (if any)
        const bool is_read = idx < a.n_reads;
        if (is_read) {
            r = idx;
            S = 0;
            E = a.len[r];
            if (a.r_nchild[r] == 0) row = (long long)(a.r_rowstart[r] - a.row_base);
        } else {
            row = (long long)(idx - a.n_reads);
            r = (uint32_t)(a.w_parent[row] - a.read_base);
            if (a.r_nchild[r] == 0) continue;                      // scored by the read's own item
            S = a.w_start[row];
            E = a.w_end[row];
        }
        const int len = E - S;
        const uint32_t *m = a.mask + (a.off[r] >> 5);
        const int last_word = ((((a.len[r] > 0 ? a.len[r] : 1) + 63) & ~63) >> 5) - 1;
        double mean, window;
        if (len <= ws) {                                           // read.cpp:217-218
            const int hits = kw_popcount(m, S, len, last_word, lane);
            mean = 100.0 * (double)hits / (double)len;             // read.cpp:208-213 (0/0 = NaN for an empty read, as there)
            window = mean;
        } else {
            // the first iteration's mask words are requested before the first window is counted (independent loads)
            const int T = len - ws;                                // steps: base S + ws + t enters, base S + t leaves
            const unsigned sh_in = (unsigned)(S + ws) & 31u, sh_out = (unsigned)S & 31u;     // (t0 and 32 * lane are multiples of 32)
            uint2 raw_in = make_uint2(0u, 0u), raw_out = make_uint2(0u, 0u);
            if (32 * (int)lane < T) {
                raw_in = kw_raw(m, (long long)S + ws + 32 * (int)lane, last_word);
                raw_out = kw_raw(m, (long long)S + 32 * (int)lane, last_word);
            }
            int c = kw_popcount(m, S, ws, last_word, lane);        // read.cpp:220-222: the first window's sum is an exact integer
            const int c0 = c;
            int hits = 0;                                          // ones entering the window, per lane
            double best = (double)c / wsd;                         // read.cpp:223
            KwAnchor an;
            kw_set_anchor(an, k, best, c);
            int cmin = c, trec = c;                                // lowest / highest after-step count of the current epoch
            int H = 0, H_trec = -0x7FFFFFFF;                       // cached epoch limit and the record level it was computed for
            // inside the loop the NEXT iteration's words are requested before this iteration's (dependent) arithmetic
            // starts: one memory latency per 1024 steps would otherwise be all a warp does
            for (int t0 = 0; t0 < T; t0 += 1024) {
                const int tl = t0 + 32 * (int)lane;
                const int nv = T - tl;
                uint32_t in = 0, out = 0;
                if (nv > 0) {
                    in = __funnelshift_r(raw_in.x, raw_in.y, sh_in);
                    out = __funnelshift_r(raw_out.x, raw_out.y, sh_out);
                    if (nv < 32) {
                        const uint32_t vm = (1u << nv) - 1u;
                        in &= vm;
                        out &= vm;
                    }
                }
                if (tl + 1024 < T) {
                    raw_in = kw_raw(m, (long long)S + ws + tl + 1024, last_word);
                    raw_out = kw_raw(m, (long long)S + tl + 1024, last_word);
                }
                hits += __popc(in);
                const uint32_t pin = in & ~out, pout = out & ~in, both = in & out;
                const bool valid = nv > 0;
                const int np = __popc(pin), nm = __popc(pout), delta = np - nm;
                int incl = delta;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= (unsigned)d) incl += t;
                }
                const int cs = c + incl - delta;                   // count at the start of this lane's word
                // Levels the word can visit, first by the cheap bound [cs - #minus, cs + #plus] (a step that subtracts
                // and adds dips one level more). The exact extremes (nibble table) are only needed by a word that
                // might lower the epoch's minimum, raise its record level, or be flagged: decided for the whole warp.
                int mn = -nm, mx = np;                             // lowest / highest after-step partial sum (bounds)
                {
                    const bool want = valid && (cs - nm < cmin || cs + np > trec);
                    if (__any_sync(0xffffffffu, want)) {
                        int d = 0;
                        mn = 99;
                        mx = -99;
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const unsigned e = lut[((pin >> (4 * q)) & 15u) | (((pout >> (4 * q)) & 15u) << 4)];
                            const int lo_q = d + (int)((e >> 4) & 15u) - 4, hi_q = d + (int)((e >> 8) & 15u) - 4;
                            mn = lo_q < mn ? lo_q : mn;
                            mx = hi_q > mx ? hi_q : mx;
                            d += (int)(e & 15u) - 4;
                        }
                    }
                }
                const int hi_level = cs + (mx > 0 ? mx : 0);
                const bool differs = valid && (in | out) != 0u;
                int cur = 0;
                for (;;) {
                    // first level whose first visit ends the epoch: beyond the anchor's binade, or inside an edge interval
                    // (a function of the anchor and of the record level: both change rarely, so it is kept across iterations)
                    if (H_trec != trec) {
                        H = an.c_edge + 1;
                        for (int i = 0; i < k.n_edges; ++i)
                            if (k.ehi[i] >= trec) {
                                const int h = k.elo[i] > trec + 1 ? k.elo[i] : trec + 1;
                                H = h < H ? h : H;
                            }
                        H_trec = trec;
                    }
                    const bool in_range = valid && (int)lane >= cur;
                    const bool flag = in_range && ((an.unsafe && differs) || hi_level >= H);
                    const unsigned fm = __ballot_sync(0xffffffffu, flag);
                    int first = fm ? __ffs(fm) - 1 : 32;
                    const bool seg = in_range && (int)lane < first;
                    const int seg_min = __reduce_min_sync(0xffffffffu, seg ? cs + mn : 0x7FFFFFFF);
                    const int seg_max = __reduce_max_sync(0xffffffffu, seg ? hi_level : -0x7FFFFFFF);
                    cmin = seg_min < cmin ? seg_min : cmin;
                    trec = seg_max > trec ? seg_max : trec;
                    if (first == 32) break;
                    // The flagged word, one lane per step. Only the step that does something irreversible is done with the
                    // reference's own operations: the first one that reaches the level H (or, from an odd value in a tie
                    // binade, the first that does anything). The steps before it are still inside the epoch (F), the steps
                    // after it belong to the epoch of the new anchor -- which may end in this very word again.
                    {
                        const uint32_t win = __shfl_sync(0xffffffffu, in, first), wout = __shfl_sync(0xffffffffu, out, first);
                        const int cw0 = __shfl_sync(0xffffffffu, cs, first);
                        const uint32_t upto = 0xFFFFFFFFu >> (31u - lane);             // steps 0 .. lane
                        const int lvl = cw0 + __popc(win & ~wout & upto) - __popc(wout & ~win & upto);   // level after step `lane`
                        int p = 0;
                        for (;;) {
                            if (H_trec != trec) {
                                H = an.c_edge + 1;
                                for (int i = 0; i < k.n_edges; ++i)
                                    if (k.ehi[i] >= trec) {
                                        const int h = k.elo[i] > trec + 1 ? k.elo[i] : trec + 1;
                                        H = h < H ? h : H;
                                    }
                                H_trec = trec;
                            }
                            const bool stop = (int)lane >= p && (an.unsafe ? (((win | wout) >> lane) & 1u) != 0u : lvl >= H);
                            const unsigned sm = __ballot_sync(0xffffffffu, stop);
                            const int ts = sm ? __ffs(sm) - 1 : 32;
                            const bool before = (int)lane >= p && (int)lane < ts;
                            const int smin = __reduce_min_sync(0xffffffffu, before ? lvl : 0x7FFFFFFF);
                            const int smax = __reduce_max_sync(0xffffffffu, before ? lvl : -0x7FFFFFFF);
                            cmin = smin < cmin ? smin : cmin;
                            trec = smax > trec ? smax : trec;
                            if (ts == 32) break;
                            const double f = kw_eval(an, k, cmin);                       // close the epoch
                            best = f < best ? f : best;
                            int cw = __shfl_sync(0xffffffffu, lvl, ts > 0 ? ts - 1 : 0);
                            if (ts == 0) cw = cw0;
                            double w = kw_eval(an, k, cw);                               // the chain's value before step ts
                            if ((wout >> ts) & 1u) { w -= k.rq; --cw; }                  // read.cpp:229
                            if ((win >> ts) & 1u) { w += k.rq; ++cw; }                   // read.cpp:230
                            best = w < best ? w : best;                                  // read.cpp:231-232
                            kw_set_anchor(an, k, w, cw);
                            cmin = cw;
                            trec = cw;
                            H_trec = -0x7FFFFFFF;                                        // new anchor: the limit must be recomputed
                            p = ts + 1;
                        }
                    }
                    cur = first + 1;
                }
                c += __shfl_sync(0xffffffffu, incl, 31);
            }
            {
                const double f = kw_eval(an, k, cmin);
                best = f < best ? f : best;
            }
            if (best < 0.5 / wsd) best = 0.0;                      // read.cpp:233-234
            hits = __reduce_add_sync(0xffffffffu, hits) + c0;
            mean = 100.0 * (double)hits / (double)len;             // read.cpp:208-213
            window = 100.0 * best;
        }
        if (lane == 0) {
            const uint8_t passed = fl_hard_cutoffs(a.p, len, mean, window);        // read.cpp:65-73
            if (is_read) {
                a.r_mean[r] = mean;
                a.r_window[r] = window;
                a.r_passed[r] = passed;
            }
            if (row >= 0) {
                a.w_mean[row] = mean;
                a.w_window[row] = window;
                a.w_passed[row] = passed;
            }
        }
    }
}

__global__ void k_identity_rows(uint32_t n, const int32_t *__restrict__ len, uint32_t *w_parent, int32_t *w_start,
                                int32_t *w_end, unsigned long long read_base) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    w_parent[i] = (uint32_t)(read_base + i);
    w_start[i] = 0;
    w_end[i] = len[i];
}

// --contam, per read: the percentage of its bases covered by a contaminant 16-mer, in the expression k_kmer_window
// evaluates for a read's mean in k-mer mode (read.cpp:208-213: 0 below 16 bases, NaN for an empty read), and whether it
// is above max_contam (a NaN never is). One warp per read over its mask words.
__global__ void __launch_bounds__(256) k_contam_reads(const uint32_t *__restrict__ mask, const uint64_t *__restrict__ off,
                                                      const int32_t *__restrict__ len, uint32_t n, double max_contam,
                                                      double *__restrict__ pct, uint8_t *__restrict__ removed) {
    const unsigned lane = threadIdx.x & 31;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t r = warp; r < n; r += n_warps) {
        const int L = len[r];
        const uint32_t *m = mask + (off[r] >> 5);
        int hits = 0;
        for (int w = (int)lane; w * 32 < L; w += 32) {
            uint32_t v = __ldg(m + w);
            if (L - w * 32 < 32) v &= (1u << (L - w * 32)) - 1u;
            hits += __popc(v);
        }
        hits = __reduce_add_sync(0xffffffffu, hits);
        if (lane == 0) {
            const double c = 100.0 * (double)hits / (double)L;
            pct[r] = c;
            removed[r] = c > max_contam ? 1 : 0;
        }
    }
}

// --contam, per row of the batch: a removed read's rows are not passed and take no part in the ranking (w_excl)
__global__ void k_contam_rows(const uint32_t *__restrict__ parent, const uint8_t *__restrict__ removed, size_t n,
                              uint8_t *__restrict__ passed, uint8_t *__restrict__ excl) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint8_t x = removed[parent[i]];
        excl[i] = x;
        if (x) passed[i] = 0;
    }
}

template <typename T>
cudaError_t grow(DevVec<T> &v, size_t n, size_t keep, cudaStream_t s) { return v.reserve(n, keep, s); }

}  // namespace

int fl_reserve_reads(fl_ctx *c, size_t n_total) {
    size_t k = c->n_reads;
    cudaStream_t s = c->stream;
    FL_CUDA(c, grow(c->r_len, n_total, k, s));
    FL_CUDA(c, grow(c->r_first, n_total, k, s));
    FL_CUDA(c, grow(c->r_last, n_total, k, s));
    FL_CUDA(c, grow(c->r_nbad, n_total, k, s));
    FL_CUDA(c, grow(c->r_nchild, n_total, k, s));
    FL_CUDA(c, grow(c->r_mean, n_total, k, s));
    FL_CUDA(c, grow(c->r_window, n_total, k, s));
    FL_CUDA(c, grow(c->r_passed, n_total, k, s));
    FL_CUDA(c, grow(c->r_rowstart, n_total, k, s));
    return FL_OK;
}

int fl_reserve_rows(fl_ctx *c, size_t n_total) {
    size_t k = c->n_rows;
    cudaStream_t s = c->stream;
    FL_CUDA(c, grow(c->w_parent, n_total, k, s));
    FL_CUDA(c, grow(c->w_start, n_total, k, s));
    FL_CUDA(c, grow(c->w_end, n_total, k, s));
    FL_CUDA(c, grow(c->w_mean, n_total, k, s));
    FL_CUDA(c, grow(c->w_window, n_total, k, s));
    FL_CUDA(c, grow(c->w_passed, n_total, k, s));
    return FL_OK;
}

// the window-size dependent constants of k_kmer_window (mirrors kw_consts of tests/models/kmer_window_model.c)
static void kw_make_consts(int ws, KwConsts *k) {
    memset(k, 0, sizeof(*k));
    k->rq = 1.0 / (double)ws;                                       // read.cpp:229-230: qualities[i] / window_size with q == 1.0
    long long b;
    memcpy(&b, &k->rq, 8);
    k->e_rq = (int)((b >> 52) & 0x7FF) - 1023;
    k->mant_rq = ((unsigned long long)b & ((1ull << 52) - 1ull)) | (1ull << 52);
    for (int e = k->e_rq; e <= 1 && k->n_edges < KW_MAX_EDGES; ++e) {     // edges 2^e of every binade a count 0..ws can reach
        const double x = ldexp(1.0, e) * (double)ws;
        if (x > (double)ws + 3.0) break;
        k->elo[k->n_edges] = (int)floor(x) - 2;
        k->ehi[k->n_edges] = (int)ceil(x) + 2;
        k->n_edges++;
    }
}

// k-mer mode, first half: probe + paint, then the counting pass of k_kmer_scan; with --trim / --split it ends by sending the
// batch's row count to the host (ev_rows), which score_kmer_back waits for
static ScanArgs scan_args_of(fl_ctx *ctx, const BatchView &b) {
    const size_t rb = ctx->n_reads, wb = ctx->n_rows;
    ScanArgs sa{};
    sa.mask = ctx->sc_mask.p; sa.off = b.off; sa.len = b.len; sa.n = b.n; sa.p = ctx->p;
    sa.r_len = ctx->r_len.p + rb; sa.r_first = ctx->r_first.p + rb; sa.r_last = ctx->r_last.p + rb;
    sa.r_nbad = ctx->r_nbad.p + rb; sa.r_nchild = ctx->r_nchild.p + rb;
    sa.r_rowstart = ctx->r_rowstart.p + rb; sa.rows_per_read = ctx->sc_u64b.p;
    sa.item_len = ctx->sc_items.p;
    sa.read_base = rb; sa.row_base = wb;
    return sa;
}

static unsigned scan_blocks_of(fl_ctx *ctx, size_t n) {
    unsigned scan_blocks = fl_blocks(n * 32, 256);
    if (scan_blocks > (unsigned)ctx->sm_count * 8) scan_blocks = (unsigned)ctx->sm_count * 8;
    return scan_blocks;
}

static int count_rows(fl_ctx *ctx, const BatchView &b);
static int contam_rows(fl_ctx *ctx, size_t row0);

int fl_probe_paint(fl_ctx *ctx, const KmerSet &set, const BatchView &b, uint32_t *mask, int timer) {
    const size_t n = b.n;
    cudaStream_t st = ctx->stream;
    FL_CUDA(ctx, ctx->sc_u64a.reserve(n + 1, 0, st));
    k_tiles_of<<<fl_blocks(n, 256), 256, 0, st>>>(b.len, b.n, ctx->sc_u64a.p);
    ctx->launches++;
    FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64a.p, ctx->sc_u64a.p, n, ctx->d_scalars));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->sc_u64a.p + n, ctx->d_scalars, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    ProbeArgs pa{};
    pa.seq2b = b.seq2b; pa.off = b.off; pa.len = b.len; pa.tile_start = ctx->sc_u64a.p;
    pa.n = b.n; pa.bitmap = set.bitmap; pa.anchor = set.anchor; pa.mask = mask;
    pa.filter = set.filter; pa.filter_log2_words = ctx->filter_log2_words; pa.filter_kind = set.filter_kind;
    // persistent grid; the kernel reads the tile count from tile_start[n], so nothing here waits for the scan
    unsigned long long tiles_bound = (b.padded_bases + FL_TILE_BASES - 1) / FL_TILE_BASES + n;
    unsigned blocks = (unsigned)((tiles_bound + 7) / 8);
    unsigned max_blocks = (unsigned)ctx->sm_count * 4;
    if (blocks > max_blocks) blocks = max_blocks;
    if (blocks < 1) blocks = 1;
    // Measured and dropped: a minimizer-keyed
    // pre-filter with per-lane load de-duplication, L2 eviction hints, the persisting-L2 window, .L2::64B table loads.
    KernelTimer kt(ctx, timer);
    if (set.use_anchor) {
        const int filt = !set.use_filter ? 0 : ((set.filter_kind & 4) ? 2 : ((set.filter_kind & 8) ? 3 : 1));
        if (filt == 0) k_probe_paint<0, true><<<blocks, 256, 0, st>>>(pa);
        else if (filt == 1) k_probe_paint<1, true><<<blocks, 256, 0, st>>>(pa);
        else if (filt == 2) k_probe_paint<2, true><<<blocks, 256, 0, st>>>(pa);
        else k_probe_paint<3, true><<<blocks, 256, 0, st>>>(pa);
    } else if (set.use_filter) {                        // plain bitmap (FL_ANCHOR=0: cross-checks and profiling)
        k_probe_paint<1, false><<<blocks, 256, 0, st>>>(pa);
    } else {
        k_probe_paint<0, false><<<blocks, 256, 0, st>>>(pa);
    }
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

static int score_kmer_front(fl_ctx *ctx, const BatchView &b) {
    if (!b.seq2b) { ctx->set_error("k-mer scoring needs seq2b"); return FL_EINVAL; }
    FL_TRY(fl_reserve_reads(ctx, ctx->n_reads + b.n));
    // ---- kernel A: probe + paint ----
    FL_CUDA(ctx, ctx->sc_mask.reserve((size_t)(b.padded_bases >> 5) + 1, 0, ctx->stream));
    FL_TRY(fl_probe_paint(ctx, ctx->ref, b, ctx->sc_mask.p, FL_KERNEL_PROBE_PAINT));
    return count_rows(ctx, b);
}

// B, counting pass over sc_mask: first / last, bad ranges, how many children (k_kmer_scan); with --trim / --split it ends
// by sending the batch's row count to the host (ev_rows)
static int count_rows(fl_ctx *ctx, const BatchView &b) {
    const size_t n = b.n;
    cudaStream_t st = ctx->stream;
    const size_t rb = ctx->n_reads;
    FL_CUDA(ctx, ctx->sc_u64b.reserve(n + 1, 0, st));
    FL_CUDA(ctx, ctx->sc_items.reserve(n + 8, 0, st));
    const ScanArgs sa = scan_args_of(ctx, b);
    k_kmer_scan<false><<<scan_blocks_of(ctx, n), 256, 0, st>>>(sa);
    ctx->launches++;
    if (ctx->p.trim || ctx->p.split_set) {
        FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64b.p, ctx->r_rowstart.p + rb, n, ctx->d_scalars));
        FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars + FL_HSCALAR_ROWS, ctx->d_scalars, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        if (!ctx->ev_rows) FL_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_rows, cudaEventDisableTiming));
        FL_CUDA(ctx, cudaEventRecord(ctx->ev_rows, st));
    }
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

// B, emitting pass: the batch's n_rows_batch rows (children, or the read itself) get parent / start / end
static int emit_rows(fl_ctx *ctx, const BatchView &b, size_t n_rows_batch) {
    const size_t n = b.n, wb = ctx->n_rows;
    cudaStream_t st = ctx->stream;
    FL_CUDA(ctx, ctx->sc_items.reserve(n + n_rows_batch + 8, n, st));
    ScanArgs sa = scan_args_of(ctx, b);
    sa.w_parent = ctx->w_parent.p + wb; sa.w_start = ctx->w_start.p + wb; sa.w_end = ctx->w_end.p + wb;
    k_kmer_scan<true><<<scan_blocks_of(ctx, n), 256, 0, st>>>(sa);
    ctx->launches++;
    return FL_OK;
}

// k-mer mode, second half: rows (children or the reads themselves), then mean + window quality per item (k_kmer_window)
static int score_kmer_back(fl_ctx *ctx, const BatchView &b) {
    const size_t n = b.n;
    cudaStream_t st = ctx->stream;
    const size_t rb = ctx->n_reads, wb = ctx->n_rows;
    const bool may_have_children = ctx->p.trim || ctx->p.split_set;
    size_t n_rows_batch = n;
    if (may_have_children) {
        FL_CUDA(ctx, cudaEventSynchronize(ctx->ev_rows));            // the one host round trip of the path
        n_rows_batch = (size_t)ctx->h_scalars[FL_HSCALAR_ROWS];
    }
    FL_TRY(fl_reserve_rows(ctx, ctx->n_rows + n_rows_batch));
    size_t n_items = n;
    if (!may_have_children) {
        k_identity_rows<<<fl_blocks(n, 256), 256, 0, st>>>(b.n, b.len, ctx->w_parent.p + wb, ctx->w_start.p + wb,
                                                          ctx->w_end.p + wb, rb);
        ctx->launches++;
    } else {
        n_items = n + n_rows_batch;
        FL_TRY(emit_rows(ctx, b, n_rows_batch));
    }
    FL_CUDA(ctx, ctx->sc_order.reserve(n_items, 0, st));
    FL_TRY(fl_order_by_length(ctx, ctx->sc_items.p, n_items, ctx->sc_order.p));
    {
        WinArgs wa{};
        wa.mask = ctx->sc_mask.p; wa.off = b.off; wa.len = b.len; wa.order = ctx->sc_order.p;
        wa.n_items = (uint32_t)n_items; wa.n_reads = b.n; wa.p = ctx->p;
        kw_make_consts(ctx->p.window_size, &wa.k);
        wa.r_nchild = ctx->r_nchild.p + rb; wa.r_rowstart = ctx->r_rowstart.p + rb;
        wa.row_base = wb; wa.read_base = rb;
        wa.w_parent = ctx->w_parent.p + wb; wa.w_start = ctx->w_start.p + wb; wa.w_end = ctx->w_end.p + wb;
        wa.r_mean = ctx->r_mean.p + rb; wa.r_window = ctx->r_window.p + rb; wa.r_passed = ctx->r_passed.p + rb;
        wa.w_mean = ctx->w_mean.p + wb; wa.w_window = ctx->w_window.p + wb; wa.w_passed = ctx->w_passed.p + wb;
        wa.work = ctx->d_scalars + 26;
        FL_CUDA(ctx, cudaMemsetAsync(wa.work, 0, sizeof(unsigned long long), st));
        unsigned blocks = fl_blocks(n_items * 32, 256);
        const unsigned cap = (unsigned)ctx->sm_count * 8;
        if (blocks > cap) blocks = cap;
        {
            KernelTimer kt(ctx, FL_KERNEL_KMER_STATS);
            k_kmer_window<<<blocks, 256, 0, st>>>(wa);
        }
        ctx->launches++;
    }
    FL_CUDA(ctx, cudaGetLastError());
    ctx->n_reads += n;
    ctx->n_rows += n_rows_batch;
    return FL_OK;
}

// --trim_q, first half: the quality mask, the counting pass of k_kmer_scan (it sends the row count to the host), then the
// parents' mean / window quality by the plain Phred pass while that count travels
static int score_qual_front(fl_ctx *ctx, const BatchView &b) {
    if (!b.qual) {
        ctx->set_error("FASTA input not supported without an external reference (no quality string and the k-mer set is empty)");
        return FL_EINVAL;                                   // main.cpp:103-106
    }
    FL_TRY(fl_reserve_reads(ctx, ctx->n_reads + b.n));
    FL_TRY(fl_qual_mask(ctx, b));
    {
        KernelTimer kt(ctx, FL_KERNEL_ROW_SCAN);
        FL_TRY(count_rows(ctx, b));
    }
    const size_t rb = ctx->n_reads;
    return fl_phred_pass(ctx, b, PhredOut{ctx->r_mean.p + rb, ctx->r_window.p + rb, ctx->r_passed.p + rb, false});
}

// --trim_q, second half: the rows, then the children's scores (fl_qtrim.cu)
static int score_qual_back(fl_ctx *ctx, const BatchView &b) {
    FL_CUDA(ctx, cudaEventSynchronize(ctx->ev_rows));                // the one host round trip of the path
    const size_t n_rows_batch = (size_t)ctx->h_scalars[FL_HSCALAR_ROWS];
    FL_TRY(fl_reserve_rows(ctx, ctx->n_rows + n_rows_batch));
    {
        KernelTimer kt(ctx, FL_KERNEL_ROW_SCAN);
        FL_TRY(emit_rows(ctx, b, n_rows_batch));
    }
    FL_TRY(fl_score_qual_rows(ctx, b, n_rows_batch));
    FL_CUDA(ctx, cudaGetLastError());
    ctx->n_reads += b.n;
    ctx->n_rows += n_rows_batch;
    return FL_OK;
}

int fl_score_complete(fl_ctx *ctx) {
    if (!ctx->kmer_pending) return FL_OK;
    ctx->kmer_pending = false;
    const int slot = ctx->kmer_pending_slot;
    ctx->kmer_pending_slot = -1;
    const size_t row0 = ctx->n_rows;
    if (ctx->pending_qual) FL_TRY(score_qual_back(ctx, ctx->kmer_pending_view));
    else FL_TRY(score_kmer_back(ctx, ctx->kmer_pending_view));
    FL_TRY(contam_rows(ctx, row0));
    if (slot >= 0) {                                              // the staged inputs are free once these kernels have run
        FL_CUDA(ctx, cudaEventRecord(ctx->stg[slot].consumed, ctx->stream));
        ctx->stg[slot].in_use = true;
    }
    return FL_OK;
}

int fl_check_trim_q(fl_ctx *ctx) {
    if (ctx->p.trim_q > 0 && ctx->ref.n > 0) {
        ctx->set_error("trim_q cannot be used with an assembly or read reference (the k-mer set is not empty)");
        return FL_EINVAL;
    }
    if (ctx->contam.n > 0 && !(ctx->p.max_contam >= 0.0 && ctx->p.max_contam < 100.0)) {
        ctx->set_error("max_contam must be at least 0 and less than 100 when the contaminant set is not empty");
        return FL_EINVAL;
    }
    return FL_OK;
}

// --contam, before the batch is scored: its reads' contaminant percentages and removal flags (r_contam, r_removed)
static int contam_reads(fl_ctx *ctx, const BatchView &b) {
    if (!b.seq2b) { ctx->set_error("a contaminant set needs the reads' bases (seq2b or ascii)"); return FL_EINVAL; }
    const size_t rb = ctx->n_reads, n = b.n;
    cudaStream_t st = ctx->stream;
    FL_CUDA(ctx, ctx->r_contam.reserve(rb + n, rb, st));
    FL_CUDA(ctx, ctx->r_removed.reserve(rb + n, rb, st));
    FL_CUDA(ctx, ctx->sc_cmask.reserve((size_t)(b.padded_bases >> 5) + 1, 0, st));
    FL_TRY(fl_probe_paint(ctx, ctx->contam, b, ctx->sc_cmask.p, FL_KERNEL_CONTAM));
    {
        KernelTimer kt(ctx, FL_KERNEL_CONTAM);
        k_contam_reads<<<scan_blocks_of(ctx, n), 256, 0, st>>>(ctx->sc_cmask.p, b.off, b.len, b.n, ctx->p.max_contam,
                                                               ctx->r_contam.p + rb, ctx->r_removed.p + rb);
    }
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

// --contam, once rows [row0, n_rows) exist: those of removed reads are excluded
static int contam_rows(fl_ctx *ctx, size_t row0) {
    if (ctx->contam.n == 0 || ctx->n_rows == row0) return FL_OK;
    const size_t n = ctx->n_rows - row0;
    FL_CUDA(ctx, ctx->w_excl.reserve(ctx->n_rows, row0, ctx->stream));
    unsigned blocks = fl_blocks(n, 256);
    if (blocks > (unsigned)ctx->sm_count * 8) blocks = (unsigned)ctx->sm_count * 8;
    {
        KernelTimer kt(ctx, FL_KERNEL_CONTAM);
        k_contam_rows<<<blocks, 256, 0, ctx->stream>>>(ctx->w_parent.p + row0, ctx->r_removed.p, n, ctx->w_passed.p + row0,
                                                       ctx->w_excl.p + row0);
    }
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

int fl_score_view(fl_ctx *ctx, const BatchView &b, bool defer) {
    if (b.n == 0) return FL_OK;
    FL_TRY(fl_sets_ready(ctx));
    FL_TRY(fl_check_trim_q(ctx));
    ctx->finalized = false;
    if (ctx->contam.n > 0) FL_TRY(contam_reads(ctx, b));
    const size_t row0 = ctx->n_rows;
    const bool rows = ctx->p.trim || ctx->p.split_set;
    const bool qual = ctx->ref.n == 0;
    if (qual && !(rows && ctx->p.trim_q > 0)) {                  // read.cpp:35: kmers->empty()
        FL_TRY(fl_score_phred(ctx, b));
        return contam_rows(ctx, row0);
    }
    if (qual) FL_TRY(score_qual_front(ctx, b));
    else FL_TRY(score_kmer_front(ctx, b));
    if (defer && rows) {
        ctx->kmer_pending = true;
        ctx->pending_qual = qual;
        ctx->kmer_pending_view = b;
        return FL_OK;
    }
    FL_TRY(qual ? score_qual_back(ctx, b) : score_kmer_back(ctx, b));
    return contam_rows(ctx, row0);
}

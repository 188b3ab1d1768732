// filtlong_b200/csrc/fl_kmers.cu -- device-built, device-resident reference 16-mer set.
//
// Replaces Kmers (reference src/kmers.cpp:28-239). The key space is exactly 2^32, so membership is
// a direct-address bitmap (512 MiB of the 80 GB HBM3): no collisions, no rehash, one 32-byte
// sector per probe. Two build modes:
//
//   one copy        (kmers.cpp:137-139, assembly):  every forward / reverse 16-mer -> atomicOr.
//   multiple copies (kmers.cpp:142-166, short reads): the reference's sequential state machine
//       "set? skip | Bloom miss -> Bloom insert | Bloom hit, uncounted -> count=2 | ++count, >=4 ->
//       set" is order dependent only through Bloom false positives. In closed, order-free form
//       (derivation in DESIGN.md / SURVEY H4): give every add its index t in the add stream
//       (file, record, position, forward before reverse: kmers.cpp:54-55,109-120); per k-mer X
//       keep cnt(X) (saturating at 4) and t_first(X); per Bloom bit keep
//       bit_time[b] = min over X with b in bits(X) of t_first(X); then
//           FP(X)  <=>  for all 13 hashes j: bit_time[b_j(X)] < t_first(X)
//           X in set  <=>  cnt(X) >= 4  or  (cnt(X) == 3 and FP(X)).
//       cnt lives in four "seen >= i" bitmaps (2 GiB), t_first and bit_time in direct-address
//       arrays (32 GiB + 15 GiB) -- transient, released after the build.
#include "fl_device.cuh"

namespace {

__constant__ uint32_t c_salts[FL_BLOOM_K] = {   // bloom_filter.h:183-195,519-528 as configured by kmers.cpp:32-36
    0x1B5793D2u, 0x81BDFA38u, 0xEB8E30D5u, 0x45B52496u, 0x85C1FE3Cu, 0x3DACB627u, 0x78776869u,
    0x94A40D1Eu, 0x5F9BB638u, 0x40FB59D5u, 0x8174BDB2u, 0x0B466EAAu, 0x209D29A7u};

struct BuildArgs {
    const uint32_t *seq2b;
    const uint32_t *nmask;
    const uint64_t *off;
    const int32_t *len;
    const unsigned long long *tile_start;   // [n+1]
    const unsigned long long *add_start;    // [n] add-stream index of the sequence's first add
    uint32_t n;
    unsigned long long n_tiles;
    uint32_t *bitmap;
    uint32_t *seen0, *seen1, *seen2, *seen3;
    unsigned long long *tfirst;
    unsigned long long add_base;
};

__device__ __forceinline__ void set_bit(uint32_t *bm, uint32_t k) {
    uint32_t bit = 1u << (k & 31);
    uint32_t *w = bm + (k >> 5);
    if (!(*w & bit)) atomicOr(w, bit);
}

__device__ __forceinline__ bool has_bit(const uint32_t *bm, uint32_t k) { return (bm[k >> 5] >> (k & 31)) & 1u; }

// claim exactly one new "seen" level for this add (linearizable saturating counter)
__device__ __forceinline__ void bump_seen(const BuildArgs &a, uint32_t k) {
    uint32_t bit = 1u << (k & 31);
    size_t w = k >> 5;
    uint32_t *lv[4] = {a.seen0, a.seen1, a.seen2, a.seen3};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (lv[i][w] & bit) continue;
        uint32_t old = atomicOr(lv[i] + w, bit);
        if (!(old & bit)) return;
    }
}

template <bool MULTI>
__device__ __forceinline__ void add_kmer(const BuildArgs &a, uint32_t k, unsigned long long t) {
    if (!MULTI) {
        set_bit(a.bitmap, k);                          // kmers.cpp:137-139
    } else {
        if (has_bit(a.bitmap, k)) return;              // kmers.cpp:144-145 (assembly / earlier promotions)
        if (t < a.tfirst[k]) atomicMin(a.tfirst + k, t);
        bump_seen(a, k);
    }
}

template <bool MULTI>
__global__ void __launch_bounds__(256) k_kmers_add(BuildArgs a) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    for (unsigned long long tile = warp; tile < a.n_tiles; tile += n_warps) {
        uint32_t s = fl_find_seq(a.tile_start, a.n, tile);
        int L = a.len[s];
        if (L < FL_K) continue;                        // kmers.cpp:99-100
        unsigned long long off = a.off[s];
        const uint32_t *seqw = a.seq2b + (off >> 4);
        const uint32_t *nm = a.nmask ? a.nmask + (off >> 5) : nullptr;
        unsigned long long padded = ((unsigned long long)L + FL_ALIGN_BASES - 1) & ~(unsigned long long)(FL_ALIGN_BASES - 1);
        unsigned long long tile_base = (tile - a.tile_start[s]) * FL_TILE_BASES;
        unsigned long long t0 = MULTI ? a.add_base + a.add_start[s] : 0ull;
        for (int step = 0; step < FL_TILE_STEPS; ++step) {
            unsigned long long sb = tile_base + (unsigned long long)step * FL_STEP_BASES;
            if (sb >= (unsigned long long)L) break;
            LaneWords w = fl_load_lane_words(seqw, sb, padded, lane);
            unsigned long long lb = sb + 32ull * lane;   // first base of the lane's run
            uint32_t m0 = 0, m1 = 0;
            if (nm) {
                m0 = (lb < padded) ? __ldg(nm + (lb >> 5)) : 0u;
                m1 = (lb + 32 < padded) ? __ldg(nm + ((lb + 32) >> 5)) : 0u;
            }
            unsigned long long mm = ((unsigned long long)m1 << 32) | m0;
#pragma unroll 4
            for (int p = 0; p < 32; ++p) {
                unsigned long long b = lb + p;           // k-mer start; valid if b + 15 < L
                if (b + (FL_K - 1) >= (unsigned long long)L) break;
                uint32_t fwd = fl_kmer_at(w, p);
                uint32_t rev = fl_reverse_pairs(~fwd);   // complement, newest base on top (kmers.cpp:115-116)
                uint32_t nb = (uint32_t)(mm >> p) & 0xFFFFu;
                if (nb) rev &= ~(fl_spread16(nb) * 3u);  // non-ACGT -> 0 on the reverse strand (kmers.cpp:199-219)
                add_kmer<MULTI>(a, fwd, t0 + 2ull * b);          // forward first (kmers.cpp:109,119)
                add_kmer<MULTI>(a, rev, t0 + 2ull * b + 1ull);   // then reverse (kmers.cpp:110,120)
            }
        }
    }
}

__global__ void k_tiles_and_adds(const int32_t *__restrict__ len, uint32_t n, unsigned long long *__restrict__ tiles,
                                 unsigned long long *__restrict__ adds) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int L = len[i];
    tiles[i] = fl_tiles_of(L);
    if (adds) adds[i] = L >= FL_K ? 2ull * (unsigned long long)(L - (FL_K - 1)) : 0ull;
}

// pass 2 of the multiple-copy resolution: bit_time[b] = min t_first over k-mers touching b
__global__ void __launch_bounds__(256) k_bloom_times(const uint32_t *__restrict__ seen0,
                                                     const unsigned long long *__restrict__ tfirst,
                                                     unsigned long long *__restrict__ bittime) {
    const size_t n_words = (size_t)1 << 27;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (size_t)gridDim.x * blockDim.x) {
        uint32_t bits = seen0[w];
        while (bits) {
            int b = __ffs(bits) - 1;
            bits &= bits - 1;
            uint32_t k = (uint32_t)(w << 5) | (uint32_t)b;
            unsigned long long t = tfirst[k];
#pragma unroll
            for (int j = 0; j < FL_BLOOM_K; ++j) {
                unsigned long long idx = fl_bloom_hash(k, c_salts[j]) % FL_BLOOM_BITS;
                if (t < bittime[idx]) atomicMin(bittime + idx, t);
            }
        }
    }
}

// pass 3: promote cnt >= 4, and cnt == 3 with a Bloom false positive on the first sighting
__global__ void __launch_bounds__(256) k_promote(const uint32_t *__restrict__ seen2, const uint32_t *__restrict__ seen3,
                                                 const unsigned long long *__restrict__ tfirst,
                                                 const unsigned long long *__restrict__ bittime,
                                                 uint32_t *__restrict__ bitmap) {
    const size_t n_words = (size_t)1 << 27;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (size_t)gridDim.x * blockDim.x) {
        uint32_t s3 = seen2[w];
        if (!s3) continue;
        uint32_t s4 = seen3[w];
        uint32_t promote = s4;
        uint32_t bits = s3 & ~s4;          // exactly three sightings
        while (bits) {
            int b = __ffs(bits) - 1;
            bits &= bits - 1;
            uint32_t k = (uint32_t)(w << 5) | (uint32_t)b;
            unsigned long long t = tfirst[k];
            bool fp = true;
#pragma unroll
            for (int j = 0; j < FL_BLOOM_K; ++j) {
                unsigned long long idx = fl_bloom_hash(k, c_salts[j]) % FL_BLOOM_BITS;
                if (!(bittime[idx] < t)) { fp = false; break; }
            }
            if (fp) promote |= 1u << b;
        }
        if (promote) bitmap[w] |= promote;
    }
}

__global__ void __launch_bounds__(256) k_popcount(const uint32_t *__restrict__ bm, size_t n_words,
                                                  unsigned long long *__restrict__ out) {
    unsigned long long c = 0;
    const uint4 *v = reinterpret_cast<const uint4 *>(bm);
    size_t n4 = n_words >> 2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        uint4 x = v[i];
        c += __popc(x.x) + __popc(x.y) + __popc(x.z) + __popc(x.w);
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) c += __shfl_down_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

// pre-filter build: every member of the bitmap sets its two filter bits
__global__ void __launch_bounds__(256) k_filter_build(const uint32_t *__restrict__ bm, unsigned long long *__restrict__ filter,
                                                      unsigned log2_words, int kind) {
    const size_t n_words = (size_t)1 << 27;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (size_t)gridDim.x * blockDim.x) {
        uint32_t bits = bm[w];
        while (bits) {
            const int b = __ffs(bits) - 1;
            bits &= bits - 1;
            const uint32_t kmer = (uint32_t)(w << 5) | (uint32_t)b;
            if (kind & 4) {                                  // group of 4: once per alignment, like the anchored table
#pragma unroll
                for (unsigned r = 0; r < 4; ++r) {
                    const uint32_t word = fl_filter_word_group4(kmer, r, log2_words);
                    const unsigned long long fb = fl_filter_bits_role(kmer, r, kind);
                    if ((filter[word] & fb) != fb) atomicOr(filter + word, fb);
                }
            } else if (kind & 8) {                           // pair: as the earlier and as the later neighbour
#pragma unroll
                for (unsigned role = 0; role < 2; ++role) {
                    const uint32_t word = fl_filter_word_pair(kmer, role, log2_words);
                    const unsigned long long fb = fl_filter_bits_role(kmer, role, kind);
                    if ((filter[word] & fb) != fb) atomicOr(filter + word, fb);
                }
            } else {
                uint32_t word;
                unsigned long long fb;
                fl_filter_slot(kmer, log2_words, kind, word, fb);
                if ((filter[word] & fb) != fb) atomicOr(filter + word, fb);
            }
        }
    }
}

// anchored table build: every member of the bitmap is entered once per alignment (fl_anchor_slot)
__global__ void __launch_bounds__(256) k_anchor_build(const uint32_t *__restrict__ bm, uint32_t *__restrict__ anchor) {
    const size_t n_words = (size_t)1 << 27;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (size_t)gridDim.x * blockDim.x) {
        uint32_t bits = bm[w];
        while (bits) {
            const int b = __ffs(bits) - 1;
            bits &= bits - 1;
            const uint32_t kmer = (uint32_t)(w << 5) | (uint32_t)b;
#pragma unroll
            for (unsigned r = 0; r < 4; ++r) {
                uint32_t word, bit;
                fl_anchor_slot(kmer, r, word, bit);
                atomicOr(anchor + word, 1u << bit);
            }
        }
    }
}

__global__ void k_contains(const uint32_t *__restrict__ bm, const uint32_t *__restrict__ q, uint32_t n,
                           uint8_t *__restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (bm[q[i] >> 5] >> (q[i] & 31)) & 1u;
}

}  // namespace

int fl_kmers_ensure_bitmap(fl_ctx *ctx) {
    if (ctx->d_bitmap) return FL_OK;
    FL_CUDA(ctx, cudaMalloc(&ctx->d_bitmap, (size_t)1 << 29));
    FL_CUDA(ctx, cudaMemsetAsync(ctx->d_bitmap, 0, (size_t)1 << 29, ctx->stream));
    return FL_OK;
}

static void free_multi_state(fl_ctx *ctx) {
    for (int i = 0; i < 4; ++i) {
        if (ctx->d_seen[i]) cudaFree(ctx->d_seen[i]);
        ctx->d_seen[i] = nullptr;
    }
    if (ctx->d_tfirst) cudaFree(ctx->d_tfirst);
    if (ctx->d_bittime) cudaFree(ctx->d_bittime);
    ctx->d_tfirst = nullptr;
    ctx->d_bittime = nullptr;
}

// all or nothing: a partial allocation failure frees what was taken, so a later call starts clean
static int ensure_multi_state(fl_ctx *ctx) {
    if (ctx->d_tfirst && ctx->d_bittime && ctx->d_seen[0] && ctx->d_seen[1] && ctx->d_seen[2] && ctx->d_seen[3]) return FL_OK;
    free_multi_state(ctx);
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = cudaMalloc(&ctx->d_seen[i], (size_t)1 << 29);
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_tfirst, ((size_t)1 << 32) * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_bittime, (size_t)FL_BLOOM_BITS * sizeof(unsigned long long));
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = cudaMemsetAsync(ctx->d_seen[i], 0, (size_t)1 << 29, ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(ctx->d_tfirst, 0xFF, ((size_t)1 << 32) * sizeof(unsigned long long), ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(ctx->d_bittime, 0xFF, (size_t)FL_BLOOM_BITS * sizeof(unsigned long long), ctx->stream);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        free_multi_state(ctx);
        ctx->set_error(std::string("multiple-copy build state (49 GiB): ") + cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? FL_ENOMEM : FL_ECUDA;
    }
    return FL_OK;
}

int fl_kmers_add_view(fl_ctx *ctx, const BatchView &b, int multi) {
    if (b.n == 0) return FL_OK;
    if (!b.seq2b) { ctx->set_error("fl_kmers_add_batch: seq2b is required"); return FL_EINVAL; }
    FL_TRY(fl_kmers_ensure_bitmap(ctx));
    if (multi) FL_TRY(ensure_multi_state(ctx));
    size_t n = b.n;
    FL_CUDA(ctx, ctx->sc_u64a.reserve(n + 1, 0, ctx->stream));
    FL_CUDA(ctx, ctx->sc_u64b.reserve(n + 1, 0, ctx->stream));
    k_tiles_and_adds<<<fl_blocks(n, 256), 256, 0, ctx->stream>>>(b.len, b.n, ctx->sc_u64a.p, multi ? ctx->sc_u64b.p : nullptr);
    ctx->launches++;
    unsigned long long *totals = ctx->d_scalars;   // [0] tiles, [1] adds
    FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64a.p, ctx->sc_u64a.p, n, totals));
    if (multi) FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64b.p, ctx->sc_u64b.p, n, totals + 1));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->sc_u64a.p + n, totals, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, ctx->stream));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars, totals, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    unsigned long long n_tiles = ctx->h_scalars[0];
    unsigned long long n_adds = multi ? ctx->h_scalars[1] : 0;
    if (n_tiles == 0) return FL_OK;

    BuildArgs a{};
    a.seq2b = b.seq2b; a.nmask = b.nmask; a.off = b.off; a.len = b.len;
    a.tile_start = ctx->sc_u64a.p; a.add_start = ctx->sc_u64b.p;
    a.n = b.n; a.n_tiles = n_tiles; a.bitmap = ctx->d_bitmap;
    a.seen0 = ctx->d_seen[0]; a.seen1 = ctx->d_seen[1]; a.seen2 = ctx->d_seen[2]; a.seen3 = ctx->d_seen[3];
    a.tfirst = ctx->d_tfirst; a.add_base = ctx->add_counter;
    unsigned long long warps_needed = n_tiles;
    unsigned blocks = (unsigned)((warps_needed + 7) / 8);
    unsigned max_blocks = (unsigned)ctx->sm_count * 8;
    if (blocks > max_blocks) blocks = max_blocks;
    {
        KernelTimer kt(ctx, FL_KERNEL_KMERS_ADD);
        if (multi) k_kmers_add<true><<<blocks, 256, 0, ctx->stream>>>(a);
        else k_kmers_add<false><<<blocks, 256, 0, ctx->stream>>>(a);
    }
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    if (multi) {
        ctx->add_counter += n_adds;
        ctx->multi_pending = true;
    }
    ctx->kmers_count_stale = true;
    return FL_OK;
}

int fl_kmers_recount(fl_ctx *ctx) {
    if (!ctx->d_bitmap) { ctx->n_kmers = 0; ctx->kmers_count_stale = false; return FL_OK; }
    if (ctx->multi_pending) {
        unsigned blocks = (unsigned)ctx->sm_count * 16;
        k_bloom_times<<<blocks, 256, 0, ctx->stream>>>(ctx->d_seen[0], ctx->d_tfirst, ctx->d_bittime);
        k_promote<<<blocks, 256, 0, ctx->stream>>>(ctx->d_seen[2], ctx->d_seen[3], ctx->d_tfirst, ctx->d_bittime, ctx->d_bitmap);
        ctx->launches += 2;
        ctx->multi_pending = false;
    }
    FL_CUDA(ctx, cudaMemsetAsync(ctx->d_scalars, 0, sizeof(unsigned long long), ctx->stream));
    k_popcount<<<(unsigned)ctx->sm_count * 8, 256, 0, ctx->stream>>>(ctx->d_bitmap, (size_t)1 << 27, ctx->d_scalars);
    ctx->launches++;
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars, ctx->d_scalars, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->n_kmers = ctx->h_scalars[0];
    ctx->kmers_count_stale = false;
    // The pre-filter is used while it has filter_min_bits_per_key bits per member (fl_internal.cuh: on the H100 a 20 M-member
    // set probes faster without it). Larger sets (config 3's, or a 3 Gbp assembly that fills 75 % of the key space) are
    // probed directly.
    const size_t filter_words = (size_t)1 << ctx->filter_log2_words;
    ctx->use_filter = ctx->filter_enabled && ctx->n_kmers > 0 && ctx->n_kmers * (uint64_t)ctx->filter_min_bits_per_key <= filter_words * 64;
    // Which flavour: the probe kernel is bound by L1TEX sector look-ups on a sparse set, one per filter word it loads, so a
    // word shared by the four 16-mers of a table group (or by two neighbours) cuts them 4x (2x) -- at 4x (2x) the insertions.
    // Small sets can afford that (false positives, each a wasted random HBM sector, stay below ~5 %); the thresholds
    // (filter_group4_max, filter_pair_max) come from a sweep of config 3's reads against sets of 5 to 20 M members.
    if (ctx->filter_kind_request >= 0) ctx->filter_kind = ctx->filter_kind_request;
    else if (!ctx->anchor_enabled) ctx->filter_kind = 2 | 16;
    else if (ctx->n_kmers <= ctx->filter_group4_max) ctx->filter_kind = 2 | 4 | 16;
    else if (ctx->n_kmers <= ctx->filter_pair_max) ctx->filter_kind = 2 | 8 | 16;
    else ctx->filter_kind = 2 | 16;
    if (!ctx->anchor_enabled) ctx->filter_kind &= ~(4 | 8);        // the keyed flavours follow the anchored table's groups
    if (ctx->use_filter) {
        if (!ctx->d_filter) FL_CUDA(ctx, cudaMalloc(&ctx->d_filter, filter_words * sizeof(unsigned long long)));
        FL_CUDA(ctx, cudaMemsetAsync(ctx->d_filter, 0, filter_words * sizeof(unsigned long long), ctx->stream));
        k_filter_build<<<(unsigned)ctx->sm_count * 16, 256, 0, ctx->stream>>>(ctx->d_bitmap, ctx->d_filter, ctx->filter_log2_words, ctx->filter_kind);
        ctx->launches++;
        FL_CUDA(ctx, cudaGetLastError());
    }
    // the table the probe kernel reads: one 32-byte sector per four consecutive 16-mers of a read
    ctx->use_anchor = ctx->anchor_enabled && ctx->n_kmers > 0;
    if (ctx->use_anchor) {
        const size_t anchor_bytes = (size_t)1 << 31;
        if (!ctx->d_anchor) FL_CUDA(ctx, cudaMalloc(&ctx->d_anchor, anchor_bytes));
        FL_CUDA(ctx, cudaMemsetAsync(ctx->d_anchor, 0, anchor_bytes, ctx->stream));
        k_anchor_build<<<(unsigned)ctx->sm_count * 16, 256, 0, ctx->stream>>>(ctx->d_bitmap, ctx->d_anchor);
        ctx->launches++;
        FL_CUDA(ctx, cudaGetLastError());
    }
    return FL_OK;
}

// ---- C ABI ------------------------------------------------------------------------------------
extern "C" int fl_kmers_finalize(fl_ctx *ctx, uint64_t *n_kmers_out) {
    FL_ENTER(ctx);
    if (ctx->kmers_count_stale || ctx->multi_pending) FL_TRY(fl_kmers_recount(ctx));
    if (n_kmers_out) *n_kmers_out = ctx->n_kmers;
    return FL_OK;
}

extern "C" int fl_kmers_contains(fl_ctx *ctx, const uint32_t *kmers, uint32_t n, uint8_t *out) {
    if (!ctx || (!kmers && n) || (!out && n)) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_TRY(fl_kmers_finalize(ctx, nullptr));
    if (n == 0) return FL_OK;
    if (!ctx->d_bitmap) { memset(out, 0, n); return FL_OK; }
    FL_CUDA(ctx, ctx->sc_u32a.reserve((size_t)n + (n + 3) / 4, 0, ctx->stream));
    uint32_t *dq = ctx->sc_u32a.p;
    uint8_t *dout = reinterpret_cast<uint8_t *>(dq + n);
    FL_CUDA(ctx, cudaMemcpyAsync(dq, kmers, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    k_contains<<<fl_blocks(n, 256), 256, 0, ctx->stream>>>(ctx->d_bitmap, dq, n, dout);
    ctx->launches++;
    FL_CUDA(ctx, cudaMemcpyAsync(out, dout, n, cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return FL_OK;
}

extern "C" int fl_kmers_export(fl_ctx *ctx, uint32_t *out, uint64_t cap, uint64_t *n_out) {
    FL_ENTER(ctx);
    FL_TRY(fl_kmers_finalize(ctx, nullptr));
    if (n_out) *n_out = ctx->n_kmers;
    if (!ctx->d_bitmap || !out || cap == 0) return FL_OK;
    std::vector<uint32_t> host((size_t)1 << 27);
    FL_CUDA(ctx, cudaMemcpyAsync(host.data(), ctx->d_bitmap, (size_t)1 << 29, cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    uint64_t k = 0;
    for (size_t w = 0; w < host.size() && k < cap; ++w) {
        uint32_t bits = host[w];
        while (bits && k < cap) {
            int b = __builtin_ctz(bits);
            bits &= bits - 1;
            out[k++] = (uint32_t)(w << 5) | (uint32_t)b;
        }
    }
    return FL_OK;
}

extern "C" int fl_kmers_bitmap_dev(fl_ctx *ctx, void **dev_ptr, uint64_t *n_bytes) {
    if (!ctx || !dev_ptr) return FL_EINVAL;
    FL_ENTER(ctx);
    FL_TRY(fl_kmers_ensure_bitmap(ctx));
    *dev_ptr = ctx->d_bitmap;
    if (n_bytes) *n_bytes = (uint64_t)1 << 29;
    return FL_OK;
}

extern "C" int fl_kmers_bitmap_changed(fl_ctx *ctx) {
    FL_ENTER(ctx);
    ctx->kmers_count_stale = true;
    return FL_OK;
}

extern "C" int fl_kmers_probe_info(fl_ctx *ctx, int32_t info[4]) {
    FL_ENTER(ctx);
    if (!info) return FL_EINVAL;
    if (ctx->kmers_count_stale || ctx->multi_pending) FL_TRY(fl_kmers_recount(ctx));
    info[0] = ctx->use_filter ? 1 : 0;
    info[1] = ctx->filter_kind;
    info[2] = (int32_t)ctx->filter_log2_words;
    info[3] = ctx->use_anchor ? 1 : 0;
    return FL_OK;
}

extern "C" int fl_kmers_release_build_state(fl_ctx *ctx) {
    FL_ENTER(ctx);
    if (ctx->multi_pending) FL_TRY(fl_kmers_recount(ctx));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    free_multi_state(ctx);
    return FL_OK;
}

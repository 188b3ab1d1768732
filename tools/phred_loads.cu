// tools/phred_loads.cu -- load-only probes for tools/phred_loads.py. Not part of the library.
//
// Each probe walks the quality arena the way k_phred_sum (KIND 0) or k_phred_win's filter pass (KIND 1, window 250,
// 8 bases per lane) does -- one warp per read, reads claimed from a shared counter through `order`, the same
// addresses, the same block size and dynamic shared memory, as many blocks per SM as the kernel has or as fit -- and
// does nothing with the bytes but XOR them into one word per read. What is left is the time the loads take, by mechanism:
//   MODE 0  one step ahead in registers: a uint4 per lane (KIND 0), three clamped 32-bit words per lane (KIND 1)
//   MODE 1  a ring of D tiles of 512 bytes per warp in shared memory, filled by lane 0 with cp.async.bulk
//   MODE 2  the same ring, filled by every lane with 16-byte cp.async
//   MODE 3  (KIND 0 only) what k_phred_sum does: D private 16-byte slots per lane, each lane copying its own chunk of
//           the step D ahead with cp.async and one commit group per step, cp.async.wait_group D-1 before reading a
//           slot; no barrier, no producer lane, a cold start per read
// DEEP: the warp holds the next read's descriptor while it walks this one, the ring is refilled across the read
// boundary, and short reads are claimed eight per atomicAdd. Without it a read starts cold.
// k_chunked (below): the same walks cut into chunks, with a bulk L2 prefetch ahead, and both walks in one pass.
#include <cstdint>
#include <cuda_runtime.h>

#define THREADS 256
#define TILE 512
#define FULL 0xffffffffu

struct Args {
    const uint8_t *qual;
    const unsigned long long *off;
    const int32_t *len;
    const uint32_t *order;
    uint32_t n;
    unsigned long long *work;
    uint32_t *out;
    int table_bytes;      // dynamic shared memory the real kernel's tables take: the ring starts behind it
};

__device__ __forceinline__ bool mbar_done(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0u;
}

template <int MODE, int D, bool DEEP>
struct Feed {
    uint32_t d_r, d_o, qtail, ci, pq, iss, po, cseq, ring, bars;
    int d_L, ppos, pend, ready, freed, start;
    bool done;

    __device__ void init(unsigned char *ring_all, unsigned long long *bars_all, int start_, unsigned lane) {
        const unsigned warp = threadIdx.x >> 5;
        ring = (uint32_t)__cvta_generic_to_shared(ring_all + warp * (TILE * D));
        bars = (uint32_t)__cvta_generic_to_shared(bars_all + warp * D);
        if (lane < D) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bars + 8u * lane), "r"(MODE == 1 ? 1 : 32) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        d_r = d_o = 0u; d_L = 0; qtail = ci = 0u; done = false;
        pq = 0xFFFFFFFFu; iss = po = 0u; ppos = pend = 0; cseq = 0u; ready = freed = 0; start = start_;
    }
    __device__ int tiles_of(int L) const { return (((L + 63) & ~63) - start + TILE - 1) / TILE; }
    __device__ void claim(const Args &a, int skip_len, unsigned lane) {
        const unsigned cn = (DEEP && qtail != 0u && __shfl_sync(FULL, d_L, (qtail - 1u) & 31u) < 4096) ? 8u : 1u;
        unsigned long long it = 0;
        if (lane == 0) it = atomicAdd(a.work, (unsigned long long)cn);
        it = __shfl_sync(FULL, it, 0);
        const unsigned k = (lane - qtail) & 31u;
        if (k < cn) {
            d_L = 0;
            if (it + k < a.n) {
                const uint32_t r = a.order[it + k];
                const int L = a.len[r];
                if (L > skip_len) { d_r = r; d_L = L; d_o = (uint32_t)(a.off[r] >> 6); }
            }
        }
        qtail += cn;
        done = it + cn >= a.n;
    }
    __device__ void produce(const uint8_t *qual, unsigned lane) {
        for (;;) {
            if (iss - (cseq + (uint32_t)freed) >= (uint32_t)D) break;
            if (ppos >= pend) {
                if (pq + 1u == qtail) break;
                ++pq;
                const int L = __shfl_sync(FULL, d_L, pq & 31u);
                po = __shfl_sync(FULL, d_o, pq & 31u);
                ppos = start;
                pend = L ? (L + 63) & ~63 : 0;
                continue;
            }
            const uint32_t stage = iss & (D - 1), bar = bars + 8u * stage;
            const int bytes = min(TILE, pend - ppos);
            const uint8_t *src = qual + ((unsigned long long)po << 6) + ppos;
            if (MODE == 1) {
                if (lane == 0) {
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"(ring + stage * TILE), "l"(src), "r"(bytes), "r"(bar) : "memory");
                }
            } else {
                if (16 * (int)lane < bytes)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(ring + stage * TILE + 16u * lane), "l"(src + 16 * lane) : "memory");
                asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
            }
            ppos += TILE;
            ++iss;
        }
    }
    __device__ bool next(const Args &a, int skip_len, unsigned lane, uint32_t &r, int &L, const uint8_t *&q) {
        for (;;) {
            while (!done && qtail - ci < (DEEP ? 2u : 1u)) claim(a, skip_len, lane);
            produce(a.qual, lane);
            if (ci == qtail) return false;
            L = __shfl_sync(FULL, d_L, ci & 31u);
            if (L) break;
            ++ci;
        }
        r = __shfl_sync(FULL, d_r, ci & 31u);
        q = a.qual + ((unsigned long long)__shfl_sync(FULL, d_o, ci & 31u) << 6);
        return true;
    }
    __device__ void wait(int need) {
        while (ready < need) {
            const uint32_t t = cseq + (uint32_t)ready;
            while (!mbar_done(bars + 8u * (t & (D - 1)), (t / D) & 1u)) {}
            ++ready;
        }
    }
    __device__ void release(int upto, const uint8_t *qual, unsigned lane) {
        wait(upto);
        __syncwarp();
        freed = upto;
        produce(qual, lane);
    }
    __device__ void end_read(int L, const uint8_t *qual, unsigned lane) {
        const int nt = tiles_of(L);
        while (freed < nt) release(freed + 1, qual, lane);
        cseq += (uint32_t)nt;
        ready = freed = 0;
        ++ci;
    }
    __device__ uint32_t at(uint32_t p) const { return ring + ((cseq * TILE + p) & (TILE * D - 1)); }
};

__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}

// KIND 0: k_phred_sum's walk (16 bytes per lane per 512-byte step from byte H on). KIND 1: k_phred_win's filter
// pass (window WS, K bytes per lane per step, three words at byte j + K lane, from byte 0 on).
#define H 256
#define WS 250
#define K 8
#define NW 2

template <int KIND, int MODE, int D, bool DEEP>
__global__ void __launch_bounds__(THREADS) k_probe(Args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ unsigned long long s_bar[THREADS / 32][D];
    const unsigned lane = threadIdx.x & 31;
    // the real kernels fill their tables here; the probe only owns the space
    for (int i = threadIdx.x; i < a.table_bytes / 4; i += blockDim.x) reinterpret_cast<uint32_t *>(smem_raw)[i] = 0u;
    __syncthreads();
    const int skip = KIND == 0 ? H : WS;
    if constexpr (MODE == 3) {
        static_assert(KIND == 0, "per-lane slots: k_phred_sum's walk only");
        const uint32_t slot0 = (uint32_t)__cvta_generic_to_shared(smem_raw + a.table_bytes) + 16u * threadIdx.x;
        for (;;) {
            unsigned long long it = 0;
            if (lane == 0) it = atomicAdd(a.work, 1ull);
            it = __shfl_sync(FULL, it, 0);
            if (it >= a.n) break;
            const uint32_t r = a.order[it];
            const int L = a.len[r];
            if (L <= skip) continue;
            const uint8_t *ql = a.qual + a.off[r] + 16 * lane;
#pragma unroll
            for (int d = 0; d < D; ++d) {
                if (TILE * d + 16 * (int)lane < L - H)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot0 + d * (THREADS * 16)), "l"(ql + H + TILE * d) : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
            }
            uint32_t x = 0, slot = slot0;
            for (int j = H; j < L; j += TILE) {
                uint32_t c0, c1, c2, c3;
                asm volatile("cp.async.wait_group %4;\n\tld.shared.v4.u32 {%0, %1, %2, %3}, [%5];"
                             : "=r"(c0), "=r"(c1), "=r"(c2), "=r"(c3) : "n"(D - 1), "r"(slot) : "memory");
                if (D * TILE + 16 * (int)lane < L - j)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot), "l"(ql + j + D * TILE) : "memory");
                asm volatile("cp.async.commit_group;" ::: "memory");
                slot = slot == slot0 + (D - 1) * (THREADS * 16) ? slot0 : slot + THREADS * 16;
                x ^= c0 ^ c1 ^ c2 ^ c3;          // (a lane past the read's end reads a stale slot: not compared either)
            }
            x = __reduce_xor_sync(FULL, x);
            if (lane == 0) a.out[r] = x;
        }
    } else if (MODE == 0) {
        for (;;) {
            unsigned long long it = 0;
            if (lane == 0) it = atomicAdd(a.work, 1ull);
            it = __shfl_sync(FULL, it, 0);
            if (it >= a.n) break;
            const uint32_t r = a.order[it];
            const int L = a.len[r];
            if (L <= skip) continue;
            const uint8_t *q = a.qual + a.off[r];
            uint32_t x = 0;
            if (KIND == 0) {
                const uint4 *qv = reinterpret_cast<const uint4 *>(q);
                uint4 pre = make_uint4(0u, 0u, 0u, 0u);
                if (H + 16 * (int)lane < L) pre = __ldg(qv + ((H >> 4) + (int)lane));
                for (int j = H; j < L; j += TILE) {
                    x ^= pre.x ^ pre.y ^ pre.z ^ pre.w;
                    const int pn = j + TILE + 16 * (int)lane;
                    if (pn < L) pre = __ldg(qv + (pn >> 4));
                }
            } else {
                const uint32_t *q32 = reinterpret_cast<const uint32_t *>(q);
                const int maxword = (((L + 63) & ~63) >> 2) - 1;
                uint32_t pre[NW + 1];
#pragma unroll
                for (int i = 0; i <= NW; ++i) pre[i] = __ldg(q32 + min(((K * (int)lane) >> 2) + i, maxword));
                for (int j = 0; j < L; j += WS) {
                    x ^= pre[0] ^ pre[1] ^ pre[2];
                    if (j + WS < L) {
#pragma unroll
                        for (int i = 0; i <= NW; ++i) pre[i] = __ldg(q32 + min(((j + WS + K * (int)lane) >> 2) + i, maxword));
                    }
                }
            }
            x = __reduce_xor_sync(FULL, x);
            if (lane == 0) a.out[r] = x;
        }
    } else {
        Feed<MODE, D, DEEP> feed;
        feed.init(smem_raw + a.table_bytes, &s_bar[0][0], KIND == 0 ? H : 0, lane);
        for (;;) {
            uint32_t r;
            int L;
            const uint8_t *q;
            if (!feed.next(a, skip, lane, r, L, q)) break;
            uint32_t x = 0;
            if (KIND == 0) {
                for (int j = H, tile = 0; j < L; j += TILE, ++tile) {
                    feed.wait(tile + 1);
                    uint32_t c0, c1, c2, c3;
                    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(c0), "=r"(c1), "=r"(c2), "=r"(c3)
                                 : "r"(feed.at((uint32_t)(j - H)) + 16u * lane) : "memory");
                    feed.release(tile + 1, a.qual, lane);
                    x ^= c0 ^ c1 ^ c2 ^ c3;
                }
            } else {
                const int nt = feed.tiles_of(L);
                for (int j = 0; j < L; j += WS) {
                    feed.wait(min(nt, (j + 31 * K + 4 * NW + 4 + TILE - 1) / TILE));
                    const uint32_t p = (uint32_t)(j + K * (int)lane) & ~3u;
                    x ^= lds32(feed.at(p)) ^ lds32(feed.at(p + 4u)) ^ lds32(feed.at(p + 8u));
                    const int below = min(nt, ((j + WS) & ~3) / TILE);
                    if (below != feed.freed) feed.release(below, a.qual, lane);
                }
            }
            x = __reduce_xor_sync(FULL, x);       // (bytes beyond the padded extent are whatever the stage held:
            if (lane == 0) a.out[r] = x;          //  the probe's result is not compared with anything)
            feed.end_read(L, a.qual, lane);
        }
    }
}

// Chunked walks with a bulk L2 prefetch. The read is cut into chunks of CH bytes; on entering chunk c lane 0 issues
// cp.async.bulk.prefetch.L2 for chunk c + D (chunks 0 .. D-1 at the read's start), clamped to the read's padded extent
// (offsets are 64-byte aligned, extents whole 64-byte lines, so every prefetch is 16-byte aligned and a multiple of 16).
// The loads themselves stay one step ahead in registers, as in MODE 0. D = 0: no bulk prefetch.
//   KIND 0  k_phred_sum's walk, KIND 1  k_phred_win's walk, each on its own
//   KIND 2  both over the same chunk: the sum's 512-byte steps that start in it, then the window steps that end in it
__device__ __forceinline__ void prefetch_chunk(const uint8_t *q, int pos, int bytes, int padded) {
    if (pos >= padded) return;
    const int end = pos + bytes < padded ? pos + bytes : padded;
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(q + pos), "r"((uint32_t)(end - pos)) : "memory");
}

template <int KIND, int CH, int D>
__global__ void __launch_bounds__(THREADS) k_chunked(Args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const unsigned lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < a.table_bytes / 4; i += blockDim.x) reinterpret_cast<uint32_t *>(smem_raw)[i] = 0u;
    __syncthreads();
    const int skip = KIND == 0 ? H : WS;
    for (;;) {
        unsigned long long it = 0;
        if (lane == 0) it = atomicAdd(a.work, 1ull);
        it = __shfl_sync(FULL, it, 0);
        if (it >= a.n) break;
        const uint32_t r = a.order[it];
        const int L = a.len[r];
        if (L <= skip) continue;
        const uint8_t *q = a.qual + a.off[r];
        const int padded = (L + 63) & ~63;
        const uint4 *qv = reinterpret_cast<const uint4 *>(q);
        const uint32_t *q32 = reinterpret_cast<const uint32_t *>(q);
        const int maxword = (padded >> 2) - 1;
        uint32_t x = 0;
        uint4 spre = make_uint4(0u, 0u, 0u, 0u);
        uint32_t wpre[NW + 1];
        if (KIND != 1 && H + 16 * (int)lane < L) spre = __ldg(qv + ((H >> 4) + (int)lane));
        if (KIND != 0) {
#pragma unroll
            for (int i = 0; i <= NW; ++i) wpre[i] = __ldg(q32 + min(((K * (int)lane) >> 2) + i, maxword));
        }
        if (D > 0 && lane == 0)
            for (int c = 0; c < D; ++c) prefetch_chunk(q, c * CH, CH, padded);
        int js = H, jw = 0;                  // next sum step, next window step
        for (int c0 = 0; c0 < L; c0 += CH) {
            const int cend = c0 + CH < L ? c0 + CH : L;
            if (D > 0 && lane == 0) prefetch_chunk(q, c0 + D * CH, CH, padded);
            if (KIND != 1) {
                for (; js < cend; js += TILE) {
                    x ^= spre.x ^ spre.y ^ spre.z ^ spre.w;
                    const int pn = js + TILE + 16 * (int)lane;
                    if (pn < L) spre = __ldg(qv + (pn >> 4));
                }
            }
            if (KIND != 0) {
                for (; jw < L && min(jw + WS, L) <= cend; jw += WS) {
                    x ^= wpre[0] ^ wpre[1] ^ wpre[2];
                    if (jw + WS < L) {
#pragma unroll
                        for (int i = 0; i <= NW; ++i) wpre[i] = __ldg(q32 + min(((jw + WS + K * (int)lane) >> 2) + i, maxword));
                    }
                }
            }
        }
        x = __reduce_xor_sync(FULL, x);
        if (lane == 0) a.out[r] = x;
    }
}

template <int KIND, int CH, int D>
static int launch_chunked(const Args &a, int sms, int occ, cudaStream_t st) {
    auto k = k_chunked<KIND, CH, D>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, a.table_bytes);
    if (e != cudaSuccess) return (int)e;
    int resident = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, k, THREADS, a.table_bytes);
    if (e != cudaSuccess) return (int)e;
    if (resident < 1) return -2;
    if (occ > resident) occ = resident;
    k<<<sms * occ, THREADS, a.table_bytes, st>>>(a);
    return -(100 + occ);
}

// Runs one chunked probe launch with table_bytes of dynamic shared memory; returns as probe_launch does.
extern "C" int chunked_launch(int kind, int ch, int depth, int table_bytes, int occ, const void *qual, const void *off,
                              const void *len, const void *order, uint32_t n, void *work, void *out, int sms, void *stream) {
    Args a;
    a.qual = (const uint8_t *)qual; a.off = (const unsigned long long *)off; a.len = (const int32_t *)len;
    a.order = (const uint32_t *)order; a.n = n; a.work = (unsigned long long *)work; a.out = (uint32_t *)out;
    a.table_bytes = table_bytes;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(work, 0, 8, st);
    if (e != cudaSuccess) return (int)e;
#define CCASE(KIND_, CH_, D_) \
    if (kind == KIND_ && ch == CH_ && depth == D_) return launch_chunked<KIND_, CH_, D_>(a, sms, occ, st);
#define CDS(KIND_, CH_) CCASE(KIND_, CH_, 0) CCASE(KIND_, CH_, 1) CCASE(KIND_, CH_, 2)
#define CKINDS(KIND_) CDS(KIND_, 2048) CDS(KIND_, 4096) CDS(KIND_, 8192)
    CKINDS(0) CKINDS(1) CKINDS(2)
    return -1;
}

template <int KIND, int MODE, int D, bool DEEP>
static int launch(const Args &a, int sms, int occ, cudaStream_t st) {
    const int smem = a.table_bytes + (MODE ? TILE * D * (THREADS / 32) : 0);
    auto k = k_probe<KIND, MODE, D, DEEP>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    int resident = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, k, THREADS, smem);
    if (e != cudaSuccess) return (int)e;
    if (resident < 1) return -2;
    if (occ > resident) occ = resident;
    k<<<sms * occ, THREADS, smem, st>>>(a);
    return -(100 + occ);                       // what ran: blocks per SM, as -(100 + n)
}

// Runs one probe launch. Returns -(100 + blocks per SM actually launched), -1 for an unknown variant, -2 when the
// variant does not fit an SM, or a positive cudaError_t.
extern "C" int probe_launch(int kind, int mode, int depth, int deep, int occ, const void *qual, const void *off, const void *len,
                            const void *order, uint32_t n, void *work, void *out, int sms, void *stream) {
    Args a;
    a.qual = (const uint8_t *)qual; a.off = (const unsigned long long *)off; a.len = (const int32_t *)len;
    a.order = (const uint32_t *)order; a.n = n; a.work = (unsigned long long *)work; a.out = (uint32_t *)out;
    a.table_bytes = kind == 0 ? 32768 : 49152;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(work, 0, 8, st);
    if (e != cudaSuccess) return (int)e;
#define CASE(KIND_, MODE_, D_, DEEP_) \
    if (kind == KIND_ && mode == MODE_ && depth == D_ && deep == DEEP_) return launch<KIND_, MODE_, D_, DEEP_>(a, sms, occ, st);
#define KINDS(MODE_, D_, DEEP_) CASE(0, MODE_, D_, DEEP_) CASE(1, MODE_, D_, DEEP_)
    KINDS(0, 1, false)
    KINDS(1, 2, false) KINDS(1, 4, false) KINDS(1, 8, false)
    KINDS(1, 2, true) KINDS(1, 4, true) KINDS(1, 8, true)
    KINDS(2, 2, true) KINDS(2, 4, true) KINDS(2, 8, true)
    CASE(0, 3, 2, false) CASE(0, 3, 3, false) CASE(0, 3, 4, false)
    return -1;
}

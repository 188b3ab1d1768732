// filtlong_b200/csrc/fl_contam_k.cu -- the contaminant set for k-mers of 17 to 32 bases (--contam_k, DESIGN.md §4.12).
//
// A 16-mer set is a 2^32-bit direct-address bitmap (fl_kmers.cu). Longer k-mers do not fit in a bitmap, so a long set is a
// device open-addressing hash set of canonical k-mers: min(forward, reverse complement) in 2-bit codes, first base in the
// high bits. Empty is ~0, which is never canonical for K <= 32 (for K = 32 its reverse complement is 0). A bucket is one
// 32-byte sector of four slots, reached through a bijective 64-bit mix of the key, with linear probing from bucket to
// bucket. The table is sized by fl_contam_configure for at most 4/5 of its slots; every add checks that the members so far
// plus the batch's windows stay within that limit, so no insert meets a full table, and the probe loops are capped at the
// table's size as well. Behind the table sit two counters: distinct members and palindromes (canonical k-mers equal to their
// own reverse complement, even K only), so that the set of forward and reverse k-mers has 2 * distinct - palindromes members.
//
//   k_ck_insert  one warp per tile of a contaminant batch: every window of K bases without a non-ACGT base (nmask) adds its
//                canonical k-mer (load the bucket, compare, claim an empty slot by CAS).
//   k_ck_paint   one warp per tile of a read batch: the read's k-mers from its 2-bit codes, looked up eight at a time per
//                lane (two 16-byte loads of one sector each), and hits of the k-mer starts dilated by K - 1 into the 1-bit
//                mask that k_contam_reads counts -- k_probe_paint's layout and seams.
#include <cmath>

#include "fl_device.cuh"

#define CK_EMPTY (~0ull)
#define CK_LOAD_NUM 4          // load limit: members <= 4/5 of the slots
#define CK_LOAD_DEN 5
#define CK_MIN_LOG2_BUCKETS 4

namespace {

// murmur3's 64-bit finaliser: a bijection, so distinct keys never share a hash, only a bucket
__host__ __device__ __forceinline__ unsigned long long ck_mix(unsigned long long x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

__device__ __forceinline__ unsigned long long ck_revcomp(unsigned long long x, int k) {
    const unsigned long long b = __brevll(~x);
    return (((b >> 1) & 0x5555555555555555ull) | ((b & 0x5555555555555555ull) << 1)) >> (64 - 2 * k);
}

// the 64 bases from the lane's first one: A = bases 0..31, B = bases 32..63 (first base in the high bits)
struct LaneBases {
    unsigned long long a, b;
};

// forward k-mer starting at base p (0..31) of the lane's run
__device__ __forceinline__ unsigned long long ck_kmer_at(const LaneBases &w, int p, int k) {
    const unsigned long long x = p == 0 ? w.a : ((w.a << (2 * p)) | (w.b >> (64 - 2 * p)));
    return x >> (64 - 2 * k);
}

__device__ __forceinline__ unsigned long long ck_canonical(unsigned long long fwd, int k) {
    const unsigned long long rc = ck_revcomp(fwd, k);
    return rc < fwd ? rc : fwd;
}

// The lane's 32 bases and the 32 after them (the next lane's, or the next step's first ones for lane 31).
__device__ __forceinline__ LaneBases ck_load_lane(const uint32_t *__restrict__ seqw, unsigned long long step_base,
                                                  unsigned long long padded, unsigned lane) {
    const unsigned long long lb = step_base + 32ull * lane;
    uint2 v = make_uint2(0u, 0u);
    if (lb < padded) v = __ldg(reinterpret_cast<const uint2 *>(seqw + (lb >> 4)));
    uint32_t n0 = __shfl_down_sync(0xffffffffu, v.x, 1), n1 = __shfl_down_sync(0xffffffffu, v.y, 1);
    if (lane == 31) {
        const unsigned long long nb = step_base + FL_STEP_BASES;
        uint2 u = make_uint2(0u, 0u);
        if (nb < padded) u = __ldg(reinterpret_cast<const uint2 *>(seqw + (nb >> 4)));
        n0 = u.x;
        n1 = u.y;
    }
    LaneBases r;
    r.a = ((unsigned long long)v.x << 32) | v.y;
    r.b = ((unsigned long long)n0 << 32) | n1;
    return r;
}

__device__ __forceinline__ unsigned long long ck_warp_sum(unsigned long long v) {
#pragma unroll
    for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

struct CkTable {
    unsigned long long *slots;      // 4 per bucket
    unsigned long long bucket_mask; // n_buckets - 1
    int shift;                      // 64 - log2(n_buckets)
    int k;
};

__device__ __forceinline__ unsigned long long ck_bucket(const CkTable &t, unsigned long long key) { return ck_mix(key) >> t.shift; }

// 1: key is in the bucket, 0: the bucket has an empty slot (so the key is absent), -1: look in the next bucket
__device__ __forceinline__ int ck_verdict(const ulonglong2 &lo, const ulonglong2 &hi, unsigned long long key) {
    if (lo.x == key || lo.y == key || hi.x == key || hi.y == key) return 1;
    if (lo.x == CK_EMPTY || lo.y == CK_EMPTY || hi.x == CK_EMPTY || hi.y == CK_EMPTY) return 0;
    return -1;
}

// 1 when the key was new here (this thread claimed its slot)
__device__ __forceinline__ int ck_insert(const CkTable &t, unsigned long long key) {
    unsigned long long bk = ck_bucket(t, key);
    for (unsigned long long i = 0; i <= t.bucket_mask; ++i) {
        unsigned long long *s = t.slots + 4 * bk;
        const ulonglong2 lo = __ldcg(reinterpret_cast<const ulonglong2 *>(s)), hi = __ldcg(reinterpret_cast<const ulonglong2 *>(s + 2));
        if (lo.x == key || lo.y == key || hi.x == key || hi.y == key) return 0;
        const unsigned long long v[4] = {lo.x, lo.y, hi.x, hi.y};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (v[j] != CK_EMPTY) continue;     // a slot once taken never changes
            const unsigned long long old = atomicCAS(s + j, CK_EMPTY, key);
            if (old == CK_EMPTY) return 1;
            if (old == key) return 0;
        }
        bk = (bk + 1) & t.bucket_mask;
    }
    return 0;   // unreachable: the add checks the load limit first
}

__device__ __forceinline__ bool ck_contains(const CkTable &t, unsigned long long key) {
    unsigned long long bk = ck_bucket(t, key);
    for (unsigned long long i = 0; i <= t.bucket_mask; ++i) {
        const unsigned long long *s = t.slots + 4 * bk;
        const int v = ck_verdict(__ldg(reinterpret_cast<const ulonglong2 *>(s)), __ldg(reinterpret_cast<const ulonglong2 *>(s + 2)), key);
        if (v >= 0) return v == 1;
        bk = (bk + 1) & t.bucket_mask;
    }
    return false;
}

struct CkArgs {
    const uint32_t *seq2b;
    const uint32_t *nmask;                   // k_ck_insert only
    const uint64_t *off;
    const int32_t *len;
    const unsigned long long *tile_start;    // [n + 1]; [n] = number of tiles
    uint32_t n;
    CkTable t;
    unsigned long long *counts;              // k_ck_insert: [0] distinct members, [1] palindromes
    uint32_t *mask;                          // k_ck_paint: 1 bit per padded base
};

__global__ void __launch_bounds__(256) k_ck_insert(CkArgs a) {
    const unsigned lane = threadIdx.x & 31;
    const int k = a.t.k;
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long n_tiles = a.tile_start[a.n];
    const unsigned long long kbits = (1ull << k) - 1ull;
    unsigned long long claimed = 0, palindromes = 0;
    for (unsigned long long tile = warp; tile < n_tiles; tile += n_warps) {
        const uint32_t s = fl_find_seq(a.tile_start, a.n, tile);
        const int L = a.len[s];
        const unsigned long long off = a.off[s];
        const uint32_t *seqw = a.seq2b + (off >> 4);
        const uint32_t *nm = a.nmask + (off >> 5);
        const unsigned long long padded = ((unsigned long long)L + FL_ALIGN_BASES - 1) & ~(unsigned long long)(FL_ALIGN_BASES - 1);
        const unsigned long long tile_base = (tile - a.tile_start[s]) * FL_TILE_BASES;
        for (int step = 0; step < FL_TILE_STEPS; ++step) {
            const unsigned long long sb = tile_base + (unsigned long long)step * FL_STEP_BASES;
            if (sb >= padded) break;
            const LaneBases w = ck_load_lane(seqw, sb, padded, lane);
            const unsigned long long lb = sb + 32ull * lane;
            const uint32_t m0 = lb < padded ? __ldg(nm + (lb >> 5)) : 0u;
            const uint32_t m1 = lb + 32 < padded ? __ldg(nm + (lb >> 5) + 1) : 0u;
            const unsigned long long mm = ((unsigned long long)m1 << 32) | m0;
            for (int p = 0; p < 32; ++p) {
                if (lb + p + (unsigned long long)(k - 1) >= (unsigned long long)L) break;
                if ((mm >> p) & kbits) continue;                 // a non-ACGT base in the window: it adds nothing
                const unsigned long long fwd = ck_kmer_at(w, p, k);
                const unsigned long long rc = ck_revcomp(fwd, k);
                const unsigned long long key = rc < fwd ? rc : fwd;
                if (ck_insert(a.t, key)) {
                    ++claimed;
                    if (rc == fwd) ++palindromes;
                }
            }
        }
    }
    claimed = ck_warp_sum(claimed);
    palindromes = ck_warp_sum(palindromes);
    if (lane == 0 && claimed) atomicAdd(a.counts, claimed);
    if (lane == 0 && palindromes) atomicAdd(a.counts + 1, palindromes);
}

// Bits p of the result: the k-mer starting at lb + p is in the set (p < nvalid). Eight look-ups are issued before any is
// judged, so a lane has sixteen 16-byte loads in flight, and the chains that run past their home bucket go on together.
__device__ __forceinline__ uint32_t ck_hits(const CkTable &t, const LaneBases &w, int nvalid) {
    uint32_t h = 0;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        unsigned long long key[8], bk[8];
        ulonglong2 lo[8], hi[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            key[i] = ck_canonical(ck_kmer_at(w, 8 * g + i, t.k), t.k);
            bk[i] = ck_bucket(t, key[i]);
            if (8 * g + i < nvalid) {
                const unsigned long long *s = t.slots + 4 * bk[i];
                lo[i] = __ldg(reinterpret_cast<const ulonglong2 *>(s));
                hi[i] = __ldg(reinterpret_cast<const ulonglong2 *>(s + 2));
            } else {
                lo[i] = hi[i] = make_ulonglong2(CK_EMPTY, CK_EMPTY);
            }
        }
        int v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = ck_verdict(lo[i], hi[i], key[i]);
        // chains past their home bucket advance together, one bucket per round, with all their loads in flight
        for (unsigned long long round = 0; round < t.bucket_mask; ++round) {
            bool pending = false;
#pragma unroll
            for (int i = 0; i < 8; ++i) pending |= v[i] < 0;
            if (!pending) break;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (v[i] >= 0) continue;
                bk[i] = (bk[i] + 1) & t.bucket_mask;
                const unsigned long long *s = t.slots + 4 * bk[i];
                lo[i] = __ldg(reinterpret_cast<const ulonglong2 *>(s));
                hi[i] = __ldg(reinterpret_cast<const ulonglong2 *>(s + 2));
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
                if (v[i] < 0) v[i] = ck_verdict(lo[i], hi[i], key[i]);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) h |= (v[i] == 1 ? 1u : 0u) << (8 * g + i);
    }
    return h;
}

// base b is covered when a k-mer starting in [b - K + 1, b] is in the set: OR of y << d for d < K, by doubling
__device__ __forceinline__ uint32_t ck_dilate(uint32_t h, uint32_t prev, int k) {
    unsigned long long y = ((unsigned long long)h << 32) | prev;
    int s = 1;
    while (2 * s <= k) {
        y |= y << s;
        s *= 2;
    }
    if (s < k) y |= y << (k - s);
    return (uint32_t)(y >> 32);
}

__global__ void __launch_bounds__(256, 2) k_ck_paint(CkArgs a) {
    const unsigned lane = threadIdx.x & 31;
    const int k = a.t.k;
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned long long n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const unsigned long long n_tiles = a.tile_start[a.n];      // read on the device: no host round trip after the scan
    for (unsigned long long tile = warp; tile < n_tiles; tile += n_warps) {
        const uint32_t s = fl_find_seq(a.tile_start, a.n, tile);
        const int L = a.len[s];
        const unsigned long long off = a.off[s];
        const uint32_t *seqw = a.seq2b + (off >> 4);
        uint32_t *maskw = a.mask + (off >> 5);
        const unsigned long long padded = ((unsigned long long)L + FL_ALIGN_BASES - 1) & ~(unsigned long long)(FL_ALIGN_BASES - 1);
        const unsigned long long tile_base = (tile - a.tile_start[s]) * FL_TILE_BASES;

        // hits of the 32 k-mer starts just before the tile (the last K - 1 of them paint into its first word)
        uint32_t carry = 0;
        if (tile_base > 0) {
            const uint2 u = __ldg(reinterpret_cast<const uint2 *>(seqw + (tile_base >> 4) - 2));   // bases tile_base - 32 ..
            const uint2 v = __ldg(reinterpret_cast<const uint2 *>(seqw + (tile_base >> 4)));       // .. tile_base + 31
            LaneBases w;
            w.a = ((unsigned long long)u.x << 32) | u.y;
            w.b = ((unsigned long long)v.x << 32) | v.y;
            const unsigned long long b = tile_base - 32 + lane;
            bool hit = false;
            if ((int)lane >= 33 - k && b + (unsigned long long)(k - 1) < (unsigned long long)L)
                hit = ck_contains(a.t, ck_canonical(ck_kmer_at(w, (int)lane, k), k));
            carry = __ballot_sync(0xffffffffu, hit);
        }
        for (int step = 0; step < FL_TILE_STEPS; ++step) {
            const unsigned long long sb = tile_base + (unsigned long long)step * FL_STEP_BASES;
            if (sb >= padded) break;
            const LaneBases w = ck_load_lane(seqw, sb, padded, lane);
            const unsigned long long lb = sb + 32ull * lane;
            const long long nv = (long long)L - (k - 1) - (long long)lb;      // starts b with b + K - 1 < L
            const int nvalid = nv <= 0 ? 0 : (nv >= 32 ? 32 : (int)nv);
            const uint32_t h = ck_hits(a.t, w, nvalid);
            uint32_t prev = __shfl_up_sync(0xffffffffu, h, 1);
            if (lane == 0) prev = carry;
            if (lb < padded) maskw[lb >> 5] = ck_dilate(h, prev, k);
            carry = __shfl_sync(0xffffffffu, h, 31);
        }
    }
}

// tiles per sequence (of its padded length) and, into *windows, the batch's sum of max(0, L - K + 1)
__global__ void k_ck_tiles(const int32_t *__restrict__ len, uint32_t n, int k, unsigned long long *__restrict__ tiles,
                           unsigned long long *__restrict__ windows) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long win = 0;
    if (i < n) {
        const int L = len[i];
        tiles[i] = fl_tiles_of(L > 0 ? (int)(((unsigned)L + FL_ALIGN_BASES - 1) & ~(FL_ALIGN_BASES - 1)) : 0);
        win = L >= k ? (unsigned long long)(L - k + 1) : 0ull;
    }
    win = ck_warp_sum(win);
    if ((threadIdx.x & 31) == 0 && win && windows) atomicAdd(windows, win);
}

__global__ void k_ck_contains(CkTable t, const unsigned long long *__restrict__ fwd, uint32_t n, uint8_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = ck_contains(t, ck_canonical(fwd[i], t.k)) ? 1 : 0;
}

CkTable table_of(const KmerSet &s) {
    CkTable t;
    t.slots = s.table;
    t.bucket_mask = s.n_buckets - 1;
    int lg = 0;
    while ((1ull << lg) < s.n_buckets) ++lg;
    t.shift = 64 - lg;
    t.k = s.k;
    return t;
}

// tile_start[0..n] of the batch on the device (no host round trip); windows: where the sum of windows goes (may be null)
int ck_tiles(fl_ctx *ctx, const BatchView &b, int k, unsigned long long *windows) {
    const size_t n = b.n;
    cudaStream_t st = ctx->stream;
    FL_CUDA(ctx, ctx->sc_u64a.reserve(n + 1, 0, st));
    k_ck_tiles<<<fl_blocks(n, 256), 256, 0, st>>>(b.len, b.n, k, ctx->sc_u64a.p, windows);
    ctx->launches++;
    FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_u64a.p, ctx->sc_u64a.p, n, ctx->d_scalars));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->sc_u64a.p + n, ctx->d_scalars, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    return FL_OK;
}

unsigned ck_grid(fl_ctx *ctx, const BatchView &b, unsigned per_sm) {
    const unsigned long long tiles_bound = (b.padded_bases + FL_TILE_BASES - 1) / FL_TILE_BASES + b.n;
    unsigned blocks = (unsigned)((tiles_bound + 7) / 8);
    if (blocks > (unsigned)ctx->sm_count * per_sm) blocks = (unsigned)ctx->sm_count * per_sm;
    return blocks < 1 ? 1 : blocks;
}

}  // namespace

// members the table may hold: CK_LOAD_NUM / CK_LOAD_DEN of its slots
static uint64_t ck_limit(uint64_t n_buckets) { return 4 * n_buckets / CK_LOAD_DEN * CK_LOAD_NUM; }

static size_t ck_bytes(uint64_t n_buckets) { return (size_t)(4 * n_buckets + 2) * sizeof(unsigned long long); }

int fl_ck_add_view(fl_ctx *ctx, KmerSet &s, const BatchView &b) {
    if (!b.seq2b || !b.nmask) { ctx->set_error("fl_contam_add: seq2b and nmask are required"); return FL_EINVAL; }
    cudaStream_t st = ctx->stream;
    unsigned long long *windows = ctx->d_scalars + 29;
    FL_CUDA(ctx, cudaMemsetAsync(windows, 0, sizeof(unsigned long long), st));
    FL_TRY(ck_tiles(ctx, b, s.k, windows));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars + 6, windows, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars + 7, s.table + 4 * s.n_buckets, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(ctx, cudaStreamSynchronize(st));
    const uint64_t batch_windows = ctx->h_scalars[6], distinct = ctx->h_scalars[7];
    if (distinct + batch_windows > s.limit) {
        char buf[320];
        snprintf(buf, sizeof buf,
                 "the contaminant %d-mer set is reserved for %llu k-mers (fl_contam_configure); it holds %llu and this batch "
                 "may add %llu more",
                 s.k, (unsigned long long)s.limit, (unsigned long long)distinct, (unsigned long long)batch_windows);
        ctx->set_error(buf);
        return FL_EINVAL;
    }
    if (batch_windows == 0) return FL_OK;
    CkArgs a{};
    a.seq2b = b.seq2b; a.nmask = b.nmask; a.off = b.off; a.len = b.len; a.tile_start = ctx->sc_u64a.p; a.n = b.n;
    a.t = table_of(s);
    a.counts = s.table + 4 * s.n_buckets;
    {
        KernelTimer kt(ctx, FL_KERNEL_KMERS_ADD);
        k_ck_insert<<<ck_grid(ctx, b, 8), 256, 0, st>>>(a);
    }
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    s.stale = true;
    return FL_OK;
}

int fl_ck_recount(fl_ctx *ctx, KmerSet &s) {
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars, s.table + 4 * s.n_buckets, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s.n = 2 * ctx->h_scalars[0] - ctx->h_scalars[1];     // forward and reverse k-mers: a palindrome is both
    s.stale = false;
    return FL_OK;
}

int fl_ck_paint(fl_ctx *ctx, const KmerSet &s, const BatchView &b, uint32_t *mask, int timer) {
    FL_TRY(ck_tiles(ctx, b, s.k, nullptr));
    CkArgs a{};
    a.seq2b = b.seq2b; a.off = b.off; a.len = b.len; a.tile_start = ctx->sc_u64a.p; a.n = b.n;
    a.t = table_of(s);
    a.mask = mask;
    {
        KernelTimer kt(ctx, timer);
        k_ck_paint<<<ck_grid(ctx, b, 2), 256, 0, ctx->stream>>>(a);
    }
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

int fl_ck_broadcast(fl_ctx *ctx, KmerSet &s, int root) {
    if (ctx->comm_rank == root && s.stale) FL_TRY(fl_ck_recount(ctx, s));
    char *p = reinterpret_cast<char *>(s.table);
    const size_t bytes = ck_bytes(s.n_buckets), piece = (size_t)1 << 30;
    for (size_t at = 0; at < bytes; at += piece)
        FL_TRY(fl_comm_broadcast_bytes(ctx, p + at, bytes - at < piece ? bytes - at : piece, root));
    if (ctx->comm_rank != root) s.stale = true;
    return FL_OK;
}

// ---- C ABI ------------------------------------------------------------------------------------
extern "C" int fl_contam_configure(fl_ctx *ctx, int k, uint64_t max_kmers) {
    FL_ENTER(ctx);
    KmerSet &s = ctx->contam;
    if (k < 16 || k > 32) { ctx->set_error("fl_contam_configure: k must be from 16 to 32"); return FL_EINVAL; }
    if (s.bitmap || s.added) { ctx->set_error("fl_contam_configure: the contaminant set has been added to"); return FL_EINVAL; }
    FL_TRY(fl_contam_check_order(ctx));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s.release();
    s.k = 16;
    s.n = 0;
    s.stale = false;
    s.n_buckets = 0;
    s.limit = 0;
    if (k == 16) return FL_OK;
    // the fewest buckets, a power of two, whose load limit holds max_kmers
    int lg = CK_MIN_LOG2_BUCKETS;
    while (lg < 58 && ck_limit(1ull << lg) < max_kmers) ++lg;
    const double gib = (double)(4.0 * std::ldexp(1.0, lg) + 2.0) * 8.0 / (1024.0 * 1024.0 * 1024.0);
    char what[200];
    snprintf(what, sizeof what, "the contaminant %d-mer set for %llu k-mers needs %.1f GiB of device memory", k,
             (unsigned long long)max_kmers, gib);
    if (lg >= 58) {                                              // more bytes than a size_t can count
        ctx->set_error(std::string(what) + ": out of memory");
        return FL_ENOMEM;
    }
    const uint64_t nb = 1ull << lg;
    cudaError_t e = cudaMalloc(&s.table, ck_bytes(nb));
    if (e == cudaSuccess) e = cudaMemsetAsync(s.table, 0xFF, 4 * nb * sizeof(unsigned long long), ctx->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(s.table + 4 * nb, 0, 2 * sizeof(unsigned long long), ctx->stream);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        if (s.table) cudaFree(s.table);
        s.table = nullptr;
        ctx->set_error(std::string(what) + ": " + cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? FL_ENOMEM : FL_ECUDA;
    }
    s.k = k;
    s.n_buckets = nb;
    s.limit = ck_limit(nb);
    return FL_OK;
}

extern "C" int fl_contam_export64(fl_ctx *ctx, uint64_t *out, uint64_t cap, uint64_t *n_out) {
    FL_ENTER(ctx);
    KmerSet &s = ctx->contam;
    if (s.k == 16) { ctx->set_error("fl_contam_export64: the contaminant set holds 16-mers (fl_contam_export)"); return FL_EINVAL; }
    FL_CUDA(ctx, cudaMemcpyAsync(ctx->h_scalars, s.table + 4 * s.n_buckets, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (n_out) *n_out = ctx->h_scalars[0];
    if (!out || cap == 0) return FL_OK;
    const size_t piece = (size_t)1 << 24, total = 4 * s.n_buckets;
    std::vector<unsigned long long> host(piece < total ? piece : total);
    uint64_t got = 0;
    for (size_t at = 0; at < total && got < cap; at += piece) {
        const size_t m = total - at < piece ? total - at : piece;
        FL_CUDA(ctx, cudaMemcpy(host.data(), s.table + at, m * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < m && got < cap; ++i)
            if (host[i] != CK_EMPTY) out[got++] = host[i];
    }
    return FL_OK;
}

extern "C" int fl_contam_contains64(fl_ctx *ctx, const uint64_t *fwd_kmers, uint32_t n, uint8_t *out) {
    if (!ctx || (!fwd_kmers && n) || (!out && n)) return FL_EINVAL;
    FL_ENTER(ctx);
    KmerSet &s = ctx->contam;
    if (s.k == 16) { ctx->set_error("fl_contam_contains64: the contaminant set holds 16-mers"); return FL_EINVAL; }
    if (n == 0) return FL_OK;
    FL_CUDA(ctx, ctx->sc_u64c.reserve((size_t)n + (n + 7) / 8, 0, ctx->stream));
    unsigned long long *dq = ctx->sc_u64c.p;
    uint8_t *dout = reinterpret_cast<uint8_t *>(dq + n);
    FL_CUDA(ctx, cudaMemcpyAsync(dq, fwd_kmers, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    k_ck_contains<<<fl_blocks(n, 256), 256, 0, ctx->stream>>>(table_of(s), dq, n, dout);
    ctx->launches++;
    FL_CUDA(ctx, cudaMemcpyAsync(out, dout, n, cudaMemcpyDeviceToHost, ctx->stream));
    FL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return FL_OK;
}

// hist[0, n_bins): members by the buckets a look-up of them reads; hist[n_bins, 2 n_bins): buckets by the buckets a
// look-up of an absent k-mer that hashes there reads (up to the first bucket with an empty slot). Last bin: that many or more.
extern "C" int fl_contam_probe_lengths(fl_ctx *ctx, uint64_t *hist, int n_bins) {
    FL_ENTER(ctx);
    KmerSet &s = ctx->contam;
    if (s.k == 16 || !hist || n_bins < 2) { ctx->set_error("fl_contam_probe_lengths: needs a long set and two bins"); return FL_EINVAL; }
    for (int i = 0; i < 2 * n_bins; ++i) hist[i] = 0;
    const uint64_t top = (uint64_t)n_bins - 1;
    auto bin = [&](uint64_t len) { return len < top ? len : top; };
    const size_t piece = (size_t)1 << 24, total = 4 * s.n_buckets;   // a multiple of 4: pieces hold whole buckets
    std::vector<unsigned long long> host(piece < total ? piece : total);
    const unsigned long long mask = s.n_buckets - 1;
    int lg = 0;
    while ((1ull << lg) < s.n_buckets) ++lg;
    uint64_t run = 0, lead = 0;          // full buckets since the last one with an empty slot; those before the first one
    bool seen_empty = false;
    for (size_t at = 0; at < total; at += piece) {
        const size_t m = total - at < piece ? total - at : piece;
        FL_CUDA(ctx, cudaMemcpy(host.data(), s.table + at, m * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < m; i += 4) {
            bool has_empty = false;
            for (int j = 0; j < 4; ++j) {
                const unsigned long long x = host[i + j];
                if (x == CK_EMPTY) { has_empty = true; continue; }
                const unsigned long long home = ck_mix(x) >> (64 - lg), here = (at + i) / 4;
                ++hist[bin(((here - home) & mask) + 1)];
            }
            if (!has_empty) { ++run; continue; }
            if (!seen_empty) lead = run;
            else for (uint64_t r = 1; r <= run; ++r) ++hist[n_bins + bin(r + 1)];
            ++hist[n_bins + 1];
            seen_empty = true;
            run = 0;
        }
    }
    for (uint64_t r = 1; r <= run + lead; ++r) ++hist[n_bins + bin(r + 1)];   // the chains that wrap around the end
    return FL_OK;
}

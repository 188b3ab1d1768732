// filtlong_b200/csrc/fl_qtrim.cu -- --trim_q: --trim / --split on Phred qualities when there is no k-mer set.
//
// "Good" plays the role that "in a reference 16-mer" plays in k-mer mode (read.cpp:79): base i of a read of length L
// is good iff it lies in a run of FL_K = 16 consecutive bases s .. s+15 (s + 15 < L) whose quality bytes are all
// >= 33 + trim_q (unsigned). So the path is k-mer mode's with one kernel swapped and the children scored differently:
//
//   k_qual_mask        the quality arena -> sc_mask, in k_probe_paint's layout (1 bit per padded base, the low bit is
//                      the word's first base, padding bits zero). One warp per read, 1024 bases per step; no per-base
//                      loop: 16-byte loads, __vcmpgeu4 four bytes at a time, a 16-wide AND by doubling (run starts)
//                      and a 16-wide OR by doubling (paint), the neighbouring words' bits from shuffles.
//   k_kmer_scan        unchanged (fl_score.cu): first / last, bad ranges, child ranges, rows -- with the deferred row
//                      count round trip of fl_reads_push.
//   parents            the plain Phred pass (fl_phred_pass), scores only: the rows come from k_kmer_scan.
//   children           k_qrows_plan + a scan place every child row's quality bytes in a 64-aligned scratch arena,
//                      k_qrows_gather copies them (one warp per row), and the SAME Phred pass scores that arena as a
//                      batch of its own: bit-identical to scoring the substring as a read (read.cpp:137 with an
//                      empty k-mer set). A childless read's row is the read itself (main.cpp:139-147): it gets the
//                      read's scores (k_qrows_childless). Children are not trimmed again: a good 16-run never overlaps
//                      a bad range, so a child's own mask is its parent's restricted to it and would give no new rows.
#include "fl_device.cuh"

namespace {

// good-quality bits of the 32 bases in a and b (bit k = base k), only the first `valid` of them
__device__ __forceinline__ uint32_t good_bits(const uint4 &a, const uint4 &b, uint32_t thr4, int valid) {
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t g = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        // one bit per byte at bits 0, 8, 16, 24; the multiply gathers them at bits 21..24 without carries
        const uint32_t t = __vcmpgeu4(w[i], thr4) & 0x01010101u;
        g |= (((t * 0x00204081u) >> 21) & 0xFu) << (4 * i);
    }
    if (valid < 32) g &= valid <= 0 ? 0u : (0xFFFFFFFFu >> (32 - valid));
    return g;
}

__global__ void __launch_bounds__(256) k_qual_mask(const uint8_t *__restrict__ qual, const uint64_t *__restrict__ off,
                                                   const int32_t *__restrict__ len, uint32_t n, uint32_t thr4,
                                                   uint32_t *__restrict__ mask) {
    const unsigned lane = threadIdx.x & 31;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t r = warp; r < n; r += n_warps) {
        const int L = len[r];
        const unsigned long long base = off[r];
        const uint4 *q = reinterpret_cast<const uint4 *>(qual + base);      // 64-aligned
        uint32_t *m = mask + (base >> 5);
        const int n_words = (int)((((unsigned)(L > 0 ? L : 0) + FL_ALIGN_BASES - 1) & ~(FL_ALIGN_BASES - 1)) >> 5);
        auto load = [&](int wi) -> uint32_t {                                 // good bits of word wi (0 beyond the read)
            if (wi >= n_words) return 0u;
            const uint4 a = __ldg(q + 2 * wi), b = __ldg(q + 2 * wi + 1);
            return good_bits(a, b, thr4, L - 32 * wi);
        };
        uint32_t g = load((int)lane);
        uint32_t carry = 0;                                                   // run starts of the previous step's last word
        for (int wb = 0; wb < n_words; wb += 32) {
            const int wi = wb + (int)lane;
            const uint32_t g_step = load(wi + 32);                            // the next step's words
            uint32_t gn = __shfl_down_sync(0xffffffffu, g, 1);
            const uint32_t halo = __shfl_sync(0xffffffffu, g_step, 0);
            if (lane == 31) gn = halo;
            // run starts: bit s set iff bases s .. s+15 are all good (bases at or beyond L never are)
            unsigned long long y = ((unsigned long long)gn << 32) | g;
            y &= y >> 1;
            y &= y >> 2;
            y &= y >> 4;
            y &= y >> 8;
            const uint32_t h = (uint32_t)y;
            // paint: base i is good iff a run starts at one of i-15 .. i
            uint32_t prev = __shfl_up_sync(0xffffffffu, h, 1);
            if (lane == 0) prev = carry;
            unsigned long long z = ((unsigned long long)h << 32) | prev;
            z |= z << 1;
            z |= z << 2;
            z |= z << 4;
            z |= z << 8;
            if (wi < n_words) m[wi] = (uint32_t)(z >> 32);
            carry = __shfl_sync(0xffffffffu, h, 31);
            g = g_step;
        }
    }
}

// per row of the batch: its length in the child arena (0 for the row of a childless read) and its padded length
__global__ void k_qrows_plan(uint32_t n_rows, const uint32_t *__restrict__ w_parent, const int32_t *__restrict__ w_start,
                             const int32_t *__restrict__ w_end, const int32_t *__restrict__ r_nchild,
                             unsigned long long read_base, int32_t *__restrict__ qlen, unsigned long long *__restrict__ qpad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_rows) return;
    const uint32_t p = (uint32_t)(w_parent[i] - read_base);
    const int L = r_nchild[p] > 0 ? w_end[i] - w_start[i] : 0;
    qlen[i] = L;
    qpad[i] = ((unsigned long long)L + FL_ALIGN_BASES - 1) & ~(unsigned long long)(FL_ALIGN_BASES - 1);
}

// one warp per child row: its quality bytes [start, end) of the parent, '!' up to the padded end
__global__ void __launch_bounds__(256) k_qrows_gather(uint32_t n_rows, const uint8_t *__restrict__ qual,
                                                      const uint64_t *__restrict__ off, const uint32_t *__restrict__ w_parent,
                                                      const int32_t *__restrict__ w_start, unsigned long long read_base,
                                                      const int32_t *__restrict__ qlen, const unsigned long long *__restrict__ qoff,
                                                      uint8_t *__restrict__ out) {
    const unsigned lane = threadIdx.x & 31;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    const uint32_t *q32 = reinterpret_cast<const uint32_t *>(qual);
    for (size_t i = warp; i < n_rows; i += n_warps) {
        const int L = qlen[i];
        if (L == 0) continue;
        const unsigned long long src = off[w_parent[i] - read_base] + (unsigned long long)w_start[i];   // first byte
        const unsigned long long end = src + (unsigned long long)L;
        uint4 *dst = reinterpret_cast<uint4 *>(out + qoff[i]);
        const int n_q = (int)((((unsigned)L + FL_ALIGN_BASES - 1) & ~(FL_ALIGN_BASES - 1)) >> 4);
        const unsigned sh = (unsigned)(src & 3u) * 8u;
        for (int j = (int)lane; j < n_q; j += 32) {                           // 16 bytes per lane and step
            uint32_t v[4] = {0x21212121u, 0x21212121u, 0x21212121u, 0x21212121u};
            const int nb = L - 16 * j;                                        // bytes of these 16 inside the child
            if (nb > 0) {
                const unsigned long long wa = (src + 16ull * (unsigned long long)j) >> 2;
                uint32_t w[5];
#pragma unroll
                for (int k = 0; k < 5; ++k) w[k] = (wa + k) * 4 < end ? __ldg(q32 + wa + k) : 0u;   // never past the read
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int nk = nb - 4 * k;
                    if (nk <= 0) break;
                    v[k] = __funnelshift_r(w[k], w[k + 1], sh);
                    if (nk < 4) {
                        const uint32_t keep = 0xFFFFFFFFu >> (32 - 8 * nk);
                        v[k] = (v[k] & keep) | (0x21212121u & ~keep);
                    }
                }
            }
            dst[j] = make_uint4(v[0], v[1], v[2], v[3]);
        }
    }
}

// the row of a childless read is the read itself: the read's scores
__global__ void k_qrows_childless(uint32_t n_rows, const uint32_t *__restrict__ w_parent, const int32_t *__restrict__ r_nchild,
                                  unsigned long long read_base, const double *__restrict__ r_mean,
                                  const double *__restrict__ r_window, const uint8_t *__restrict__ r_passed,
                                  double *__restrict__ w_mean, double *__restrict__ w_window, uint8_t *__restrict__ w_passed) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_rows) return;
    const uint32_t p = (uint32_t)(w_parent[i] - read_base);
    if (r_nchild[p] > 0) return;
    w_mean[i] = r_mean[p];
    w_window[i] = r_window[p];
    w_passed[i] = r_passed[p];
}

}  // namespace

int fl_qual_mask(fl_ctx *ctx, const BatchView &b) {
    cudaStream_t st = ctx->stream;
    FL_CUDA(ctx, ctx->sc_mask.reserve((size_t)(b.padded_bases >> 5) + 1, 0, st));
    const uint32_t thr = 33u + (uint32_t)ctx->p.trim_q;                       // 34 .. 126
    unsigned blocks = fl_blocks((size_t)b.n * 32, 256);
    if (blocks > (unsigned)ctx->sm_count * 8) blocks = (unsigned)ctx->sm_count * 8;
    {
        KernelTimer kt(ctx, FL_KERNEL_QUAL_MASK);
        k_qual_mask<<<blocks, 256, 0, st>>>(b.qual, b.off, b.len, b.n, thr * 0x01010101u, ctx->sc_mask.p);
    }
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

int fl_score_qual_rows(fl_ctx *ctx, const BatchView &b, size_t n_rows_batch) {
    if (n_rows_batch == 0) return FL_OK;
    cudaStream_t st = ctx->stream;
    const size_t rb = ctx->n_reads, wb = ctx->n_rows, m = n_rows_batch;
    const uint32_t *w_parent = ctx->w_parent.p + wb;
    const int32_t *r_nchild = ctx->r_nchild.p + rb;
    FL_CUDA(ctx, ctx->sc_qoff.reserve(m + 1, 0, st));
    FL_CUDA(ctx, ctx->sc_qlen.reserve(m + 1, 0, st));
    k_qrows_plan<<<fl_blocks(m, 256), 256, 0, st>>>((uint32_t)m, w_parent, ctx->w_start.p + wb, ctx->w_end.p + wb, r_nchild, rb,
                                                     ctx->sc_qlen.p, ctx->sc_qoff.p);
    ctx->launches++;
    FL_TRY(fl_exclusive_scan_u64(ctx, ctx->sc_qoff.p, ctx->sc_qoff.p, m, nullptr));
    // children never overlap and lie inside their parents: their bytes fit in the batch's, plus < 64 of padding each
    const uint64_t bound = b.padded_bases + (uint64_t)FL_ALIGN_BASES * m;
    FL_CUDA(ctx, ctx->sc_qual.reserve((size_t)bound + 64, 0, st));
    {
        KernelTimer kt(ctx, FL_KERNEL_QUAL_GATHER);
        unsigned blocks = fl_blocks(m * 32, 256);
        if (blocks > (unsigned)ctx->sm_count * 8) blocks = (unsigned)ctx->sm_count * 8;
        k_qrows_gather<<<blocks, 256, 0, st>>>((uint32_t)m, b.qual, b.off, w_parent, ctx->w_start.p + wb, rb, ctx->sc_qlen.p,
                                               ctx->sc_qoff.p, ctx->sc_qual.p);
    }
    ctx->launches++;
    BatchView cv{};
    cv.n = (uint32_t)m;
    cv.padded_bases = bound;
    cv.off = reinterpret_cast<const uint64_t *>(ctx->sc_qoff.p);
    cv.len = ctx->sc_qlen.p;
    cv.qual = ctx->sc_qual.p;
    {
        KernelTimer kt(ctx, FL_KERNEL_QUAL_CHILDREN);
        FL_TRY(fl_phred_pass(ctx, cv, PhredOut{ctx->w_mean.p + wb, ctx->w_window.p + wb, ctx->w_passed.p + wb, false}));
    }
    k_qrows_childless<<<fl_blocks(m, 256), 256, 0, st>>>((uint32_t)m, w_parent, r_nchild, rb, ctx->r_mean.p + rb,
                                                          ctx->r_window.p + rb, ctx->r_passed.p + rb, ctx->w_mean.p + wb,
                                                          ctx->w_window.p + wb, ctx->w_passed.p + wb);
    ctx->launches++;
    FL_CUDA(ctx, cudaGetLastError());
    return FL_OK;
}

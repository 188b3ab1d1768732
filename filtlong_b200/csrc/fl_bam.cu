// filtlong_b200/csrc/fl_bam.cu -- unaligned BAM records to the scoring arena.
//
// The host (host/bam.cpp) inflates the BAM file, walks its records, checks them and hands over a chunk of whole records
// with where each record's SEQ and QUAL start. Here the chunk is staged like a text chunk (fl_text.cu) and one warp per
// record gathers what the scoring mode reads into the arena:
//   * Phred mode: the QUAL bytes + 33, i.e. the quality line of the record's FASTQ equivalent;
//   * k-mer mode: the 4-bit SEQ codes (=ACMGRSVTWYHKDBN) as the arena's 2-bit codes. A, C, G, T are 1, 2, 4, 8 and become
//     0..3; every other code becomes 0, which is what the reference's base_to_bits_forward gives a base outside ACGT.
// Then the batch is scored like every other one (fl_score_view).
#include "fl_device.cuh"

namespace {

// W little-endian words of the chunk starting at byte offset o (any alignment); no word past last_word is read
template <int W>
__device__ __forceinline__ void bam_load(const uint32_t *__restrict__ t32, unsigned long long o, unsigned long long last_word, uint32_t (&out)[W]) {
    const unsigned long long w0 = o >> 2;
    const unsigned sh = ((unsigned)o & 3u) * 8u;
    uint32_t prev = __ldg(t32 + (w0 <= last_word ? w0 : last_word));
#pragma unroll
    for (int i = 0; i < W; ++i) {
        const unsigned long long wi = w0 + 1 + i;
        const uint32_t nxt = __ldg(t32 + (wi <= last_word ? wi : last_word));
        out[i] = __funnelshift_r(prev, nxt, sh);
        prev = nxt;
    }
}

// 2-bit arena code of a 4-bit SEQ code, two bits per code: C (2) -> 1, G (4) -> 2, T (8) -> 3, everything else -> 0
#define BAM_NIBBLE_CODES 0x30210u

// One warp per record, 32 bases per lane and step (like k_text_gather). Bases at or beyond the record's length are
// written as 0 in both arenas, as the host packer leaves them.
template <bool PHRED>
__global__ void __launch_bounds__(256) k_bam_gather(const uint8_t *__restrict__ chunk, unsigned long long n_bytes, uint32_t n_rec,
                                                    const uint32_t *__restrict__ seq_off, const uint32_t *__restrict__ qual_off,
                                                    const int32_t *__restrict__ len, const unsigned long long *__restrict__ off,
                                                    uint32_t *__restrict__ seq2b, uint8_t *__restrict__ qual) {
    const unsigned lane = threadIdx.x & 31;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    const uint32_t *t32 = reinterpret_cast<const uint32_t *>(chunk);
    const unsigned long long last_word = n_bytes ? (n_bytes - 1) >> 2 : 0;
    for (size_t r = warp; r < n_rec; r += n_warps) {
        const int L = len[r];
        const unsigned long long dof = off[r];
        const int padded = (int)(((unsigned)L + 63u) & ~63u);
        const unsigned long long src = PHRED ? qual_off[r] : seq_off[r];
        for (int b = 32 * (int)lane; b < padded; b += 1024) {
            const int nv = L - b;                                         // valid bases of these 32
            if (PHRED) {
                uint32_t c[8];
                bam_load<8>(t32, src + (unsigned long long)b, last_word, c);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int keep = nv - 4 * i;
                    const uint32_t m = keep >= 4 ? 0xFFFFFFFFu : (keep <= 0 ? 0u : (1u << (8 * keep)) - 1u);
                    c[i] = __vadd4(c[i], 0x21212121u) & m;                // QUAL + 33 (bytes wrap: no carry between them)
                }
                uint4 *dst = reinterpret_cast<uint4 *>(qual + dof + b);
                dst[0] = make_uint4(c[0], c[1], c[2], c[3]);
                dst[1] = make_uint4(c[4], c[5], c[6], c[7]);
            } else {
                uint32_t c[4];                                            // 16 bytes = 32 codes, base 2j in the high nibble of byte j
                bam_load<4>(t32, src + (unsigned long long)(b >> 1), last_word, c);
                uint32_t w[2] = {0u, 0u};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint32_t byte = (c[i] >> (8 * k)) & 0xFFu;
                        const int q = 8 * i + 2 * k;                      // base of the high nibble, 0..30
                        const uint32_t hi = (BAM_NIBBLE_CODES >> (2 * (byte >> 4))) & 3u, lo = (BAM_NIBBLE_CODES >> (2 * (byte & 15u))) & 3u;
                        w[q >> 4] |= ((hi << 2) | lo) << (28 - 2 * (q & 15));
                    }
                }
                if (nv < 32) {
                    if (nv <= 0) { w[0] = 0; w[1] = 0; }
                    else if (nv < 16) { w[0] &= ~(0xFFFFFFFFu >> (2 * nv)); w[1] = 0; }
                    else if (nv > 16) w[1] &= ~(0xFFFFFFFFu >> (2 * (nv - 16)));
                    else w[1] = 0;
                }
                reinterpret_cast<uint2 *>(seq2b + ((dof + b) >> 4))[0] = make_uint2(w[0], w[1]);
            }
        }
    }
}

}  // namespace

extern "C" int fl_reads_push_bam(fl_ctx *c, const char *chunk, uint64_t n_bytes, uint64_t n_rec, const uint32_t *seq_off,
                                 const uint32_t *qual_off, const int32_t *len) {
    FL_ENTER(c);
    if ((!chunk && n_bytes) || (n_rec && (!chunk || !seq_off || !qual_off || !len))) {
        c->set_error("fl_reads_push_bam: bad arguments");
        return FL_EINVAL;
    }
    if (n_bytes >= ((uint64_t)1 << 31)) { c->set_error("fl_reads_push_bam: a chunk must be smaller than 2 GiB"); return FL_ERANGE; }
    if (n_rec > 0xFFFFFFF0ull) { c->set_error("fl_reads_push_bam: too many records in one chunk"); return FL_ERANGE; }
    if (n_rec == 0) return FL_OK;
    FL_TRY(fl_sets_ready(c));
    const bool kmer_mode = c->ref.n > 0;
    const size_t n = (size_t)n_rec;
    // the arena's layout (padded offsets) and the input's bases (main.cpp:89); every record must lie inside the chunk
    std::vector<uint64_t> off(n);
    uint64_t padded_bases = 0;
    int64_t bases = 0;
    for (size_t i = 0; i < n; ++i) {
        const uint64_t L = (uint64_t)(len[i] < 0 ? 0 : len[i]);
        if (len[i] < 1 || (uint64_t)seq_off[i] + (L + 1) / 2 > n_bytes || (uint64_t)qual_off[i] + L > n_bytes) {
            c->set_error("fl_reads_push_bam: record " + std::to_string(i) + " does not lie inside the chunk");
            return FL_EINVAL;
        }
        off[i] = padded_bases;
        padded_bases += (L + FL_ALIGN_BASES - 1) & ~(uint64_t)(FL_ALIGN_BASES - 1);
        bases += (int64_t)L;
    }
    // stage: chunk + SEQ / QUAL offsets in one byte buffer, lengths and offsets in the slot's own arrays (copy stream,
    // double buffered like fl_reads_push)
    const int slot = c->stg_next;
    c->stg_next ^= 1;
    fl_ctx::Staging &S = c->stg[slot];
    if (!S.consumed) FL_CUDA(c, cudaEventCreateWithFlags(&S.consumed, cudaEventDisableTiming));
    if (S.in_use) FL_CUDA(c, cudaEventSynchronize(S.consumed));
    S.in_use = false;
    cudaStream_t st = c->stream, cs = c->copy_stream;
    const size_t chunk_room = ((size_t)n_bytes + 64 + 15) & ~(size_t)15;
    FL_CUDA(c, S.ascii.reserve(chunk_room + 8 * n, 0, cs));
    FL_CUDA(c, S.off.reserve(n + 1, 0, cs));
    FL_CUDA(c, S.len.reserve(n, 0, cs));
    uint32_t *d_seq_off = reinterpret_cast<uint32_t *>(S.ascii.p + chunk_room), *d_qual_off = d_seq_off + n;
    FL_CUDA(c, cudaMemcpyAsync(S.ascii.p, chunk, (size_t)n_bytes, cudaMemcpyHostToDevice, cs));
    FL_CUDA(c, cudaMemcpyAsync(d_seq_off, seq_off, n * sizeof(uint32_t), cudaMemcpyHostToDevice, cs));
    FL_CUDA(c, cudaMemcpyAsync(d_qual_off, qual_off, n * sizeof(uint32_t), cudaMemcpyHostToDevice, cs));
    FL_CUDA(c, cudaMemcpyAsync(S.len.p, len, n * sizeof(int32_t), cudaMemcpyHostToDevice, cs));
    FL_CUDA(c, cudaMemcpyAsync(S.off.p, off.data(), n * sizeof(uint64_t), cudaMemcpyHostToDevice, cs));
    FL_CUDA(c, cudaEventRecord(c->ev_copied, cs));
    FL_CUDA(c, cudaStreamWaitEvent(st, c->ev_copied, 0));
    // ---- gather into the arena, score ----
    const unsigned long long *d_off = reinterpret_cast<const unsigned long long *>(S.off.p);
    BatchView v{};
    v.n = (uint32_t)n; v.padded_bases = padded_bases; v.off = S.off.p; v.len = S.len.p;
    unsigned ggrid = fl_blocks(n * 32, 256);
    if (ggrid > (unsigned)c->sm_count * 16) ggrid = (unsigned)c->sm_count * 16;
    if (fl_wants_bases(c)) {                                             // k-mer mode, or a contaminant set to probe
        FL_CUDA(c, S.seq.reserve((size_t)(padded_bases >> 4) + 8, 0, st));
        k_bam_gather<false><<<ggrid, 256, 0, st>>>(S.ascii.p, n_bytes, (uint32_t)n, d_seq_off, d_qual_off, S.len.p, d_off, S.seq.p, nullptr);
        v.seq2b = S.seq.p;
        c->launches++;
    }
    if (!kmer_mode) {
        FL_CUDA(c, S.qual.reserve((size_t)padded_bases + 64, 0, st));
        k_bam_gather<true><<<ggrid, 256, 0, st>>>(S.ascii.p, n_bytes, (uint32_t)n, d_seq_off, d_qual_off, S.len.p, d_off, nullptr, S.qual.p);
        v.qual = S.qual.p;
        c->launches++;
    }
    FL_CUDA(c, cudaGetLastError());
    FL_TRY(fl_score_view(c, v));
    c->total_bases += bases;                                             // main.cpp:89
    FL_CUDA(c, cudaEventRecord(S.consumed, st));
    S.in_use = true;
    FL_CUDA(c, cudaStreamSynchronize(cs));                               // the caller may reuse its buffers now
    return FL_OK;
}

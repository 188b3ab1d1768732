// filtlong_b200/csrc/fl_text.cu -- the feeder: FASTQ / FASTA TEXT parsed on the device.
//
// The reference reads its input one record at a time through klib's kseq (reference src/kseq.h:161-224,
// loop at src/main.cpp:70-125) and hands each record's char buffers to `new Read(...)`. Here the caller
// hands over a chunk of the file as it is -- bytes -- and the device does the rest: newline index, record
// boundaries, validation, per-record name / comment / sequence / quality extents, a 64-bit hash of every
// name (for the duplicate check of main.cpp:113-117), the CSR of padded offsets, and the gather of the
// sequence (2-bit packed, kmers.cpp:176-196) or the quality bytes into the arena the scoring kernels read.
//
// Only the COMMON layout is parsed here: 4-line FASTQ records (@name[ comment] / sequence / +[anything] /
// quality of the same length) or 2-line FASTA records, LF line ends, non-empty names and sequences. Anything
// else (CR LF, multi-line records, blank lines, a truncated quality string ...) is reported as
// FL_TEXT_FALLBACK without scoring anything: the caller then runs its kseq-compatible host parser, which
// reproduces the reference's behaviour (and error messages) on such input.
#include "fl_device.cuh"
#include "fl_name_hash.h"

namespace {

#define TX_LINES_PER_WARP 512          // bytes per warp in the newline passes (16 per lane)

__device__ __forceinline__ uint32_t nl_mask16(const uint4 v, int nvalid) {
    // bit i set where byte i of the 16 is '\n'
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t eq = __vcmpeq4(w[i], 0x0A0A0A0Au) & 0x01010101u;
        m |= ((eq | (eq >> 7) | (eq >> 14) | (eq >> 21)) & 0xFu) << (4 * i);
    }
    if (nvalid < 16) m &= (1u << (nvalid < 0 ? 0 : nvalid)) - 1u;
    return m;
}

// does any of the first nvalid bytes of the 16 hold a NUL?
__device__ __forceinline__ bool has_nul16(const uint4 v, int nvalid) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t m = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t eq = __vcmpeq4(w[i], 0u) & 0x01010101u;
        m |= ((eq | (eq >> 7) | (eq >> 14) | (eq >> 21)) & 0xFu) << (4 * i);
    }
    if (nvalid < 16) m &= (1u << (nvalid < 0 ? 0 : nvalid)) - 1u;
    return m != 0;
}

// pass A: newlines per 512-byte block; *nul set when the text holds a NUL byte. The reference handles every field as a
// C string (main.cpp:90,268-305: a name, comment, sequence or quality ends at its first NUL for the dictionary and the
// output), which slices of the text cannot reproduce: such a chunk is the host reader's.
__global__ void __launch_bounds__(256) k_text_count(const uint8_t *__restrict__ text, unsigned long long n_bytes, unsigned long long n_blocks,
                                                    unsigned long long *__restrict__ counts, int *__restrict__ nul) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5,
                             n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    bool z = false;
    for (unsigned long long b = warp; b < n_blocks; b += n_warps) {
        const unsigned long long pos = b * TX_LINES_PER_WARP + 16ull * lane;
        uint32_t m = 0;
        if (pos < n_bytes) {
            const uint4 v = __ldg(reinterpret_cast<const uint4 *>(text + pos));
            const int nvalid = (int)(n_bytes - pos < 16 ? n_bytes - pos : 16);
            m = nl_mask16(v, nvalid);
            z |= has_nul16(v, nvalid);
        }
        const int c = __reduce_add_sync(0xffffffffu, __popc(m));
        if (lane == 0) counts[b] = (unsigned long long)c;
    }
    if (z) atomicOr(nul, 1);
}

// pass B: positions of the newlines, in order (counts[] now holds the exclusive scan)
__global__ void __launch_bounds__(256) k_text_positions(const uint8_t *__restrict__ text, unsigned long long n_bytes, unsigned long long n_blocks,
                                                        const unsigned long long *__restrict__ start, uint32_t *__restrict__ nl) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5,
                             n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    for (unsigned long long b = warp; b < n_blocks; b += n_warps) {
        const unsigned long long pos = b * TX_LINES_PER_WARP + 16ull * lane;
        uint32_t m = 0;
        if (pos < n_bytes) m = nl_mask16(__ldg(reinterpret_cast<const uint4 *>(text + pos)), (int)(n_bytes - pos < 16 ? n_bytes - pos : 16));
        int c = __popc(m), incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= (unsigned)d) incl += t;
        }
        unsigned long long o = start[b] + (unsigned long long)(incl - c);
        while (m) {
            const int i = __ffs(m) - 1;
            m &= m - 1;
            nl[o++] = (uint32_t)(pos + i);
        }
    }
}

struct RecArgs {
    const uint8_t *text;
    unsigned long long n_bytes;
    const uint32_t *nl;               // newline positions; a virtual one at n_bytes when the chunk is the file's end without one
    unsigned long long n_lines;
    uint32_t n_rec;
    int lines_per_rec;                // 4 FASTQ, 2 FASTA
    uint32_t *name_off, *name_len, *comment_len, *seq_off, *qual_off;
    int32_t *len;
    unsigned long long *name_hash, *padded;
    int *bad;                         // set when the layout is not the simple one
};

__device__ __forceinline__ bool tx_space(unsigned c) { return c == ' ' || (c >= 9 && c <= 13); }   // isspace in the C locale (kseq.h:193)

__global__ void __launch_bounds__(256) k_text_records(RecArgs a) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= a.n_rec) return;
    const unsigned long long l0 = (unsigned long long)k * a.lines_per_rec;
    auto line_end = [&](unsigned long long i) -> unsigned long long { return i < a.n_lines ? a.nl[i] : a.n_bytes; };
    const unsigned long long s0 = l0 ? line_end(l0 - 1) + 1 : 0ull;     // header line
    const unsigned long long e0 = line_end(l0);
    const unsigned long long s1 = e0 + 1, e1 = line_end(l0 + 1);        // sequence line
    bool bad = false;
    const unsigned lead = a.lines_per_rec == 4 ? '@' : '>';
    if (e0 <= s0 || a.text[s0] != lead) bad = true;
    // name: up to the first whitespace; comment: the rest of the line after that one character (kseq.h:193-194)
    unsigned long long p = s0 + 1;
    unsigned long long h = FL_NAME_HASH_INIT;                            // fl_name_hash.h, shared with the BAM walker
    while (p < e0 && !tx_space(a.text[p])) {
        h = fl_name_hash_step(h, a.text[p]);
        ++p;
    }
    h = fl_name_hash_final(h);
    const unsigned long long nlen = p - (s0 + 1);
    if (nlen == 0) bad = true;
    const unsigned long long clen = p < e0 ? e0 - (p + 1) : 0ull;
    if (e1 <= s1) bad = true;                                            // empty sequence line
    else if (a.text[s1] == '@' || a.text[s1] == '>' || a.text[s1] == '+') bad = true;   // kseq.h:199: ends the sequence there
    const unsigned long long L = e1 > s1 ? e1 - s1 : 0ull;
    if (L > 0x7FFFFFFFull) bad = true;                                   // main.cpp:69,77: int length
    unsigned long long s3 = 0;
    if (a.lines_per_rec == 4) {
        const unsigned long long s2 = e1 + 1, e2 = line_end(l0 + 2);
        s3 = e2 + 1;
        const unsigned long long e3 = line_end(l0 + 3);
        if (e2 <= s2 || a.text[s2] != '+') bad = true;
        if (e3 < s3 || e3 - s3 != L) bad = true;                         // kseq would read on / report -2: the host parser's job
        if (L && a.text[e3 - 1] == '\r') bad = true;
    }
    if (e0 > s0 && a.text[e0 - 1] == '\r') bad = true;                    // CR LF files: kseq strips the CR, slices would not
    if (L && a.text[e1 - 1] == '\r') bad = true;
    if (bad) { atomicOr(a.bad, 1); return; }
    a.name_off[k] = (uint32_t)(s0 + 1);
    a.name_len[k] = (uint32_t)nlen;
    a.comment_len[k] = (uint32_t)clen;
    a.seq_off[k] = (uint32_t)s1;
    a.qual_off[k] = (uint32_t)s3;
    a.len[k] = (int32_t)L;
    a.name_hash[k] = h;
    a.padded[k] = (L + FL_ALIGN_BASES - 1) & ~(unsigned long long)(FL_ALIGN_BASES - 1);
}

// 32 bytes of text starting at byte offset o (any alignment), as 8 little-endian words
__device__ __forceinline__ void tx_load32(const uint32_t *__restrict__ t32, unsigned long long o, unsigned long long last_word, uint32_t (&out)[8]) {
    const unsigned long long w0 = o >> 2;
    const unsigned sh = ((unsigned)o & 3u) * 8u;
    uint32_t prev = __ldg(t32 + (w0 <= last_word ? w0 : last_word));
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const unsigned long long wi = w0 + 1 + i;
        const uint32_t nxt = __ldg(t32 + (wi <= last_word ? wi : last_word));
        out[i] = __funnelshift_r(prev, nxt, sh);
        prev = nxt;
    }
}

// gather: one warp per record copies the record's sequence (packed to 2 bits) or quality bytes into the arena
template <bool PHRED>
__global__ void __launch_bounds__(256) k_text_gather(const uint8_t *__restrict__ text, unsigned long long n_bytes, uint32_t n_rec,
                                                     const uint32_t *__restrict__ src_off, const int32_t *__restrict__ len,
                                                     const unsigned long long *__restrict__ off, uint32_t *__restrict__ seq2b,
                                                     uint8_t *__restrict__ qual, uint32_t *__restrict__ nmask) {
    const unsigned lane = threadIdx.x & 31;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    const uint32_t *t32 = reinterpret_cast<const uint32_t *>(text);
    const unsigned long long last_word = n_bytes ? (n_bytes - 1) >> 2 : 0;
    for (size_t r = warp; r < n_rec; r += n_warps) {
        const int L = len[r];
        const unsigned long long so = src_off[r], dof = off[r];
        const int padded = (int)(((unsigned)L + 63u) & ~63u);
        for (int b = 32 * (int)lane; b < padded; b += 1024) {           // 32 bases per lane per iteration
            uint32_t c[8];
            tx_load32(t32, so + (unsigned long long)b, last_word, c);
            if (PHRED) {
                uint4 *dst = reinterpret_cast<uint4 *>(qual + dof + b);
                dst[0] = make_uint4(c[0], c[1], c[2], c[3]);
                dst[1] = make_uint4(c[4], c[5], c[6], c[7]);
            } else {
                uint32_t w[2] = {0u, 0u}, m = 0u;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    uint32_t code8, other4;
                    fl_pack4(c[i], code8, other4);
                    w[i >> 2] |= code8 << (24 - 8 * (i & 3));
                    m |= other4 << (4 * i);                              // non-ACGT characters (reference sequences: kmers.cpp:199-219)
                }
                // bases at or beyond L must be code 0 for nobody in particular (no kernel forms a 16-mer there), but a
                // clean tail keeps batches comparable with the host packer's
                const int nv = L - b;
                if (nv < 32) {
                    if (nv <= 0) { w[0] = 0; w[1] = 0; }
                    else if (nv < 16) { w[0] &= ~(0xFFFFFFFFu >> (2 * nv)); w[1] = 0; }
                    else if (nv < 32) { if (nv > 16) w[1] &= ~(0xFFFFFFFFu >> (2 * (nv - 16))); else w[1] = 0; }
                }
                reinterpret_cast<uint2 *>(seq2b + ((dof + b) >> 4))[0] = make_uint2(w[0], w[1]);
                if (nmask) nmask[(dof + b) >> 5] = nv >= 32 ? m : (nv <= 0 ? 0u : m & ((1u << nv) - 1u));
            }
        }
    }
}

__global__ void k_text_u32_to_u64(const uint32_t *__restrict__ in, uint32_t n, unsigned long long base, unsigned long long *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = base + in[i];
}

__global__ void k_text_sum_len(const int32_t *len, uint32_t n, unsigned long long *out, int min_len = 0) {
    unsigned long long s = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        if (len[i] >= min_len) s += (unsigned long long)len[i];
#pragma unroll
    for (int d = 16; d; d >>= 1) s += __shfl_down_sync(0xffffffffu, s, d);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// ---------------------------------------------------------------------------------------------
// FASTA reference files whose sequences are WRAPPED (kmers.cpp:75-134 reads them through kseq, which joins the lines of
// a record: kseq.h:199-203). A record is a '>' line and every line up to the next '>' line; when all of its sequence
// lines but the last have one width w (and the last is not longer) -- how every assembler and `fold` write them -- base p
// of the record is byte  first + p + p / w  of the text: no line of it has to be looked at again. Anything else (blank
// lines, CR LF, ragged lines, a line starting with '@' or '+', which kseq takes for the next record / the quality
// separator) is left to the host reader.
// ---------------------------------------------------------------------------------------------
struct FaArgs {
    const uint8_t *text;
    unsigned long long n_bytes;
    const uint32_t *nl;               // newline positions
    unsigned long long n_lines;       // real newlines
    unsigned long long NL;            // lines, counting a last one without newline
    unsigned long long *head;         // [NL] 1 on header lines; after the exclusive scan: headers before the line
    uint32_t *head_line;              // [n_rec] line index of every header
    uint32_t n_rec;
    uint32_t *seq_off, *width;        // per record: first sequence byte, line width
    int32_t *len;
    unsigned long long *padded;
    int *bad;
};

__device__ __forceinline__ unsigned long long fa_start(const FaArgs &a, unsigned long long i) { return i ? (unsigned long long)a.nl[i - 1] + 1 : 0ull; }
__device__ __forceinline__ unsigned long long fa_end(const FaArgs &a, unsigned long long i) { return i < a.n_lines ? (unsigned long long)a.nl[i] : a.n_bytes; }

// per line: header or not, and the per-line part of the validation
__global__ void __launch_bounds__(256) k_fa_heads(FaArgs a) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.NL) return;
    const unsigned long long s = fa_start(a, i), e = fa_end(a, i);
    const bool h = e > s && a.text[s] == '>';
    a.head[i] = h ? 1ull : 0ull;
    bool bad = false;
    if (i == 0 && !h) bad = true;                                   // the chunk must start a record
    if (e == s) bad = true;                                         // blank line (kseq skips it; the arithmetic cannot)
    else {
        if (a.text[e - 1] == '\r') bad = true;                      // CR LF
        if (!h && (a.text[s] == '@' || a.text[s] == '+')) bad = true;   // kseq.h:199: ends the sequence
        if (h && e - s == 1 && i >= a.n_lines) bad = true;          // a '>' that ends the file starts no record (kseq.h:193, -1)
    }
    if (bad) atomicOr(a.bad, 1);
}

// after the scan: where every header sits
__global__ void __launch_bounds__(256) k_fa_scatter(FaArgs a) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.NL) return;
    const unsigned long long s = fa_start(a, i), e = fa_end(a, i);
    if (e > s && a.text[s] == '>') a.head_line[a.head[i]] = (uint32_t)i;
}

// per record: extent, width, length
__global__ void __launch_bounds__(256) k_fa_records(FaArgs a) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.n_rec) return;
    const unsigned long long h = a.head_line[r], nxt = r + 1 < a.n_rec ? (unsigned long long)a.head_line[r + 1] : a.NL;
    const unsigned long long k = nxt - h - 1;                       // sequence lines
    unsigned long long so = 0, w = 1, L = 0;
    if (k) {
        so = fa_start(a, h + 1);
        w = fa_end(a, h + 1) - so;
        const unsigned long long last = fa_end(a, nxt - 1) - fa_start(a, nxt - 1);
        L = (k - 1) * w + last;
        if (last > w || w == 0) { atomicOr(a.bad, 1); w = 1; }
    }
    if (L > 0x7FFFFFFFull) { atomicOr(a.bad, 1); L = 0; }           // kseq's int length
    a.seq_off[r] = (uint32_t)so;
    a.width[r] = (uint32_t)w;
    a.len[r] = (int32_t)L;
    a.padded[r] = (L + FL_ALIGN_BASES - 1) & ~(unsigned long long)(FL_ALIGN_BASES - 1);
}

// per sequence line that is not its record's last: it must have the record's width
__global__ void __launch_bounds__(256) k_fa_lines(FaArgs a) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.NL || i + 1 >= a.NL) return;                         // the chunk's last line is some record's last
    const unsigned long long s = fa_start(a, i), e = fa_end(a, i);
    if (e > s && a.text[s] == '>') return;                          // header
    const unsigned long long s2 = e + 1, e2 = fa_end(a, i + 1);
    if (e2 > s2 && a.text[s2] == '>') return;                       // the next line is a header: this one is its record's last
    const unsigned long long hb = a.head[i];                        // headers before this line (>= 1 unless the chunk is bad)
    if (hb == 0) return;
    const unsigned long long h = a.head_line[hb - 1];
    const unsigned long long w = fa_end(a, h + 1) - fa_start(a, h + 1);
    if (e - s != w) atomicOr(a.bad, 1);
}

// 32 bases per lane and step, packed to 2 bits with the non-ACGT mask. The work is the arena's 32-base groups, not the
// records: an assembly is a handful of records of hundreds of megabases, a read file millions of short ones, and a group
// never straddles two records (their arena extents are multiples of 64). Each lane finds its group's record by bisection
// over the offsets.
__global__ void __launch_bounds__(256) k_fa_gather(const uint8_t *__restrict__ text, uint32_t n_rec, const uint32_t *__restrict__ seq_off,
                                                   const uint32_t *__restrict__ width, const int32_t *__restrict__ len,
                                                   const unsigned long long *__restrict__ off, unsigned long long padded_bases,
                                                   uint32_t *__restrict__ seq2b, uint32_t *__restrict__ nmask) {
    const unsigned long long n_groups = padded_bases >> 5;
    for (unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups;
         g += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long pos = g << 5;                            // arena position of the group's first base
        uint32_t lo = 0, hi = n_rec;                                      // the last record with off[r] <= pos
        while (hi - lo > 1) {
            const uint32_t mid = lo + ((hi - lo) >> 1);
            if (off[mid] <= pos) lo = mid;
            else hi = mid;
        }
        const uint32_t r = lo;
        const int L = len[r];
        const unsigned w = width[r];
        const unsigned long long so = seq_off[r];
        const unsigned b = (unsigned)(pos - off[r]);                      // < the record's padded length (empty records own no group)
        const unsigned q = b / w;
        unsigned col = b - q * w;
        unsigned long long p = so + b + q;                                // byte of base b: one newline per full line before it
        uint32_t w0 = 0, w1 = 0, m = 0;
#pragma unroll 8
        for (int i = 0; i < 32; ++i) {
            if ((int)b + i < L) {
                const unsigned ch = text[p] & 0xDFu;                      // kmers.cpp:176-196: case folded, anything but ACGT is code 0
                const unsigned code = ch == 'C' ? 1u : ch == 'G' ? 2u : ch == 'T' ? 3u : 0u;
                if (code == 0u && ch != 'A') m |= 1u << i;
                if (i < 16) w0 |= code << (30 - 2 * i);
                else w1 |= code << (30 - 2 * (i - 16));
                ++p;
                if (++col == w) { col = 0; ++p; }                         // step over the newline
            }
        }
        reinterpret_cast<uint2 *>(seq2b)[g] = make_uint2(w0, w1);
        nmask[g] = m;
    }
}

}  // namespace

// The front half of both text entry points: stage the chunk, index its newlines, validate the records of the common
// layout and lay out the arena (padded offsets). ix.done: the caller returns at once (nothing to do, or not the layout).
struct TextIndex {
    fl_ctx::Staging *S = nullptr;
    RecArgs ra{};
    const uint8_t *text = nullptr;
    unsigned long long n_rec = 0, padded_bases = 0, consumed = 0;
    const uint32_t *fa_width = nullptr;        // wrapped-FASTA index: the records' line widths (then k_fa_gather does the packing)
    bool done = false;
};

// stage the chunk (copy stream, double buffered like fl_reads_push) and count its lines
struct TextLines {
    fl_ctx::Staging *S = nullptr;
    const uint8_t *text = nullptr;
    unsigned long long n_blocks = 0, n_lines = 0, n_lines_virtual = 0;
    unsigned grid = 0;
    bool ends_with_nl = false;
    bool has_nul = false;             // a NUL byte anywhere in the chunk: not the layout
};

static int text_lines(fl_ctx *c, const char *host_text, uint64_t n_bytes, int is_last_chunk, TextLines &tl) {
    const int slot = c->stg_next;
    c->stg_next ^= 1;
    fl_ctx::Staging &S = c->stg[slot];
    tl.S = &S;
    if (!S.consumed) FL_CUDA(c, cudaEventCreateWithFlags(&S.consumed, cudaEventDisableTiming));
    if (S.in_use) FL_CUDA(c, cudaEventSynchronize(S.consumed));
    S.in_use = false;
    cudaStream_t st = c->stream;
    FL_CUDA(c, S.ascii.reserve((size_t)n_bytes + 64, 0, c->copy_stream));
    FL_CUDA(c, cudaMemcpyAsync(S.ascii.p, host_text, (size_t)n_bytes, cudaMemcpyHostToDevice, c->copy_stream));
    FL_CUDA(c, cudaEventRecord(c->ev_copied, c->copy_stream));
    FL_CUDA(c, cudaStreamWaitEvent(st, c->ev_copied, 0));
    const uint8_t *text = S.ascii.p;
    tl.text = text;
    // ---- newline index, pass A ----
    tl.n_blocks = (n_bytes + TX_LINES_PER_WARP - 1) / TX_LINES_PER_WARP;
    FL_CUDA(c, c->sc_u64a.reserve(tl.n_blocks + 1, 0, st));
    tl.grid = fl_blocks(tl.n_blocks * 32, 256);
    if (tl.grid > (unsigned)c->sm_count * 16) tl.grid = (unsigned)c->sm_count * 16;
    int *d_nul = reinterpret_cast<int *>(c->d_scalars + 29);
    FL_CUDA(c, cudaMemsetAsync(d_nul, 0, sizeof(unsigned long long), st));
    k_text_count<<<tl.grid, 256, 0, st>>>(text, n_bytes, tl.n_blocks, c->sc_u64a.p, d_nul);
    c->launches++;
    FL_TRY(fl_exclusive_scan_u64(c, c->sc_u64a.p, c->sc_u64a.p, tl.n_blocks, c->d_scalars));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars, c->d_scalars, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 1, text + n_bytes - 1, 1, cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 6, d_nul, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaStreamSynchronize(st));
    tl.has_nul = c->h_scalars[6] != 0;
    tl.n_lines = c->h_scalars[0];
    tl.ends_with_nl = (reinterpret_cast<const unsigned char *>(c->h_scalars + 1))[0] == '\n';
    tl.n_lines_virtual = tl.n_lines + ((is_last_chunk && !tl.ends_with_nl) ? 1 : 0);   // the file's last line may lack its newline
    return FL_OK;
}

// pass B of the newline index: positions, in order, into c->tx_nl
static int text_positions(fl_ctx *c, uint64_t n_bytes, const TextLines &tl) {
    FL_CUDA(c, c->tx_nl.reserve(tl.n_lines + 1, 0, c->stream));
    k_text_positions<<<tl.grid, 256, 0, c->stream>>>(tl.text, n_bytes, tl.n_blocks, c->sc_u64a.p, c->tx_nl.p);
    c->launches++;
    return FL_OK;
}

static int text_index(fl_ctx *c, const char *host_text, uint64_t n_bytes, int lpr, int is_last_chunk, bool have_cap, uint64_t cap,
                      uint64_t *n_records, int *status, TextIndex &ix) {
    TextLines tl;
    FL_TRY(text_lines(c, host_text, n_bytes, is_last_chunk, tl));
    fl_ctx::Staging &S = *tl.S;
    ix.S = &S;
    cudaStream_t st = c->stream;
    const uint8_t *text = tl.text;
    ix.text = text;
    const unsigned long long n_lines = tl.n_lines, n_lines_virtual = tl.n_lines_virtual;
    if (tl.has_nul || (lpr == 2 && (n_lines_virtual & 1ull))) {
        // a NUL (see k_text_count), or FASTA with
        // a line left over after the last pair, which may continue that record's sequence (a wrapped
        // record): the record is not what it seems, and kseq would read on. Not the simple layout.
        FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));
        *status = FL_TEXT_FALLBACK;
        ix.done = true;
        return FL_OK;
    }
    const unsigned long long n_rec = n_lines_virtual / lpr;
    ix.n_rec = n_rec;
    if (n_rec == 0 || n_rec > 0xFFFFFFF0ull) {
        // not even one whole record in the chunk (or an absurd count): let the host parser deal with this input
        FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));
        *status = is_last_chunk && n_lines_virtual == 0 ? FL_TEXT_OK : FL_TEXT_FALLBACK;
        ix.done = true;
        return FL_OK;
    }
    if (have_cap && cap < n_rec) {                          // nothing was done: *n_records tells the caller what to provide
        FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));
        *n_records = n_rec;
        c->set_error("fl_reads_push_text: the record arrays are too small");
        return FL_ERANGE;
    }
    FL_TRY(text_positions(c, n_bytes, tl));
    // ---- records ----
    const size_t n = (size_t)n_rec;
    FL_CUDA(c, c->tx_u32.reserve(5 * n + 8, 0, st));
    FL_CUDA(c, c->sc_u64b.reserve(n + 1, 0, st));       // name hashes
    FL_CUDA(c, S.off.reserve(n + 1, 0, st));            // padded lengths -> offsets
    FL_CUDA(c, S.len.reserve(n, 0, st));
    RecArgs &ra = ix.ra;
    ra = RecArgs{};
    ra.text = text; ra.n_bytes = n_bytes; ra.nl = c->tx_nl.p; ra.n_lines = n_lines; ra.n_rec = (uint32_t)n_rec; ra.lines_per_rec = lpr;
    ra.name_off = c->tx_u32.p; ra.name_len = c->tx_u32.p + n; ra.comment_len = c->tx_u32.p + 2 * n; ra.seq_off = c->tx_u32.p + 3 * n;
    ra.qual_off = c->tx_u32.p + 4 * n;
    ra.len = S.len.p; ra.name_hash = c->sc_u64b.p; ra.padded = reinterpret_cast<unsigned long long *>(S.off.p);
    int *d_bad = reinterpret_cast<int *>(c->d_scalars + 27);
    FL_CUDA(c, cudaMemsetAsync(d_bad, 0, sizeof(unsigned long long), st));
    ra.bad = d_bad;
    k_text_records<<<fl_blocks(n, 256), 256, 0, st>>>(ra);
    c->launches++;
    FL_TRY(fl_exclusive_scan_u64(c, reinterpret_cast<unsigned long long *>(S.off.p), reinterpret_cast<unsigned long long *>(S.off.p), n, c->d_scalars + 1));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 2, d_bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 3, c->d_scalars + 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 4, c->tx_nl.p + (n_rec * lpr - 1 < n_lines ? n_rec * lpr - 1 : n_lines - 1), sizeof(uint32_t),
                               cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaStreamSynchronize(st));
    if (c->h_scalars[2] != 0) {                             // not the simple layout: nothing was done
        FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));
        *status = FL_TEXT_FALLBACK;
        ix.done = true;
        return FL_OK;
    }
    ix.padded_bases = c->h_scalars[3];
    ix.consumed = (n_rec * lpr - 1 < n_lines) ? (unsigned long long)(*reinterpret_cast<uint32_t *>(c->h_scalars + 4)) + 1 : n_bytes;
    return FL_OK;
}

// The index of a FASTA reference chunk whose records may be wrapped (see k_fa_heads ...): same outputs as text_index
// (S.len, S.off, ix.ra.seq_off) plus the records' line widths. The whole chunk is consumed or nothing is.
static int fasta_index(fl_ctx *c, const char *host_text, uint64_t n_bytes, int is_last_chunk, int *status, TextIndex &ix) {
    TextLines tl;
    FL_TRY(text_lines(c, host_text, n_bytes, is_last_chunk, tl));
    fl_ctx::Staging &S = *tl.S;
    ix.S = &S;
    ix.text = tl.text;
    cudaStream_t st = c->stream;
    auto fallback = [&]() -> int {
        FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));
        *status = FL_TEXT_FALLBACK;
        ix.done = true;
        return FL_OK;
    };
    const unsigned long long NL = tl.n_lines_virtual;
    // a chunk that is not the file's last must end with a newline (the caller cuts at record starts), and there must be lines
    if (tl.has_nul || NL == 0 || NL > 0xFFFFFFF0ull || (!tl.ends_with_nl && !is_last_chunk)) return fallback();
    FL_TRY(text_positions(c, n_bytes, tl));
    FL_CUDA(c, c->sc_u64c.reserve((size_t)NL + 1, 0, st));
    FaArgs a{};
    a.text = tl.text; a.n_bytes = n_bytes; a.nl = c->tx_nl.p; a.n_lines = tl.n_lines; a.NL = NL; a.head = c->sc_u64c.p;
    int *d_bad = reinterpret_cast<int *>(c->d_scalars + 27);
    FL_CUDA(c, cudaMemsetAsync(d_bad, 0, sizeof(unsigned long long), st));
    a.bad = d_bad;
    const unsigned lgrid = fl_blocks((size_t)NL, 256);
    k_fa_heads<<<lgrid, 256, 0, st>>>(a);
    c->launches++;
    FL_TRY(fl_exclusive_scan_u64(c, c->sc_u64c.p, c->sc_u64c.p, (size_t)NL, c->d_scalars + 1));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 2, d_bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 3, c->d_scalars + 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaStreamSynchronize(st));
    const unsigned long long n_rec = c->h_scalars[3];
    if (c->h_scalars[2] != 0 || n_rec == 0 || n_rec > 0xFFFFFFF0ull) return fallback();
    const size_t n = (size_t)n_rec;
    ix.n_rec = n_rec;
    FL_CUDA(c, c->tx_u32.reserve(3 * n + 8, 0, st));
    FL_CUDA(c, S.off.reserve(n + 1, 0, st));
    FL_CUDA(c, S.len.reserve(n, 0, st));
    a.n_rec = (uint32_t)n_rec;
    a.head_line = c->tx_u32.p; a.seq_off = c->tx_u32.p + n; a.width = c->tx_u32.p + 2 * n;
    a.len = S.len.p; a.padded = reinterpret_cast<unsigned long long *>(S.off.p);
    k_fa_scatter<<<lgrid, 256, 0, st>>>(a);
    k_fa_records<<<fl_blocks(n, 256), 256, 0, st>>>(a);
    k_fa_lines<<<lgrid, 256, 0, st>>>(a);
    c->launches += 3;
    FL_TRY(fl_exclusive_scan_u64(c, reinterpret_cast<unsigned long long *>(S.off.p), reinterpret_cast<unsigned long long *>(S.off.p), n, c->d_scalars + 1));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 2, d_bad, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 3, c->d_scalars + 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaStreamSynchronize(st));
    if (c->h_scalars[2] != 0) return fallback();
    ix.padded_bases = c->h_scalars[3];
    ix.consumed = n_bytes;
    ix.ra = RecArgs{};
    ix.ra.seq_off = a.seq_off;
    ix.fa_width = a.width;
    return FL_OK;
}

extern "C" int fl_reads_push_text(fl_ctx *c, const char *host_text, uint64_t n_bytes, int format, int is_last_chunk,
                                  const fl_text_records *out, uint64_t *n_records, uint64_t *bytes_consumed, int *status) {
    FL_ENTER(c);
    if (!host_text || !n_records || !bytes_consumed || !status || (format != FL_TEXT_FASTQ && format != FL_TEXT_FASTA)) {
        c->set_error("fl_reads_push_text: bad arguments");
        return FL_EINVAL;
    }
    if (n_bytes >= ((uint64_t)1 << 31)) { c->set_error("fl_reads_push_text: a chunk must be smaller than 2 GiB"); return FL_ERANGE; }
    *n_records = 0;
    *bytes_consumed = 0;
    *status = FL_TEXT_OK;
    if (n_bytes == 0) return FL_OK;
    FL_TRY(fl_sets_ready(c));
    const bool kmer_mode = c->ref.n > 0;
    if (!kmer_mode && format == FL_TEXT_FASTA) { *status = FL_TEXT_FALLBACK; return FL_OK; }    // main.cpp:103-106 is the host's error to print
    const int lpr = format == FL_TEXT_FASTQ ? 4 : 2;
    TextIndex ix;
    FL_TRY(text_index(c, host_text, n_bytes, lpr, is_last_chunk, out != nullptr, out ? out->cap : 0, n_records, status, ix));
    if (ix.done) return FL_OK;
    fl_ctx::Staging &S = *ix.S;
    cudaStream_t st = c->stream;
    const uint8_t *text = ix.text;
    const unsigned long long n_rec = ix.n_rec, padded_bases = ix.padded_bases, consumed = ix.consumed;
    const size_t n = (size_t)n_rec;
    RecArgs &ra = ix.ra;
    // ---- gather into the arena, score ----
    BatchView v{};
    v.n = (uint32_t)n_rec; v.padded_bases = padded_bases; v.off = S.off.p; v.len = S.len.p;
    unsigned ggrid = fl_blocks(n * 32, 256);
    if (ggrid > (unsigned)c->sm_count * 16) ggrid = (unsigned)c->sm_count * 16;
    if (fl_wants_bases(c)) {                                   // k-mer mode, or a contaminant set to probe
        FL_CUDA(c, S.seq.reserve((size_t)(padded_bases >> 4) + 8, 0, st));
        k_text_gather<false><<<ggrid, 256, 0, st>>>(text, n_bytes, (uint32_t)n_rec, ra.seq_off, S.len.p, reinterpret_cast<unsigned long long *>(S.off.p),
                                                    S.seq.p, nullptr, nullptr);
        v.seq2b = S.seq.p;
        c->launches++;
    }
    if (!kmer_mode) {
        FL_CUDA(c, S.qual.reserve((size_t)padded_bases + 64, 0, st));
        k_text_gather<true><<<ggrid, 256, 0, st>>>(text, n_bytes, (uint32_t)n_rec, ra.qual_off, S.len.p, reinterpret_cast<unsigned long long *>(S.off.p),
                                                   nullptr, S.qual.p, nullptr);
        v.qual = S.qual.p;
        c->launches++;
    }
    FL_CUDA(c, cudaGetLastError());
    // the caller's record index (offsets are relative to the chunk's first byte)
    if (out) {
        auto dl32 = [&](uint32_t *dst, const uint32_t *src) -> int {
            if (dst) FL_CUDA(c, cudaMemcpyAsync(dst, src, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
            return FL_OK;
        };
        auto dl64 = [&](uint64_t *dst, const uint32_t *src, DevVec<unsigned long long> &tmp, size_t slot_i) -> int {
            if (!dst) return FL_OK;
            FL_CUDA(c, tmp.reserve(3 * n + 8, 0, st));
            unsigned long long *t = tmp.p + slot_i * n;
            k_text_u32_to_u64<<<fl_blocks(n, 256), 256, 0, st>>>(src, (uint32_t)n, 0ull, t);
            FL_CUDA(c, cudaMemcpyAsync(dst, t, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
            return FL_OK;
        };
        FL_TRY(dl32(out->name_len, ra.name_len));
        FL_TRY(dl32(out->comment_len, ra.comment_len));
        FL_TRY(dl64(out->name_off, ra.name_off, c->sc_u64c, 0));
        FL_TRY(dl64(out->seq_off, ra.seq_off, c->sc_u64c, 1));
        FL_TRY(dl64(out->qual_off, ra.qual_off, c->sc_u64c, 2));
        if (out->len) FL_CUDA(c, cudaMemcpyAsync(out->len, S.len.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (out->name_hash) FL_CUDA(c, cudaMemcpyAsync(out->name_hash, c->sc_u64b.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        FL_CUDA(c, cudaStreamSynchronize(st));       // the index is the caller's as soon as the call returns
    }
    FL_TRY(fl_score_view(c, v));
    k_text_sum_len<<<c->sm_count, 256, 0, st>>>(S.len.p, (uint32_t)n_rec, c->d_scalars + 16);     // main.cpp:89
    c->launches++;
    FL_CUDA(c, cudaGetLastError());
    FL_CUDA(c, cudaEventRecord(S.consumed, st));
    S.in_use = true;
    FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));   // the caller may reuse its buffer now
    *n_records = n_rec;
    *bytes_consumed = consumed;
    return FL_OK;
}

// A 16-mer set from TEXT (kmers.cpp:75-134 behind kseq): the same front half, then the sequences -- every record's,
// also those shorter than 16, which add nothing (kmers.cpp:99-100) but are counted (kmers.cpp:96) -- packed with their
// non-ACGT mask and handed to the build kernels.
static int add_text(fl_ctx *c, KmerSet &set, const char *entry, const char *host_text, uint64_t n_bytes, int format, int is_last_chunk,
                    int require_multiple_copies, uint64_t *n_records, uint64_t *n_bases, uint64_t *bytes_consumed, int *status) {
    if (!host_text || !n_records || !n_bases || !bytes_consumed || !status || (format != FL_TEXT_FASTQ && format != FL_TEXT_FASTA)) {
        c->set_error(std::string(entry) + ": bad arguments");
        return FL_EINVAL;
    }
    if (n_bytes >= ((uint64_t)1 << 31)) { c->set_error(std::string(entry) + ": a chunk must be smaller than 2 GiB"); return FL_ERANGE; }
    *n_records = 0;
    *n_bases = 0;
    *bytes_consumed = 0;
    *status = FL_TEXT_OK;
    if (require_multiple_copies) FL_TRY(fl_kmers_check_multi(c, entry));
    if (n_bytes == 0) return FL_OK;
    TextIndex ix;
    if (format == FL_TEXT_FASTA && !c->fasta_two_line_only) FL_TRY(fasta_index(c, host_text, n_bytes, is_last_chunk, status, ix));
    else FL_TRY(text_index(c, host_text, n_bytes, format == FL_TEXT_FASTQ ? 4 : 2, is_last_chunk, false, 0, n_records, status, ix));
    if (ix.done) return FL_OK;
    fl_ctx::Staging &S = *ix.S;
    cudaStream_t st = c->stream;
    const size_t n = (size_t)ix.n_rec;
    BatchView v{};
    v.n = (uint32_t)ix.n_rec; v.padded_bases = ix.padded_bases; v.off = S.off.p; v.len = S.len.p;
    unsigned ggrid = fl_blocks(n * 32, 256);
    if (ggrid > (unsigned)c->sm_count * 16) ggrid = (unsigned)c->sm_count * 16;
    FL_CUDA(c, S.seq.reserve((size_t)(ix.padded_bases >> 4) + 8, 0, st));
    FL_CUDA(c, S.nmask.reserve((size_t)(ix.padded_bases >> 5) + 8, 0, st));
    if (ix.fa_width) {
        unsigned fgrid = fl_blocks((size_t)(ix.padded_bases >> 5), 256);
        if (fgrid > (unsigned)c->sm_count * 16) fgrid = (unsigned)c->sm_count * 16;
        if (fgrid)
            k_fa_gather<<<fgrid, 256, 0, st>>>(ix.text, (uint32_t)ix.n_rec, ix.ra.seq_off, ix.fa_width, S.len.p,
                                               reinterpret_cast<unsigned long long *>(S.off.p), ix.padded_bases, S.seq.p, S.nmask.p);
    } else
        k_text_gather<false><<<ggrid, 256, 0, st>>>(ix.text, n_bytes, (uint32_t)ix.n_rec, ix.ra.seq_off, S.len.p,
                                                    reinterpret_cast<unsigned long long *>(S.off.p), S.seq.p, nullptr, S.nmask.p);
    c->launches++;
    v.seq2b = S.seq.p;
    v.nmask = S.nmask.p;
    // bases of the sequences that take part (the progress line of kmers.cpp:101,123-126 counts only those)
    unsigned long long *d_sum = c->d_scalars + 28;
    FL_CUDA(c, cudaMemsetAsync(d_sum, 0, sizeof(unsigned long long), st));
    k_text_sum_len<<<c->sm_count, 256, 0, st>>>(S.len.p, (uint32_t)ix.n_rec, d_sum, 16);
    c->launches++;
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 5, d_sum, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaGetLastError());
    FL_TRY(fl_kmers_add_view(c, set, v, require_multiple_copies ? 1 : 0));  // synchronises the stream on its way
    FL_CUDA(c, cudaEventRecord(S.consumed, st));
    S.in_use = true;
    FL_CUDA(c, cudaStreamSynchronize(c->copy_stream));   // the caller may reuse its buffer now
    FL_CUDA(c, cudaStreamSynchronize(st));
    *n_records = ix.n_rec;
    *n_bases = c->h_scalars[5];
    *bytes_consumed = ix.consumed;
    return FL_OK;
}

extern "C" int fl_kmers_add_text(fl_ctx *c, const char *host_text, uint64_t n_bytes, int format, int is_last_chunk, int require_multiple_copies,
                                 uint64_t *n_records, uint64_t *n_bases, uint64_t *bytes_consumed, int *status) {
    FL_ENTER(c);
    return add_text(c, c->ref, "fl_kmers_add_text", host_text, n_bytes, format, is_last_chunk, require_multiple_copies, n_records, n_bases, bytes_consumed, status);
}

extern "C" int fl_contam_add_text(fl_ctx *c, const char *host_text, uint64_t n_bytes, int format, int is_last_chunk, uint64_t *n_records,
                                  uint64_t *n_bases, uint64_t *bytes_consumed, int *status) {
    FL_ENTER(c);
    FL_TRY(fl_contam_check_order(c));
    return add_text(c, c->contam, "fl_contam_add_text", host_text, n_bytes, format, is_last_chunk, 0, n_records, n_bases, bytes_consumed, status);
}

// pinned host memory for the caller's chunk ring (the host side links no CUDA runtime of its own)
extern "C" int fl_host_alloc(uint64_t n_bytes, void **out) {
    if (!out) return FL_EINVAL;
    *out = nullptr;
    return cudaHostAlloc(out, (size_t)n_bytes, cudaHostAllocPortable) == cudaSuccess ? FL_OK : FL_ENOMEM;
}

extern "C" void fl_host_free(void *p) {
    if (p) cudaFreeHost(p);
}

// page-lock memory the caller already owns (and may already be filling): lets a reader thread start on the
// input while the CUDA context is still coming up
extern "C" int fl_host_register(void *p, uint64_t n_bytes) {
    if (!p) return FL_EINVAL;
    if (cudaHostRegister(p, (size_t)n_bytes, cudaHostRegisterPortable) == cudaSuccess) return FL_OK;
    (void)cudaGetLastError();
    return FL_ENOMEM;
}

extern "C" void fl_host_unregister(void *p) {
    if (p && cudaHostUnregister(p) != cudaSuccess) (void)cudaGetLastError();
}

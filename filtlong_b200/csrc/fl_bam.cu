// filtlong_b200/csrc/fl_bam.cu -- unaligned BAM records to the scoring arena.
//
// The host (host/bam.cpp) inflates the BAM file, walks its records, checks them and hands over a chunk of whole records
// with where each record's SEQ and QUAL start. Here the chunk is staged like a text chunk (fl_text.cu) and one warp per
// record gathers what the scoring mode reads into the arena:
//   * Phred mode: the QUAL bytes + 33, i.e. the quality line of the record's FASTQ equivalent;
//   * k-mer mode: the 4-bit SEQ codes (=ACMGRSVTWYHKDBN) as the arena's 2-bit codes. A, C, G, T are 1, 2, 4, 8 and become
//     0..3; every other code becomes 0, which is what the reference's base_to_bits_forward gives a base outside ACGT.
// Then the batch is scored like every other one (fl_score_view).
//
// On the way out, k_bam_build writes the BAM records of pass 2 (fl_bam_build, fl_bam_writer): whole records and the
// header copied, the children of trimmed and split reads built from their parent, with --keep_mods re-based
// modification tags (fl_bam_mods.h). DESIGN 4.13.
#include "fl_bam_mods.h"
#include "fl_device.cuh"

namespace {

// W little-endian words of the chunk starting at byte offset o (any alignment, negative allowed); no word before word 0
// or past last_word is read
template <int W>
__device__ __forceinline__ void bam_load(const uint32_t *__restrict__ t32, long long o, long long last_word, uint32_t (&out)[W]) {
    const long long w0 = o >> 2;                                          // floor, also for o < 0
    const unsigned sh = ((unsigned)o & 3u) * 8u;
    uint32_t prev = __ldg(t32 + min(max(w0, 0ll), last_word));
#pragma unroll
    for (int i = 0; i < W; ++i) {
        const long long wi = w0 + 1 + i;
        const uint32_t nxt = __ldg(t32 + min(max(wi, 0ll), last_word));
        out[i] = __funnelshift_r(prev, nxt, sh);
        prev = nxt;
    }
}

// 2-bit arena code of a 4-bit SEQ code, two bits per code: C (2) -> 1, G (4) -> 2, T (8) -> 3, everything else -> 0
#define BAM_NIBBLE_CODES 0x30210u
// the same for the complement: A (1) -> 3, C (2) -> 2, G (4) -> 1, T (8) -> 0, everything else -> 0
#define BAM_NIBBLE_RC_CODES 0x0012Cu

// One warp per record, 32 bases per lane and step (like k_text_gather). Bases at or beyond the record's length are
// written as 0 in both arenas, as the host packer leaves them.
//
// reverse (may be NULL: all forward): the record stores its read reverse-complemented (BAM flag 0x10), and the arena gets
// the read in its original orientation. Arena bases [b, b + 32) then come from the stored bases [L - b - 32, L - b),
// last first: in Phred mode the QUAL bytes in reverse order, in k-mer mode the SEQ codes in reverse order, complemented.
// The first stored base can be odd (the codes start half a byte into the first loaded byte) and, near the read's end,
// negative (before the record, for the first record of a chunk before the chunk: the loads clamp at word 0); every
// arena base it would feed lies at or past L and is masked to 0.
template <bool PHRED>
__global__ void __launch_bounds__(256) k_bam_gather(const uint8_t *__restrict__ chunk, unsigned long long n_bytes, uint32_t n_rec,
                                                    const uint32_t *__restrict__ seq_off, const uint32_t *__restrict__ qual_off,
                                                    const int32_t *__restrict__ len, const uint8_t *__restrict__ reverse,
                                                    const unsigned long long *__restrict__ off, uint32_t *__restrict__ seq2b,
                                                    uint8_t *__restrict__ qual) {
    const unsigned lane = threadIdx.x & 31;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((size_t)gridDim.x * blockDim.x) >> 5;
    const uint32_t *t32 = reinterpret_cast<const uint32_t *>(chunk);
    const long long last_word = n_bytes ? (long long)((n_bytes - 1) >> 2) : 0;
    for (size_t r = warp; r < n_rec; r += n_warps) {
        const int L = len[r];
        const bool rev = reverse && reverse[r];                          // one warp per record: uniform
        const unsigned long long dof = off[r];
        const int padded = (int)(((unsigned)L + 63u) & ~63u);
        const long long src = PHRED ? qual_off[r] : seq_off[r];
        for (int b = 32 * (int)lane; b < padded; b += 1024) {
            const int nv = L - b;                                         // valid bases of these 32
            if (PHRED) {
                uint32_t c[8];
                bam_load<8>(t32, src + (rev ? nv - 32 : b), last_word, c);
                if (rev) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint32_t t = c[i];
                        c[i] = __byte_perm(c[7 - i], 0, 0x0123);
                        c[7 - i] = __byte_perm(t, 0, 0x0123);
                    }
                }
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
                uint32_t w[2] = {0u, 0u};
                if (!rev) {
                    bam_load<4>(t32, src + (b >> 1), last_word, c);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint32_t byte = (c[i] >> (8 * k)) & 0xFFu;
                            const int q = 8 * i + 2 * k;                  // base of the high nibble, 0..30
                            const uint32_t hi = (BAM_NIBBLE_CODES >> (2 * (byte >> 4))) & 3u, lo = (BAM_NIBBLE_CODES >> (2 * (byte & 15u))) & 3u;
                            w[q >> 4] |= ((hi << 2) | lo) << (28 - 2 * (q & 15));
                        }
                    }
                } else {
                    // stored codes from n0 = 2 * src + nv - 32 on (a code index); the 16 bytes from code n0 & ~1 give arena
                    // bases 31 - q for their codes q; an odd n0 moves them one base on, and base 0 is then the high code of
                    // the 17th byte
                    const long long n0 = 2 * src + nv - 32;
                    bam_load<4>(t32, n0 >> 1, last_word, c);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint32_t byte = (c[i] >> (8 * k)) & 0xFFu;
                            const int q = 31 - (8 * i + 2 * k);           // arena base of the high nibble, 31..1
                            const uint32_t hi = (BAM_NIBBLE_RC_CODES >> (2 * (byte >> 4))) & 3u, lo = (BAM_NIBBLE_RC_CODES >> (2 * (byte & 15u))) & 3u;
                            w[q >> 4] |= hi << (30 - 2 * (q & 15));
                            w[(q - 1) >> 4] |= lo << (30 - 2 * ((q - 1) & 15));
                        }
                    }
                    if (n0 & 1) {
                        const long long wb = (n0 >> 1) + 16;                     // the 17th byte
                        const uint32_t byte = (__ldg(t32 + min(max(wb >> 2, 0ll), last_word)) >> (8 * (unsigned)(wb & 3))) & 0xFFu;
                        w[1] = __funnelshift_r(w[1], w[0], 2);
                        w[0] = (w[0] >> 2) | (((BAM_NIBBLE_RC_CODES >> (2 * (byte >> 4))) & 3u) << 30);
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


// 4 little-endian bytes at any address of a buffer that is readable 4 bytes past it
__device__ __forceinline__ uint32_t ld_u32(const uint8_t *p) {
    const uintptr_t a = (uintptr_t)p;
    const uint32_t *w = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
    return __funnelshift_r(__ldg(w), __ldg(w + 1), (unsigned)(a & 3) * 8u);
}

// ODD: byte k of a SEQ slice that starts at an odd base, from the packed bytes src of the base before it: the low nibble
// of src[k], then the high nibble of src[k + 1]
template <bool ODD>
__device__ __forceinline__ uint8_t piece_byte(const uint8_t *src, uint64_t k) {
    return ODD ? (uint8_t)((src[k] << 4) | (src[k + 1] >> 4)) : src[k];
}
template <bool ODD>
__device__ __forceinline__ uint32_t piece_word(const uint8_t *src) {
    const uint32_t w = ld_u32(src);
    return ODD ? ((w << 4) & 0xF0F0F0F0u) | ((ld_u32(src + 1) >> 4) & 0x0F0F0F0Fu) : w;
}

// dst[0, n) from src (any alignments), by the whole warp: bytes up to a 16-byte boundary of dst, then 16-byte stores of
// words gathered with funnel shifts, then the bytes left
template <bool ODD>
__device__ void warp_copy(uint8_t *dst, const uint8_t *src, uint64_t n, unsigned lane) {
    uint64_t head = (16 - ((uintptr_t)dst & 15)) & 15;
    if (head > n) head = n;
    if (lane < head) dst[lane] = piece_byte<ODD>(src, lane);
    const uint64_t body = (n - head) >> 4;
    uint4 *d = reinterpret_cast<uint4 *>(dst + head);
    const uint8_t *q = src + head;
    for (uint64_t i = lane; i < body; i += 32)
        d[i] = make_uint4(piece_word<ODD>(q + 16 * i), piece_word<ODD>(q + 16 * i + 4), piece_word<ODD>(q + 16 * i + 8),
                          piece_word<ODD>(q + 16 * i + 12));
    for (uint64_t k = head + 16 * body + lane; k < n; k += 32) dst[k] = piece_byte<ODD>(src, k);
}

// nibbles of x equal to `code`, among the nibbles whose lowest bit is set in m
__device__ __forceinline__ uint32_t nibbles_eq(uint32_t x, uint32_t code, uint32_t m) {
    const uint32_t z = x ^ (code * 0x11111111u);
    return __popc(~(z | (z >> 1) | (z >> 2) | (z >> 3)) & m);
}

// adds to cnt[0..3] the bases A, C, G, T (codes 1, 2, 4, 8) among SEQ positions [a, b), by the whole warp: 8 bases per
// lane and word, compared nibble-wise and counted with __popc (base 2j of a word in the high nibble of byte j)
__device__ void warp_count(const uint8_t *seq, uint32_t a, uint32_t b, unsigned lane, uint32_t cnt[4]) {
    uint32_t c[4] = {0, 0, 0, 0};
    for (uint32_t w = a / 8 + lane; w * 8ull < b; w += 32) {
        const uint32_t x = ld_u32(seq + 4ull * w), p0 = w * 8;
        uint32_t m = 0x11111111u;
        if (p0 < a || p0 + 8 > b) {
            m = 0;
#pragma unroll
            for (uint32_t k = 0; k < 8; ++k)
                if (p0 + k >= a && p0 + k < b) m |= 1u << (8 * (k >> 1) + ((k & 1) ? 0 : 4));
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) c[i] += nibbles_eq(x, 1u << i, m);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) cnt[i] += __reduce_add_sync(0xFFFFFFFFu, c[i]);
}

struct BamItemScratch {
    uint32_t before[8];            // A, C, G, T before the child's start, then before its end
    uint32_t mm_len, ml_n;         // the child's MM value and ML values
    uint32_t mm_at, ml_at;         // write pass: where its next group goes, from the child's first byte
};

// misc[]: the total, the first item outside the batch, the first child whose name is too long, the two counts
enum { BM_TOTAL = 0, BM_BAD = 1, BM_LONG = 2, BM_KEPT = 3, BM_INVALID = 4, BM_N = 5 };

// One warp per record: its children are consecutive items, so its SEQ and its MM string are walked once for all of
// them (children in the order of their starts; see fl_mm_rebase). Raw items are copied by one warp each. The size pass
// (WRITE = false) sizes every item, counts the bases before each child's ends and checks the record's tags; after an
// exclusive scan of the sizes the write pass writes every item at its offset. The serial parts -- aux fields, the MM
// walk, ML slices, the fixed fields and name -- are lane 0's; SEQ, QUAL and raw bytes are the warp's.
template <bool WRITE>
__global__ void __launch_bounds__(256) k_bam_build(const uint8_t *__restrict__ batch, unsigned long long n_bytes,
                                                   const fl_bam_item *__restrict__ items, unsigned long long n_items, int keep_mods,
                                                   BamItemScratch *__restrict__ scr, uint8_t *__restrict__ status,
                                                   unsigned long long *__restrict__ size, const unsigned long long *__restrict__ off,
                                                   uint8_t *__restrict__ out, unsigned long long *__restrict__ misc) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned long long warp = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5,
                             n_warps = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    for (unsigned long long i = warp; i < n_items; i += n_warps) {
        const fl_bam_item it = items[i];
        if (it.s < 0) {
            if (WRITE) warp_copy<false>(out + off[i], batch + it.off, (uint32_t)it.e, lane);
            else if (lane == 0) {
                status[i] = 0;
                size[i] = (uint32_t)it.e;
                if (it.e < 0 || it.off > n_bytes || (unsigned long long)it.e > n_bytes - it.off) atomicMin(misc + BM_BAD, i);
            }
            continue;
        }
        if (i > 0 && items[i - 1].s >= 0 && items[i - 1].off == it.off) continue;     // not its record's first child
        unsigned long long j_end = i + 1;
        while (j_end < n_items && items[j_end].s >= 0 && items[j_end].off == it.off) ++j_end;
        const uint8_t *rec = batch + it.off;
        if (!WRITE) {                          // the record and its fields lie in the batch, the children in the record
            bool ok = it.off + 36 <= n_bytes && 4ull + fl_rd32(rec) <= n_bytes - it.off;
            if (ok) {
                const uint64_t l_name = rec[12], n_cigar = rec[16] | (rec[17] << 8), l_seq = fl_rd32(rec + 20);
                ok = l_name >= 1 && 36 + l_name + 4 * n_cigar + (l_seq + 1) / 2 + l_seq <= 4ull + fl_rd32(rec);
                for (unsigned long long j = i; j < j_end; ++j) ok = ok && items[j].s < items[j].e && (uint64_t)items[j].e <= l_seq;
            }
            if (!ok) {
                if (lane == 0) {
                    atomicMin(misc + BM_BAD, i);
                    for (unsigned long long j = i; j < j_end; ++j) { size[j] = 0; status[j] = 0; }
                }
                continue;
            }
        }
        const uint32_t l_name = rec[12], n_cigar = rec[16] | (rec[17] << 8), l_seq = fl_rd32(rec + 20);
        const uint8_t *seq = rec + 36 + l_name + 4 * n_cigar, *qual = seq + (l_seq + 1) / 2, *end = rec + 4 + fl_rd32(rec);
        FlModTags t;
        fl_mod_tags(qual + l_seq, end, l_seq, &t);
        bool valid;
        if (!WRITE) {
            int stat = 0;
            valid = false;
            if (keep_mods && t.has_mm) {
                uint32_t tot[4] = {0, 0, 0, 0};
                warp_count(seq, 0, l_seq, lane, tot);
                const uint64_t count[5] = {tot[0], tot[1], tot[2], tot[3], l_seq};
                valid = fl_mods_valid(t, count);
                stat = valid ? FL_BAM_MODS_KEPT : FL_BAM_MODS_INVALID;
            }
            if (valid) {                                                 // the bases before each child's ends, in one walk
                uint32_t p = 0, run[4] = {0, 0, 0, 0};
                for (unsigned long long j = i; j < j_end; ++j) {
                    const uint32_t s = (uint32_t)items[j].s, e = (uint32_t)items[j].e;
                    if (s < p) { p = 0; run[0] = run[1] = run[2] = run[3] = 0; }
                    warp_count(seq, p, s, lane, run);
                    if (lane == 0) for (int b = 0; b < 4; ++b) scr[j].before[b] = run[b];
                    warp_count(seq, s, e, lane, run);
                    if (lane == 0) for (int b = 0; b < 4; ++b) scr[j].before[4 + b] = run[b];
                    p = e;
                }
            }
            if (lane == 0) {
                for (unsigned long long j = i; j < j_end; ++j) { scr[j].mm_len = 0; scr[j].ml_n = 0; }
                if (valid)                                               // group by group, the children in order
                    for (uint32_t p = 0; p < t.mm_len;) {
                        uint32_t head, codes;
                        int b;
                        fl_mm_head(t.mm, t.mm_len, p, &head, &b, &codes);
                        FlMMCursor cur = fl_mm_cursor(p + head);
                        for (unsigned long long j = i; j < j_end; ++j) {
                            const uint64_t bs = b == 4 ? (uint64_t)items[j].s : scr[j].before[b], be = b == 4 ? (uint64_t)items[j].e : scr[j].before[4 + b];
                            uint64_t k0, k1;
                            scr[j].mm_len += head + fl_mm_rebase(t.mm, t.mm_len, cur, bs, be, nullptr, &k0, &k1) + 1;
                            if (t.has_ml) scr[j].ml_n += (uint32_t)((k1 - k0) * codes);
                        }
                        uint64_t calls;
                        p = fl_mm_group_end(t.mm, cur, &calls);
                    }
                for (unsigned long long j = i; j < j_end; ++j) {
                    const int s = items[j].s, e = items[j].e;
                    const uint32_t nb = fl_child_name_bytes(l_name - 1, s, e);
                    if (nb > 255) atomicMin(misc + BM_LONG, j);
                    size[j] = fl_child_core_bytes(nb, (uint32_t)(e - s)) + t.rg_bytes + (valid ? fl_child_mods_bytes(t, scr[j].mm_len, scr[j].ml_n) : 0);
                    status[j] = (uint8_t)stat;
                }
                if (stat) atomicAdd(misc + (stat == FL_BAM_MODS_KEPT ? BM_KEPT : BM_INVALID), j_end - i);
            }
            continue;
        }
        valid = status[i] == FL_BAM_MODS_KEPT;
        const bool no_qual = qual[0] == 0xFF;
        for (unsigned long long j = i; j < j_end; ++j) {
            const int s = items[j].s, e = items[j].e;
            const uint32_t n = (uint32_t)(e - s), nb = fl_child_name_bytes(l_name - 1, s, e), nseq = (n + 1) / 2;
            uint8_t *dst = out + off[j], *dseq = dst + 36 + nb, *dqual = dseq + nseq;
            if (s & 1) warp_copy<true>(dseq, seq + s / 2, nseq, lane);
            else warp_copy<false>(dseq, seq + s / 2, nseq, lane);
            if (no_qual) for (uint32_t k = lane; k < n; k += 32) dqual[k] = 0xFF;
            else warp_copy<false>(dqual, qual + s, n, lane);
            __syncwarp();
            if (lane) continue;
            if (n & 1) dseq[nseq - 1] &= 0xF0;
            for (int k = 0; k < 36; ++k) dst[k] = rec[k];
            const uint32_t bs = (uint32_t)(size[j] - 4);
            for (int k = 0; k < 4; ++k) { dst[k] = (uint8_t)(bs >> (8 * k)); dst[20 + k] = (uint8_t)(n >> (8 * k)); }
            dst[12] = (uint8_t)nb;
            uint8_t *w = dst + 36;
            for (uint32_t k = 0; k + 1 < l_name; ++k) *w++ = rec[36 + k];
            *w++ = '_';
            w += fl_dec_write((uint64_t)s + 1, w);
            *w++ = '-';
            w += fl_dec_write((uint64_t)e, w);
            *w = 0;
            w = dqual + n;
            for (const uint8_t *a = qual + l_seq; a < end;) {          // the RG fields fl_mod_tags counted: up to one that
                const uint8_t *next = fl_aux_next(a, end);               // does not parse
                if (!next) break;
                if (a[0] == 'R' && a[1] == 'G') for (const uint8_t *x = a; x < next; ++x) *w++ = *x;
                a = next;
            }
            if (!valid) continue;
            const uint32_t mm_field = 4 + scr[j].mm_len, ml_field = t.has_ml ? 8 + scr[j].ml_n : 0;
            uint8_t *mm = t.ml_first ? w + ml_field : w, *ml = t.ml_first ? w : w + mm_field;
            mm[0] = 'M'; mm[1] = 'M'; mm[2] = 'Z'; mm[3 + scr[j].mm_len] = 0;
            if (t.has_ml) {
                ml[0] = 'M'; ml[1] = 'L'; ml[2] = 'B'; ml[3] = 'C';
                for (int k = 0; k < 4; ++k) ml[4 + k] = (uint8_t)(scr[j].ml_n >> (8 * k));
            }
            uint8_t *mn = w + mm_field + ml_field;
            mn[0] = 'M'; mn[1] = 'N'; mn[2] = 'I';
            for (int k = 0; k < 4; ++k) mn[3 + k] = (uint8_t)(n >> (8 * k));
            scr[j].mm_at = (uint32_t)(mm + 3 - dst);
            scr[j].ml_at = (uint32_t)(ml + 8 - dst);
        }
        if (!valid || lane) continue;
        uint64_t ml_group = 0, calls;                                    // the group's first ML value
        for (uint32_t p = 0; p < t.mm_len;) {                            // group by group, the children in order
            uint32_t head, codes;
            int b;
            fl_mm_head(t.mm, t.mm_len, p, &head, &b, &codes);
            FlMMCursor cur = fl_mm_cursor(p + head);
            for (unsigned long long j = i; j < j_end; ++j) {
                uint8_t *dst = out + off[j];
                uint32_t at = scr[j].mm_at;
                for (uint32_t k = 0; k < head; ++k) dst[at++] = t.mm[p + k];
                const uint64_t bs = b == 4 ? (uint64_t)items[j].s : scr[j].before[b], be = b == 4 ? (uint64_t)items[j].e : scr[j].before[4 + b];
                uint64_t k0, k1;
                at += fl_mm_rebase(t.mm, t.mm_len, cur, bs, be, dst + at, &k0, &k1);
                dst[at++] = ';';
                scr[j].mm_at = at;
                if (!t.has_ml) continue;
                uint32_t mat = scr[j].ml_at;
                for (uint64_t k = ml_group + k0 * codes; k < ml_group + k1 * codes; ++k) dst[mat++] = t.ml[k];
                scr[j].ml_at = mat;
            }
            p = fl_mm_group_end(t.mm, cur, &calls);
            ml_group += calls * codes;
        }
    }
}

}  // namespace

namespace {

// fl_reads_push_bam and fl_reads_push_bam_strand; what: the entry point's name, for its messages
int push_bam(fl_ctx *c, const char *what, const char *chunk, uint64_t n_bytes, uint64_t n_rec, const uint32_t *seq_off,
             const uint32_t *qual_off, const int32_t *len, const uint8_t *reverse) {
    const std::string fn(what);
    if ((!chunk && n_bytes) || (n_rec && (!chunk || !seq_off || !qual_off || !len))) {
        c->set_error(fn + ": bad arguments");
        return FL_EINVAL;
    }
    if (n_bytes >= ((uint64_t)1 << 31)) { c->set_error(fn + ": a chunk must be smaller than 2 GiB"); return FL_ERANGE; }
    if (n_rec > 0xFFFFFFF0ull) { c->set_error(fn + ": too many records in one chunk"); return FL_ERANGE; }
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
            c->set_error(fn + ": record " + std::to_string(i) + " does not lie inside the chunk");
            return FL_EINVAL;
        }
        off[i] = padded_bases;
        padded_bases += (L + FL_ALIGN_BASES - 1) & ~(uint64_t)(FL_ALIGN_BASES - 1);
        bases += (int64_t)L;
    }
    // stage: chunk + SEQ / QUAL offsets + reverse flags in one byte buffer, lengths and offsets in the slot's own arrays
    // (copy stream, double buffered like fl_reads_push)
    const int slot = c->stg_next;
    c->stg_next ^= 1;
    fl_ctx::Staging &S = c->stg[slot];
    if (!S.consumed) FL_CUDA(c, cudaEventCreateWithFlags(&S.consumed, cudaEventDisableTiming));
    if (S.in_use) FL_CUDA(c, cudaEventSynchronize(S.consumed));
    S.in_use = false;
    cudaStream_t st = c->stream, cs = c->copy_stream;
    const size_t chunk_room = ((size_t)n_bytes + 64 + 15) & ~(size_t)15;
    FL_CUDA(c, S.ascii.reserve(chunk_room + 8 * n + (reverse ? n : 0), 0, cs));
    FL_CUDA(c, S.off.reserve(n + 1, 0, cs));
    FL_CUDA(c, S.len.reserve(n, 0, cs));
    uint32_t *d_seq_off = reinterpret_cast<uint32_t *>(S.ascii.p + chunk_room), *d_qual_off = d_seq_off + n;
    FL_CUDA(c, cudaMemcpyAsync(S.ascii.p, chunk, (size_t)n_bytes, cudaMemcpyHostToDevice, cs));
    FL_CUDA(c, cudaMemcpyAsync(d_seq_off, seq_off, n * sizeof(uint32_t), cudaMemcpyHostToDevice, cs));
    FL_CUDA(c, cudaMemcpyAsync(d_qual_off, qual_off, n * sizeof(uint32_t), cudaMemcpyHostToDevice, cs));
    uint8_t *d_reverse = nullptr;
    if (reverse) {
        d_reverse = reinterpret_cast<uint8_t *>(d_qual_off + n);
        FL_CUDA(c, cudaMemcpyAsync(d_reverse, reverse, n, cudaMemcpyHostToDevice, cs));
    }
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
        k_bam_gather<false><<<ggrid, 256, 0, st>>>(S.ascii.p, n_bytes, (uint32_t)n, d_seq_off, d_qual_off, S.len.p, d_reverse, d_off, S.seq.p, nullptr);
        v.seq2b = S.seq.p;
        c->launches++;
    }
    if (!kmer_mode) {
        FL_CUDA(c, S.qual.reserve((size_t)padded_bases + 64, 0, st));
        k_bam_gather<true><<<ggrid, 256, 0, st>>>(S.ascii.p, n_bytes, (uint32_t)n, d_seq_off, d_qual_off, S.len.p, d_reverse, d_off, nullptr, S.qual.p);
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

}  // namespace

extern "C" int fl_reads_push_bam(fl_ctx *c, const char *chunk, uint64_t n_bytes, uint64_t n_rec, const uint32_t *seq_off,
                                 const uint32_t *qual_off, const int32_t *len) {
    FL_ENTER(c);
    return push_bam(c, "fl_reads_push_bam", chunk, n_bytes, n_rec, seq_off, qual_off, len, nullptr);
}

extern "C" int fl_reads_push_bam_strand(fl_ctx *c, const char *chunk, uint64_t n_bytes, uint64_t n_rec, const uint32_t *seq_off,
                                        const uint32_t *qual_off, const int32_t *len, const uint8_t *reverse) {
    FL_ENTER(c);
    return push_bam(c, "fl_reads_push_bam_strand", chunk, n_bytes, n_rec, seq_off, qual_off, len, reverse);
}

// ---- BAM output (fl_bam_build, fl_bam_writer) ----

struct BamBuildBufs {
    DevVec<uint8_t> batch, status;
    DevVec<fl_bam_item> items;
    DevVec<BamItemScratch> scr;
    DevVec<unsigned long long> size, off, misc;
};

namespace {

// The two passes over device buffers. The records go to grow->p + at (grown to hold them, its first `at` bytes kept)
// when grow is given, else to out[0, cap). name_of: the record at a batch offset's read name, for the message of a name
// that does not fit (nullptr: the item is named by its index).
int bam_build_run(fl_ctx *c, BamBuildBufs &b, const uint8_t *d_batch, uint64_t n_bytes, const fl_bam_item *d_items, uint64_t n_items,
                  int keep_mods, DevVec<uint8_t> *grow, uint64_t at, uint8_t *out, uint64_t cap, uint64_t *n_out, uint64_t counts[2],
                  const fl_bam_item *h_items, const char *h_batch) {
    cudaStream_t st = c->stream;
    const size_t n = (size_t)n_items;
    FL_CUDA(c, b.scr.reserve(n + 1, 0, st));
    FL_CUDA(c, b.status.reserve(n + 1, 0, st));
    FL_CUDA(c, b.size.reserve(n + 1, 0, st));
    FL_CUDA(c, b.off.reserve(n + 1, 0, st));
    FL_CUDA(c, b.misc.reserve(BM_N, 0, st));
    FL_CUDA(c, cudaMemsetAsync(b.misc.p, 0, BM_N * sizeof(unsigned long long), st));
    FL_CUDA(c, cudaMemsetAsync(b.misc.p + BM_BAD, 0xFF, 2 * sizeof(unsigned long long), st));
    unsigned grid = fl_blocks(n * 32, 256);
    if (grid > (unsigned)c->sm_count * 16) grid = (unsigned)c->sm_count * 16;
    if (grid == 0) grid = 1;
    {
        KernelTimer kt(c, FL_KERNEL_BAM_BUILD);
        k_bam_build<false><<<grid, 256, 0, st>>>(d_batch, n_bytes, d_items, n_items, keep_mods, b.scr.p, b.status.p, b.size.p, nullptr,
                                                 nullptr, b.misc.p);
        c->launches++;
    }
    FL_CUDA(c, cudaGetLastError());
    FL_TRY(fl_exclusive_scan_u64(c, b.size.p, b.off.p, n, b.misc.p + BM_TOTAL));
    unsigned long long misc[BM_N];
    FL_CUDA(c, cudaMemcpyAsync(misc, b.misc.p, sizeof misc, cudaMemcpyDeviceToHost, st));
    FL_CUDA(c, cudaStreamSynchronize(st));
    if (misc[BM_BAD] != ~0ull) {
        c->set_error("fl_bam_build: item " + std::to_string(misc[BM_BAD]) + " does not lie inside the batch");
        return FL_EINVAL;
    }
    if (misc[BM_LONG] != ~0ull) {
        std::string what = "item " + std::to_string(misc[BM_LONG]);
        if (h_items && h_batch) {
            const fl_bam_item &it = h_items[misc[BM_LONG]];
            const char *name = h_batch + it.off + 36;
            what = std::string(name) + "_" + std::to_string(it.s + 1) + "-" + std::to_string(it.e);
        }
        c->set_error("the name of child read " + what + " is too long for a BAM record");
        return FL_EINVAL;
    }
    const uint64_t total = misc[BM_TOTAL];
    *n_out = total;
    if (grow) {
        FL_CUDA(c, grow->reserve((size_t)(at + total + 16), (size_t)at, st));
        out = grow->p + at;
    } else if (total > cap) {
        c->set_error("fl_bam_build: the output buffer holds " + std::to_string(cap) + " bytes, " + std::to_string(total) + " are needed");
        return FL_ERANGE;
    }
    {
        KernelTimer kt(c, FL_KERNEL_BAM_BUILD);
        k_bam_build<true><<<grid, 256, 0, st>>>(d_batch, n_bytes, d_items, n_items, keep_mods, b.scr.p, b.status.p, b.size.p, b.off.p, out,
                                                b.misc.p);
        c->launches++;
    }
    FL_CUDA(c, cudaGetLastError());
    if (counts) { counts[0] += misc[BM_KEPT]; counts[1] += misc[BM_INVALID]; }
    return FL_OK;
}

// copies the host batch and items to the device (the batch readable 16 bytes past its end)
int bam_stage(fl_ctx *c, BamBuildBufs &b, const void *host_batch, uint64_t n_bytes, const fl_bam_item *items, uint64_t n_items) {
    cudaStream_t st = c->stream;
    FL_CUDA(c, b.batch.reserve((size_t)n_bytes + 16, 0, st));
    FL_CUDA(c, b.items.reserve((size_t)n_items + 1, 0, st));
    if (n_bytes) FL_CUDA(c, cudaMemcpyAsync(b.batch.p, host_batch, (size_t)n_bytes, cudaMemcpyHostToDevice, st));
    if (n_items) FL_CUDA(c, cudaMemcpyAsync(b.items.p, items, (size_t)n_items * sizeof(fl_bam_item), cudaMemcpyHostToDevice, st));
    return FL_OK;
}

}  // namespace

extern "C" int fl_bam_build_device(fl_ctx *c, const void *dev_batch, uint64_t n_bytes, const fl_bam_item *dev_items, uint64_t n_items,
                                   int keep_mods, void *dev_out, uint64_t cap, uint64_t *n_out, uint64_t counts[2]) {
    FL_ENTER(c);
    if ((!dev_batch && n_bytes) || (!dev_items && n_items) || !n_out || (!dev_out && cap)) {
        c->set_error("fl_bam_build_device: bad arguments");
        return FL_EINVAL;
    }
    BamBuildBufs b;
    FL_TRY(bam_build_run(c, b, static_cast<const uint8_t *>(dev_batch), n_bytes, dev_items, n_items, keep_mods, nullptr, 0,
                         static_cast<uint8_t *>(dev_out), cap, n_out, counts, nullptr, nullptr));
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    return FL_OK;
}

extern "C" int fl_bam_build(fl_ctx *c, const void *host_batch, uint64_t n_bytes, const fl_bam_item *items, uint64_t n_items, int keep_mods,
                            void *host_out, uint64_t cap, uint64_t *n_out, uint64_t counts[2]) {
    FL_ENTER(c);
    if ((!host_batch && n_bytes) || (!items && n_items) || !n_out || (!host_out && cap)) {
        c->set_error("fl_bam_build: bad arguments");
        return FL_EINVAL;
    }
    BamBuildBufs b;
    DevVec<uint8_t> out;
    FL_TRY(bam_stage(c, b, host_batch, n_bytes, items, n_items));
    FL_TRY(bam_build_run(c, b, b.batch.p, n_bytes, b.items.p, n_items, keep_mods, &out, 0, nullptr, 0, n_out, counts, items,
                         static_cast<const char *>(host_batch)));
    if (*n_out > cap) {
        c->set_error("fl_bam_build: the output buffer holds " + std::to_string(cap) + " bytes, " + std::to_string(*n_out) + " are needed");
        return FL_ERANGE;
    }
    if (*n_out) FL_CUDA(c, cudaMemcpyAsync(host_out, out.p, (size_t)*n_out, cudaMemcpyDeviceToHost, c->stream));
    FL_CUDA(c, cudaStreamSynchronize(c->stream));
    return FL_OK;
}

struct fl_bam_writer {
    fl_ctx *c;
    BamBuildBufs b;
    DevVec<uint8_t> stream, zout;      // the bytes held back, then the batch's records; the members of the whole blocks
    uint64_t held = 0;
};

extern "C" int fl_bam_writer_create(fl_ctx *c, fl_bam_writer **out) {
    FL_ENTER(c);
    if (!out) { c->set_error("fl_bam_writer_create: NULL out"); return FL_EINVAL; }
    *out = new fl_bam_writer{c, {}, {}, {}, 0};
    return FL_OK;
}

extern "C" int fl_bam_writer_push(fl_bam_writer *w, const void *host_batch, uint64_t n_bytes, const fl_bam_item *items, uint64_t n_items,
                                  int keep_mods, int last, void *host_out, uint64_t cap, uint64_t *n_out, uint64_t counts[2]) {
    if (!w) return FL_EINVAL;
    fl_ctx *c = w->c;
    FL_ENTER(c);
    if ((!host_batch && n_bytes) || (!items && n_items) || !n_out || (!host_out && cap)) {
        c->set_error("fl_bam_writer_push: bad arguments");
        return FL_EINVAL;
    }
    cudaStream_t st = c->stream;
    uint64_t built = 0;
    FL_TRY(bam_stage(c, w->b, host_batch, n_bytes, items, n_items));
    FL_TRY(bam_build_run(c, w->b, w->b.batch.p, n_bytes, w->b.items.p, n_items, keep_mods, &w->stream, w->held, nullptr, 0, &built, counts,
                         items, static_cast<const char *>(host_batch)));
    const uint64_t total = w->held + built, whole = last ? total : total / FL_BGZF_BLOCK * FL_BGZF_BLOCK;
    FL_CUDA(c, w->zout.reserve((size_t)fl_bgzf_bound(whole), 0, st));
    FL_TRY(fl_bgzf_compress_device(c, w->stream.p, whole, w->zout.p, fl_bgzf_bound(whole), 0, n_out));
    if (*n_out > cap) {
        c->set_error("fl_bam_writer_push: the output buffer holds " + std::to_string(cap) + " bytes, " + std::to_string(*n_out) + " are needed");
        return FL_ERANGE;
    }
    if (*n_out) FL_CUDA(c, cudaMemcpyAsync(host_out, w->zout.p, (size_t)*n_out, cudaMemcpyDeviceToHost, st));
    w->held = total - whole;                                             // < FL_BGZF_BLOCK: nothing to move when whole == 0,
    if (w->held && whole)                                                // else FL_BGZF_BLOCK <= whole: the ranges do not overlap
        FL_CUDA(c, cudaMemcpyAsync(w->stream.p, w->stream.p + whole, (size_t)w->held, cudaMemcpyDeviceToDevice, st));
    FL_CUDA(c, cudaStreamSynchronize(st));
    return FL_OK;
}

extern "C" void fl_bam_writer_destroy(fl_bam_writer *w) {
    if (!w) return;
    cudaSetDevice(w->c->device);
    delete w;
}

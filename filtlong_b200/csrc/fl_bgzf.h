// filtlong_b200/csrc/fl_bgzf.h -- the parts of the BGZF compressor (fl_bgzf.cu) that are plain arithmetic, written
// once for the host and the device so that a CPU test pins what the kernel computes:
//   * length-limited Huffman code lengths and canonical (bit-reversed, as deflate sends them) codes, RFC 1951 3.2.2;
//   * CRC-32 (the gzip trailer's, polynomial 0xEDB88320) of one piece, and the GF(2) shift that combines the CRCs of
//     consecutive pieces, so that every thread of a block checksums its own slice.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

#define FL_BGZF_MAX_BITS 15        // literal/length and distance codes
#define FL_BGZF_MAX_CL_BITS 7      // the code-length code

// Code lengths for m symbols whose weights w[0..m) are sorted ascending (all > 0). On return w[i] is the length of the
// i-th symbol of that order; no length exceeds maxbits. m == 1 gives length 1. Kraft sum is exactly 1 for m >= 2.
// 2^maxbits must be >= m.
//
// First the unrestricted Huffman code, computed in place on the sorted weights (Moffat and Katajainen, "In-place
// calculation of minimum-redundancy codes", 1995): a left-to-right pass pairs the two lightest of {leaves, internal
// nodes} and stores parent links, a right-to-left pass turns the links into internal depths, a last pass hands the
// leaf depths out level by level. If the longest length exceeds maxbits the lengths are clamped and the Kraft excess
// is removed by lengthening the least frequent symbols, then any slack is given back to the most frequent ones.
__host__ __device__ inline void fl_huff_lengths_sorted(uint32_t *w, int m, int maxbits) {
    if (m <= 0) return;
    if (m == 1) { w[0] = 1; return; }
    int root = 0, leaf = 2, next;
    w[0] += w[1];
    for (next = 1; next < m - 1; ++next) {
        if (leaf >= m || w[root] < w[leaf]) { w[next] = w[root]; w[root++] = (uint32_t)next; }
        else w[next] = w[leaf++];
        if (leaf >= m || (root < next && w[root] < w[leaf])) { w[next] += w[root]; w[root++] = (uint32_t)next; }
        else w[next] += w[leaf++];
    }
    w[m - 2] = 0;
    for (next = m - 3; next >= 0; --next) w[next] = w[w[next]] + 1;
    int avail = 1, used = 0, depth = 0;
    root = m - 2;
    next = m - 1;
    while (avail > 0) {
        while (root >= 0 && (int)w[root] == depth) { ++used; --root; }
        while (avail > used) { w[next--] = (uint32_t)depth; --avail; }
        avail = 2 * used;
        ++depth;
        used = 0;
    }
    // w[0] (the lightest symbol) has the longest length
    if ((int)w[0] <= maxbits) return;
    const uint32_t full = 1u << maxbits;
    uint32_t kraft = 0;
    for (int i = 0; i < m; ++i) {
        if ((int)w[i] > maxbits) w[i] = (uint32_t)maxbits;
        kraft += full >> w[i];
    }
    for (int i = 0; kraft > full; i = (i + 1) % m)     // lengthen the lightest symbols first
        if ((int)w[i] < maxbits) { kraft -= full >> (w[i] + 1); ++w[i]; }
    for (bool changed = true; changed && kraft < full;) {   // give slack back, heaviest symbols first
        changed = false;
        for (int i = m - 1; i >= 0 && kraft < full; --i)
            if (w[i] > 1 && kraft + (full >> w[i]) <= full) { kraft += full >> w[i]; --w[i]; changed = true; }
    }
}

// Canonical codes (RFC 1951 3.2.2) for lengths len[0..n), returned bit-reversed in code[] because deflate packs
// Huffman codes starting from their most significant bit into an LSB-first stream. bl / next_code: maxbits + 2 entries.
__host__ __device__ inline void fl_huff_canonical(const uint8_t *len, int n, int maxbits, uint16_t *code, uint32_t *bl,
                                                  uint32_t *next_code) {
    for (int b = 0; b <= maxbits + 1; ++b) bl[b] = 0;
    for (int i = 0; i < n; ++i) bl[len[i]]++;
    bl[0] = 0;
    uint32_t c = 0;
    for (int b = 1; b <= maxbits + 1; ++b) { c = (c + bl[b - 1]) << 1; next_code[b] = c; }
    for (int i = 0; i < n; ++i) {
        const int L = len[i];
        if (!L) { code[i] = 0; continue; }
        uint32_t v = next_code[L]++, r = 0;
        for (int k = 0; k < L; ++k) { r = (r << 1) | (v & 1u); v >>= 1; }
        code[i] = (uint16_t)r;
    }
}

// ---- CRC-32 ----------------------------------------------------------------------------------------------------------
// Polynomials are kept reflected, as the table-driven CRC uses them: bit 31 is x^0.
#define FL_CRC32_POLY 0xEDB88320u

__host__ __device__ inline uint32_t fl_crc32_table_entry(uint32_t b) {
    uint32_t r = b;
    for (int k = 0; k < 8; ++k) r = (r & 1u) ? (r >> 1) ^ FL_CRC32_POLY : r >> 1;
    return r;
}

// a * b mod P
__host__ __device__ inline uint32_t fl_gf2_mulmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int k = 0; k < 32; ++k) {
        if (a & (0x80000000u >> k)) p ^= b;
        b = (b & 1u) ? (b >> 1) ^ FL_CRC32_POLY : b >> 1;    // b * x
    }
    return p;
}

// x^(8 n) mod P: what a CRC register is multiplied by when n zero bytes follow
__host__ __device__ inline uint32_t fl_crc32_shift(uint64_t n) {
    uint32_t r = 0x80000000u, sq = 0x00800000u;   // x^0, x^8
    for (; n; n >>= 1) {
        if (n & 1u) r = fl_gf2_mulmod(r, sq);
        sq = fl_gf2_mulmod(sq, sq);
    }
    return r;
}

// The gzip CRC of a message from the XOR of its pieces' raw CRCs (register started at 0, no final inversion), each
// already multiplied by fl_crc32_shift(bytes after the piece): the initial 0xFFFFFFFF travels through all n bytes.
__host__ __device__ inline uint32_t fl_crc32_finish(uint32_t raw_xor, uint64_t n) {
    return ~(raw_xor ^ fl_gf2_mulmod(0xFFFFFFFFu, fl_crc32_shift(n)));
}

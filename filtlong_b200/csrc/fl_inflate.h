// filtlong_b200/csrc/fl_inflate.h -- the parts of the parallel gzip inflater (fl_inflate.cu) that are plain arithmetic,
// written once for the host and the device so that a CPU test (tests/inflate_dump.cpp) runs the very same code:
//   * a bounded LSB-first bit reader: a read past the end of the compressed buffer sets an error, it never loads;
//   * canonical Huffman decode tables (RFC 1951 3.2.2) built with zlib's checks (over-subscribed and incomplete codes);
//   * the block-start test the finder runs at every bit offset (dynamic header, stored block, gzip member header);
//   * the speculative decoder: stored, fixed and dynamic blocks, gzip member headers and trailers, with 16-bit output
//     symbols -- a byte, or a marker for a byte of the unknown 32 KiB before the chunk;
//   * the round / chain / repair orchestration (host only), a template over the backend that runs the steps: the
//     device (fl_inflate.cu) or a serial CPU model.
// The two-stage scheme is the one of pugz (Kerbiriou and Chikhi, 2019) and rapidgzip (Knespel and Brunst, 2023).
#pragma once
#include <stdint.h>

#include "fl_bgzf.h"   // CRC-32 shift / finish

#define FL_INF_WINDOW 32768u
#define FL_INF_MARKER 256u            // symbol 256 + w: byte w of the 32 KiB window before the chunk
#define FL_INF_MAXEV 64u              // member starts / ends one chunk may record
#define FL_INF_LIT_LUT 9              // look-up bits of the literal/length table (longer codes: canonical walk)
#define FL_INF_DIST_LUT 8

// where a chunk starts or stops
#define FL_INF_BLOCK 0                // a deflate block header
#define FL_INF_HEADER 1               // a gzip member header (byte aligned)
#define FL_INF_END 2                  // the end of the input: no member follows
// chunk flags: any one means "this start is false" (or, for a confirmed chunk, that the data cannot be inflated here)
#define FL_INF_EBAD 1u                // invalid data: bad code, bad header, distance too far back, read past the end
#define FL_INF_EFULL 2u               // the output slot is full
#define FL_INF_EEVENTS 4u             // more member starts / ends than FL_INF_MAXEV

#ifndef __CUDACC__
#define __host__
#define __device__
#endif
#define FL_INF_HD __host__ __device__ inline

// ---- bounded bit reader -------------------------------------------------------------------------------------------
struct FlBits {
    const uint8_t *p;
    uint64_t n;                       // bytes in p
    uint64_t next;                    // next byte to load
    uint64_t buf;
    uint32_t cnt;                     // valid bits in buf
    bool err;
    FL_INF_HD void refill() {
        while (cnt <= 56 && next < n) { buf |= (uint64_t)p[next++] << cnt; cnt += 8; }
    }
    FL_INF_HD void seek(uint64_t bit) {
        next = bit >> 3; buf = 0; cnt = 0;
        if (next > n) { next = n; err = true; return; }
        refill();
        consume((uint32_t)(bit & 7u));
    }
    FL_INF_HD void init(const uint8_t *in, uint64_t nbytes, uint64_t bit) { p = in; n = nbytes; err = false; seek(bit); }
    FL_INF_HD uint64_t pos() const { return next * 8 - cnt; }
    FL_INF_HD uint32_t peek(uint32_t k) {           // k <= 32; bits past the end read as 0 (consume() catches them)
        if (cnt < k) refill();
        return (uint32_t)(buf & ((1ull << k) - 1ull));
    }
    FL_INF_HD void consume(uint32_t k) {
        if (k > cnt) { err = true; buf = 0; cnt = 0; return; }
        buf >>= k; cnt -= k;
    }
    FL_INF_HD uint32_t bits(uint32_t k) { const uint32_t v = peek(k); consume(k); return v; }
};

// ---- canonical Huffman tables ---------------------------------------------------------------------------------------
// zlib's inflate_table rules: over-subscribed is an error; incomplete is an error for the code-length code, and for the
// literal/length and distance codes unless the code is a single code of length 1. No code at all is accepted (a symbol
// decoded from it is then invalid).
#define FL_HUFF_CODES 0
#define FL_HUFF_LENS 1
#define FL_HUFF_DISTS 2

template <int LB, int NS>
struct FlHuff {
    uint16_t count[16];
    uint16_t sym[NS];
    uint16_t lut[1 << LB];            // (symbol << 4) | length for codes of <= LB bits, 0: longer (or no) code
};

// lengths only: 0 if they form a code zlib accepts
FL_INF_HD int fl_huff_check(const uint8_t *len, int n, int type, uint16_t *count) {
    for (int b = 0; b < 16; ++b) count[b] = 0;
    for (int i = 0; i < n; ++i) count[len[i]]++;
    int max = 15;
    while (max >= 1 && count[max] == 0) --max;
    if (max == 0) return 0;
    int left = 1;
    for (int b = 1; b < 16; ++b) {
        left <<= 1;
        left -= count[b];
        if (left < 0) return -1;                                   // over-subscribed
    }
    if (left > 0 && (type == FL_HUFF_CODES || max != 1)) return -1; // incomplete
    return 0;
}

template <int LB, int NS>
FL_INF_HD int fl_huff_build(FlHuff<LB, NS> *h, const uint8_t *len, int n, int type) {
    if (fl_huff_check(len, n, type, h->count)) return -1;
    uint16_t offs[16];
    offs[1] = 0;
    for (int b = 1; b < 15; ++b) offs[b + 1] = (uint16_t)(offs[b] + h->count[b]);
    for (int i = 0; i < n; ++i)
        if (len[i]) h->sym[offs[len[i]]++] = (uint16_t)i;
    for (int i = 0; i < (1 << LB); ++i) h->lut[i] = 0;
    uint32_t code = 0;
    int k = 0;
    for (int b = 1; b <= LB; ++b) {
        for (int j = 0; j < h->count[b]; ++j, ++k, ++code) {
            uint32_t r = 0, v = code;
            for (int q = 0; q < b; ++q) { r = (r << 1) | (v & 1u); v >>= 1; }
            const uint16_t e = (uint16_t)((h->sym[k] << 4) | b);
            for (uint32_t f = r; f < (1u << LB); f += 1u << b) h->lut[f] = e;
        }
        code <<= 1;
    }
    return 0;
}

// one symbol, or -1 (no such code, or past the end of the input)
template <int LB, int NS>
FL_INF_HD int fl_huff_decode(const FlHuff<LB, NS> *h, FlBits &br) {
    const uint32_t v = br.peek(15);
    const uint16_t e = h->lut[v & ((1u << LB) - 1u)];
    if (e) {
        br.consume(e & 15u);
        return br.err ? -1 : (int)(e >> 4);
    }
    int code = 0, first = 0, index = 0;                            // the canonical walk (RFC 1951 3.2.2), MSB first
    for (int b = 1; b < 16; ++b) {
        code |= (int)((v >> (b - 1)) & 1u);
        const int c = h->count[b];
        if (code - first < c) {
            br.consume((uint32_t)b);
            return br.err ? -1 : (int)h->sym[index + code - first];
        }
        index += c;
        first += c;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

typedef FlHuff<FL_INF_LIT_LUT, 288> FlLitTab;
typedef FlHuff<FL_INF_DIST_LUT, 32> FlDistTab;
typedef FlHuff<7, 19> FlClTab;

// per-decoder scratch: the tables of the current block and the code lengths of a dynamic header
struct FlInfTables {
    FlLitTab lit;
    FlDistTab dist;
    FlClTab cl;
    uint8_t lens[320];
};

FL_INF_HD uint32_t fl_inf_clen_order(int i) {
    // RFC 1951 3.2.7: the order the code-length code lengths are sent in
    const uint8_t o[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    return o[i];
}

// A dynamic block header after BFINAL / BTYPE (RFC 1951 3.2.7), with every check zlib makes. build_lut == false: only
// validate (what the finder does at every bit offset). 0: valid.
FL_INF_HD int fl_inf_dyn_header(FlBits &br, FlInfTables *t, bool build_lut) {
    const uint32_t hlit = br.bits(5) + 257, hdist = br.bits(5) + 1, hclen = br.bits(4) + 4;
    if (br.err || hlit > 286 || hdist > 30) return -1;
    uint8_t cl[19];
    for (int i = 0; i < 19; ++i) cl[i] = 0;
    for (uint32_t i = 0; i < hclen; ++i) cl[fl_inf_clen_order((int)i)] = (uint8_t)br.bits(3);
    if (br.err || fl_huff_build(&t->cl, cl, 19, FL_HUFF_CODES)) return -1;
    const uint32_t total = hlit + hdist;
    uint32_t i = 0;
    while (i < total) {
        const int s = fl_huff_decode(&t->cl, br);
        if (s < 0) return -1;
        if (s < 16) { t->lens[i++] = (uint8_t)s; continue; }
        uint32_t rep;
        uint8_t v = 0;
        if (s == 16) {
            if (i == 0) return -1;                                 // repeat with nothing before
            v = t->lens[i - 1];
            rep = 3 + br.bits(2);
        } else if (s == 17) {
            rep = 3 + br.bits(3);
        } else {
            rep = 11 + br.bits(7);
        }
        if (br.err || i + rep > total) return -1;
        while (rep--) t->lens[i++] = v;
    }
    if (t->lens[256] == 0) return -1;                              // no end-of-block code
    if (!build_lut) {
        uint16_t count[16];
        // The finder asks for complete literal/length and distance codes. zlib's encoder always sends them (it gives
        // every tree at least two codes); the one-code and no-code cases the decoder also accepts are what most random
        // bit strings that get this far look like. A start missed here is only a chunk merged into the one before.
        if (fl_huff_check(t->lens, (int)hlit, FL_HUFF_CODES, count)) return -1;
        if (fl_huff_check(t->lens + hlit, (int)hdist, FL_HUFF_CODES, count)) return -1;
        return count[0] == hdist ? -1 : 0;
    }
    if (fl_huff_build(&t->lit, t->lens, (int)hlit, FL_HUFF_LENS)) return -1;
    return fl_huff_build(&t->dist, t->lens + hlit, (int)hdist, FL_HUFF_DISTS);
}

FL_INF_HD void fl_inf_fixed_tables(FlInfTables *t) {
    for (int i = 0; i < 144; ++i) t->lens[i] = 8;
    for (int i = 144; i < 256; ++i) t->lens[i] = 9;
    for (int i = 256; i < 280; ++i) t->lens[i] = 7;
    for (int i = 280; i < 288; ++i) t->lens[i] = 8;
    fl_huff_build(&t->lit, t->lens, 288, FL_HUFF_LENS);
    for (int i = 0; i < 32; ++i) t->lens[i] = 5;
    fl_huff_build(&t->dist, t->lens, 32, FL_HUFF_DISTS);
}

// ---- gzip member header (RFC 1952 2.3) --------------------------------------------------------------------------------
FL_INF_HD uint32_t fl_inf_crc_byte(uint32_t crc, uint32_t b) { return fl_crc32_table_entry((crc ^ b) & 0xffu) ^ (crc >> 8); }

// 1f 8b 08 and no reserved flag: what a member header can start with
FL_INF_HD bool fl_inf_header_magic(const uint8_t *d, uint64_t n, uint64_t at) {
    return n - at >= 4 && d[at] == 0x1f && d[at + 1] == 0x8b && d[at + 2] == 8 && (d[at + 3] & 0xe0u) == 0;
}

// Parses a member header at byte `at`; the byte after it, or 0 when the header is invalid or truncated. zlib checks
// FHCRC (the low 16 bits of the header's CRC-32), so this does too.
FL_INF_HD uint64_t fl_inf_member_header(const uint8_t *d, uint64_t n, uint64_t at) {
    if (at > n || n - at < 10 || !fl_inf_header_magic(d, n, at)) return 0;
    const uint32_t flg = d[at + 3];
    uint64_t q = at + 10;
    if (flg & 4u) {
        if (n - q < 2) return 0;
        const uint64_t xlen = (uint64_t)d[q] | ((uint64_t)d[q + 1] << 8);
        q += 2;
        if (n - q < xlen) return 0;
        q += xlen;
    }
    for (uint32_t f = 8; f <= 16; f <<= 1) {                       // FNAME, FCOMMENT: zero-terminated
        if (!(flg & f)) continue;
        while (q < n && d[q]) ++q;
        if (q >= n) return 0;
        ++q;
    }
    if (flg & 2u) {
        if (n - q < 2) return 0;
        uint32_t crc = 0xffffffffu;
        for (uint64_t i = at; i < q; ++i) crc = fl_inf_crc_byte(crc, d[i]);
        crc = ~crc;
        if ((crc & 0xffffu) != ((uint32_t)d[q] | ((uint32_t)d[q + 1] << 8))) return 0;
        q += 2;
    }
    return q;
}

// ---- the block-start test of the finder ---------------------------------------------------------------------------------
// FL_INF_BLOCK / FL_INF_HEADER if bit offset `bit` may start a dynamic or stored block or a gzip member, else -1.
FL_INF_HD int fl_inf_candidate(const uint8_t *d, uint64_t n, uint64_t bit, FlInfTables *t) {
    if ((bit & 7u) == 0 && fl_inf_header_magic(d, n, bit >> 3)) return FL_INF_HEADER;
    FlBits br;
    br.init(d, n, bit);
    const uint32_t h = br.bits(3);
    if (br.err) return -1;
    const uint32_t type = h >> 1;
    if (type == 0) {
        const uint64_t q = (bit + 3 + 7) >> 3;
        if (q > n || n - q < 4) return -1;
        const uint32_t len = (uint32_t)d[q] | ((uint32_t)d[q + 1] << 8), nlen = (uint32_t)d[q + 2] | ((uint32_t)d[q + 3] << 8);
        return (len ^ 0xffffu) == nlen && n - q - 4 >= len ? FL_INF_BLOCK : -1;
    }
    if (type != 2) return -1;
    return fl_inf_dyn_header(br, t, false) == 0 ? FL_INF_BLOCK : -1;
}

// ---- the speculative decoder -------------------------------------------------------------------------------------------
struct FlInfEvent {
    uint64_t pos;                     // output symbol index in the chunk
    uint32_t crc, isize;              // a member's end: its trailer
    uint32_t end;                     // 0: a member starts at pos, 1: a member ends at pos
    uint32_t pad;
};

struct FlInfChunk {
    uint64_t start_bit, stop_at;      // in: where to start, and the bit from which a block boundary ends the chunk
    uint32_t start_kind;              // in
    uint32_t flags;                   // out: FL_INF_E*
    uint64_t stop_bit;                // out: where it stopped
    uint32_t stop_kind;               // out
    uint32_t n_ev;                    // out: events recorded
    uint64_t out_len;                 // out: symbols written
};

// Decodes the chunk c from c->start_bit into slot[0, cap) (16-bit symbols) and ev[0, FL_INF_MAXEV). It stops at the first
// block or member boundary at or past c->stop_at, or at the end of the input; any invalid input sets a flag and stops.
// Reads only d[0, n) and writes only slot[0, cap), ev[0, FL_INF_MAXEV), whatever the bytes are.
struct FlInfNoBlock {
    FL_INF_HD void operator()(uint64_t, uint32_t) const {}
};

// on_block(bit, btype) is called at every block header decoded (btype 0-2) and member header parsed (btype 4): what the
// CPU test compares the finder with.
template <typename SlotPtr, typename OnBlock = FlInfNoBlock>
FL_INF_HD void fl_inf_decode(const uint8_t *d, uint64_t n, FlInfChunk *c, SlotPtr slot, uint64_t cap, FlInfEvent *ev,
                             FlInfTables *t, OnBlock on_block = OnBlock()) {
    FlBits br;
    br.init(d, n, c->start_bit);
    uint64_t o = 0;
    int64_t from = -1;                // output index where the current member began in this chunk, -1: before the chunk
    uint32_t nev = 0, flags = 0, kind = c->start_kind;
    if (br.err) flags |= FL_INF_EBAD;
    while (!flags) {
        const uint64_t at = br.pos();
        if (kind == FL_INF_END) break;
        if (kind == FL_INF_HEADER) {
            const uint64_t b = at >> 3;
            if (n - b < 2 || d[b] != 0x1f || d[b + 1] != 0x8b) { kind = FL_INF_END; break; }   // the end, or ignored trailing bytes
            if (at >= c->stop_at) break;
            const uint64_t q = fl_inf_member_header(d, n, b);
            if (!q) { flags |= FL_INF_EBAD; break; }
            on_block(at, 4);
            if (nev == FL_INF_MAXEV) { flags |= FL_INF_EEVENTS; break; }
            ev[nev].pos = o; ev[nev].crc = 0; ev[nev].isize = 0; ev[nev].end = 0; ev[nev].pad = 0; ++nev;
            from = (int64_t)o;
            br.seek(q * 8);
            kind = FL_INF_BLOCK;
            continue;
        }
        if (at >= c->stop_at) break;
        const uint32_t h = br.bits(3);
        const uint32_t type = h >> 1;
        if (br.err || type == 3) { flags |= FL_INF_EBAD; break; }
        on_block(at, type);
        if (type == 0) {
            const uint64_t q = (br.pos() + 7) >> 3;
            if (q > n || n - q < 4) { flags |= FL_INF_EBAD; break; }
            const uint32_t len = (uint32_t)d[q] | ((uint32_t)d[q + 1] << 8), nlen = (uint32_t)d[q + 2] | ((uint32_t)d[q + 3] << 8);
            if ((len ^ 0xffffu) != nlen || n - q - 4 < len) { flags |= FL_INF_EBAD; break; }
            if (cap - o < len) { flags |= FL_INF_EFULL; break; }
            for (uint32_t i = 0; i < len; ++i) slot[o + i] = d[q + 4 + i];
            o += len;
            br.seek((q + 4 + len) * 8);
        } else {
            if (type == 1) fl_inf_fixed_tables(t);
            else if (fl_inf_dyn_header(br, t, true)) { flags |= FL_INF_EBAD; break; }
            for (;;) {
                const int s = fl_huff_decode(&t->lit, br);
                if (s < 0) { flags |= FL_INF_EBAD; break; }
                if (s < 256) {
                    if (o == cap) { flags |= FL_INF_EFULL; break; }
                    slot[o++] = (uint16_t)s;
                    continue;
                }
                if (s == 256) break;
                const uint32_t ls = (uint32_t)s - 257;
                if (ls >= 29) { flags |= FL_INF_EBAD; break; }
                uint32_t L;
                if (ls < 8) L = 3 + ls;
                else if (ls == 28) L = 258;
                else { const uint32_t e = (ls >> 2) - 1; L = 3 + (((4u | (ls & 3u)) << e)) + br.bits(e); }
                const int ds = fl_huff_decode(&t->dist, br);
                if (ds < 0 || ds >= 30) { flags |= FL_INF_EBAD; break; }
                uint32_t D;
                if (ds < 4) D = 1 + (uint32_t)ds;
                else { const uint32_t e = ((uint32_t)ds >> 1) - 1; D = 1 + ((2u | ((uint32_t)ds & 1u)) << e) + br.bits(e); }
                if (br.err) { flags |= FL_INF_EBAD; break; }
                const int64_t src = (int64_t)o - (int64_t)D;
                if (from >= 0 && src < from) { flags |= FL_INF_EBAD; break; }   // before the member's first byte
                if (cap - o < L) { flags |= FL_INF_EFULL; break; }
                for (uint32_t i = 0; i < L; ++i) {
                    const int64_t s2 = src + (int64_t)i;
                    slot[o + i] = s2 >= 0 ? (uint16_t)slot[(uint64_t)s2] : (uint16_t)(FL_INF_MARKER + FL_INF_WINDOW + s2);
                }
                o += L;
            }
            if (flags) break;
        }
        if (h & 1u) {                                              // the member's last block: its trailer
            const uint64_t q = (br.pos() + 7) >> 3;
            if (q > n || n - q < 8) { flags |= FL_INF_EBAD; break; }
            if (nev == FL_INF_MAXEV) { flags |= FL_INF_EEVENTS; break; }
            ev[nev].pos = o;
            ev[nev].crc = (uint32_t)d[q] | ((uint32_t)d[q + 1] << 8) | ((uint32_t)d[q + 2] << 16) | ((uint32_t)d[q + 3] << 24);
            ev[nev].isize = (uint32_t)d[q + 4] | ((uint32_t)d[q + 5] << 8) | ((uint32_t)d[q + 6] << 16) | ((uint32_t)d[q + 7] << 24);
            ev[nev].end = 1; ev[nev].pad = 0; ++nev;
            br.seek((q + 8) * 8);
            kind = FL_INF_HEADER;
        }
    }
    c->flags = flags;
    c->stop_bit = br.pos();
    c->stop_kind = kind;
    c->n_ev = nev;
    c->out_len = o;
}

// one resolved byte of a chunk: a symbol, or its window byte (window = the 32 KiB before the chunk's output)
FL_INF_HD uint8_t fl_inf_resolve(uint16_t s, const uint8_t *window) {
    return s < FL_INF_MARKER ? (uint8_t)s : window[s - FL_INF_MARKER];
}

// ---- orchestration (host) ---------------------------------------------------------------------------------------------
#include <algorithm>
#include <vector>

#define FL_INF_MAX_REPAIRS 64         // repair passes before a round declines

struct FlInfStats { uint64_t members, chunks, redecoded, rounds; };

// output symbols a chunk's slot holds for `chunk_bytes` of compressed input
inline uint64_t fl_inf_slot_cap(uint64_t chunk_bytes) { return chunk_bytes * 8 + (128u << 10); }
// device bytes per chunk of a round: slot, output, window, chunk record, events, CRC segments
inline uint64_t fl_inf_chunk_bytes_needed(uint64_t chunk_bytes) {
    return fl_inf_slot_cap(chunk_bytes) * 3 + FL_INF_WINDOW + sizeof(FlInfChunk) + FL_INF_MAXEV * sizeof(FlInfEvent) +
           FL_INF_MAXEV * 20 + 64;
}
// chunks a round should hold to keep an H100's decoders busy (132 SMs x 64 decoding threads)
#define FL_INF_FILL 8192u
// Chunk size the library picks: enough chunks to fill an H100's decoders, no fewer than 32 KiB of input each, and small
// enough that a round in `avail` device bytes still holds FL_INF_FILL chunks (a large file then takes more rounds,
// each of them with every decoder busy, rather than fewer rounds of a few long chunks).
inline uint64_t fl_inf_default_chunk(uint64_t n, uint64_t avail) {
    uint64_t c = n / FL_INF_FILL;
    c = c < (32u << 10) ? (32u << 10) : c > (4u << 20) ? (4u << 20) : c;
    c = (c + 4095) & ~4095ull;
    const uint64_t room = avail > n + 4096 ? avail - n - 4096 : 0;
    while (c > (32u << 10) && room / fl_inf_chunk_bytes_needed(c) < FL_INF_FILL) c = ((c / 2) + 4095) & ~4095ull;
    return c < (32u << 10) ? (32u << 10) : c;
}

// The whole procedure over a gzip file of n bytes. B (the backend) runs the steps over round state it holds:
//   int upload() (1, 0: no memory, -1: failed), uint64_t free_bytes(), bool alloc(R, cap) (false: no memory), bool find(m, lo, hi, bit, kind),
//   bool decode(chunk_records, K, idx, m), bool events(K, ev), bool resolve(chunk_records, K, off, win_lo, total, &bad),
//   bool crc(nseg, lo, hi, raw), bool fetch(total, dst). resolve() gets the final chunk records: the chain check may have
//   changed some without a decode.
// Returns 1 (inflated: out[0, *n_out)), 0 (declined) or -1 (the backend failed: B::error()).
// head: the input's first two bytes, on the host (the input itself may be device memory). out: where fetch() writes.
template <class B>
int fl_inf_run(B &be, const uint8_t *head, uint64_t n, uint8_t *out, uint64_t cap, uint64_t chunk_bytes, uint64_t max_dev,
               uint64_t *n_out, FlInfStats *st) {
    *st = FlInfStats{0, 0, 0, 0};
    *n_out = 0;
    if (n < 18 || head[0] != 0x1f || head[1] != 0x8b) return 0;
    uint64_t avail = be.free_bytes();
    if (max_dev && max_dev < avail) avail = max_dev;
    if (!chunk_bytes) chunk_bytes = fl_inf_default_chunk(n, avail);
    const uint64_t slot_cap = fl_inf_slot_cap(chunk_bytes), per = fl_inf_chunk_bytes_needed(chunk_bytes);
    if (avail <= n + 4096 + per) return 0;
    const uint64_t R_max = (avail - n - 4096) / per;
    const int up = be.upload();                                    // 0: no memory for the input (decline), -1: failure
    if (up <= 0) return up;

    uint64_t pos_bit = 0, pos_out = 0;
    uint32_t pos_kind = FL_INF_HEADER;
    bool open = false;                // inside a member at pos_out
    uint64_t mem_start = 0, mem_len = 0;
    uint32_t mem_raw = 0;
    std::vector<FlInfChunk> ch;
    std::vector<FlInfEvent> ev;
    std::vector<uint64_t> lo, hi, fbit, off, seg_lo, seg_hi;
    std::vector<uint32_t> fkind, win_lo, idx, raw, seg_end;   // seg_end: event index + 1 of the member end a segment closes, 0: none
    std::vector<uint8_t> bad;
    while (pos_kind != FL_INF_END) {
        // ---- chunks of this round: a known start, then nominal starts every chunk_bytes ----
        const uint64_t base = pos_bit >> 3;
        const uint64_t left = n > base ? n - base : 0;
        uint64_t R = (left + chunk_bytes - 1) / chunk_bytes;
        if (R < 1) R = 1;
        if (R > R_max) R = R_max;
        const uint64_t end_byte = base + R * chunk_bytes;
        const uint64_t round_stop = end_byte >= n ? ~0ull : end_byte * 8;
        const uint32_t m = (uint32_t)(R - 1);
        lo.resize(m); hi.resize(m); fbit.assign(m, 0); fkind.assign(m, 0);
        for (uint32_t j = 0; j < m; ++j) {
            lo[j] = (base + (j + 1) * chunk_bytes) * 8;
            hi[j] = std::min<uint64_t>(base + (j + 2) * chunk_bytes, n) * 8;
        }
        if (!be.alloc(R, slot_cap)) return 0;                     // no device memory for the round: decline
        if (m && !be.find(m, lo.data(), hi.data(), fbit.data(), fkind.data())) return -1;
        ch.clear();
        FlInfChunk c0{};
        c0.start_bit = pos_bit; c0.start_kind = pos_kind;
        ch.push_back(c0);
        for (uint32_t j = 0; j < m; ++j)
            if ((int32_t)fkind[j] >= 0) {                          // no candidate: the chunk merges into the one before
                FlInfChunk c{};
                c.start_bit = fbit[j]; c.start_kind = fkind[j];
                ch.push_back(c);
            }
        const uint32_t K = (uint32_t)ch.size();
        for (uint32_t k = 0; k + 1 < K; ++k) ch[k].stop_at = ch[k + 1].start_bit;
        ch[K - 1].stop_at = round_stop;
        st->chunks += K;
        st->rounds += 1;
        idx.resize(K);
        for (uint32_t k = 0; k < K; ++k) idx[k] = k;
        if (!be.decode(ch.data(), K, idx.data(), K)) return -1;
        // ---- chain check and repair ----
        for (int rep = 0;; ++rep) {
            // A chunk is judged only behind a predecessor that starts where its own predecessor stopped: the stop of
            // such a chunk is almost always right, so breaks that are not next to each other are repaired in one pass.
            // A chunk behind a chunk being re-decoded waits for the next pass.
            idx.clear();
            bool prev_linked = true;
            for (uint32_t k = 1; k < K; ++k) {
                const FlInfChunk &p = ch[k - 1];
                const bool p_redone = !idx.empty() && idx.back() == k - 1;
                const bool linked = !p.flags && !p_redone && p.stop_bit == ch[k].start_bit && p.stop_kind == ch[k].start_kind;
                if (p.flags || p_redone || !prev_linked || linked) { prev_linked = linked; continue; }
                prev_linked = true;
                if (p.stop_kind == FL_INF_END || p.stop_bit >= ch[k].stop_at) {
                    // what decoding from there gives, without a look: nothing, stopping where it starts
                    FlInfChunk &c = ch[k];
                    c.start_bit = c.stop_bit = p.stop_bit;
                    c.start_kind = c.stop_kind = p.stop_kind;
                    c.flags = 0; c.n_ev = 0; c.out_len = 0;
                    continue;
                }
                ch[k].start_bit = p.stop_bit;
                ch[k].start_kind = p.stop_kind;
                idx.push_back(k);
                prev_linked = false;
            }
            if (idx.empty()) break;
            if (rep == FL_INF_MAX_REPAIRS) return 0;
            st->redecoded += idx.size();
            if (!be.decode(ch.data(), K, idx.data(), (uint32_t)idx.size())) return -1;
        }
        for (uint32_t k = 0; k < K; ++k)
            if (ch[k].flags) return 0;                            // a confirmed chunk that cannot be decoded
        // ---- members, windows, CRC segments ----
        ev.resize((size_t)K * FL_INF_MAXEV);
        if (!be.events(K, ev.data())) return -1;
        off.resize(K); win_lo.resize(K);
        seg_lo.clear(); seg_hi.clear(); seg_end.clear();
        uint64_t total = 0;
        uint64_t piece = pos_out;                                 // start of the open member's piece in this round
        for (uint32_t k = 0; k < K; ++k) {
            off[k] = total;
            const uint64_t g = pos_out + total;
            if (open) {
                const int64_t w0 = (int64_t)g - (int64_t)FL_INF_WINDOW;
                const int64_t lo_ok = (int64_t)mem_start - w0;
                win_lo[k] = (uint32_t)std::max<int64_t>(0, std::min<int64_t>(lo_ok, FL_INF_WINDOW));
            } else {
                win_lo[k] = FL_INF_WINDOW;                         // starts at a member header: no marker can be valid
            }
            for (uint32_t e = 0; e < ch[k].n_ev; ++e) {
                const FlInfEvent &x = ev[(size_t)k * FL_INF_MAXEV + e];
                const uint64_t at = g + x.pos;
                if (!x.end) {
                    if (open) return 0;
                    open = true; mem_start = at; piece = at; mem_len = 0; mem_raw = 0;
                    st->members += 1;
                } else {
                    if (!open) return 0;
                    seg_lo.push_back(piece - pos_out); seg_hi.push_back(at - pos_out);
                    seg_end.push_back(k * FL_INF_MAXEV + e + 1);
                    open = false;
                }
            }
            total += ch[k].out_len;
        }
        if (open) { seg_lo.push_back(piece - pos_out); seg_hi.push_back(total); seg_end.push_back(0); }
        if (pos_out + total > cap) return 0;
        uint8_t bad_marker = 0;
        if (!be.resolve(ch.data(), K, off.data(), win_lo.data(), total, &bad_marker)) return -1;
        if (bad_marker) return 0;                                 // a back-reference before its member's start
        raw.assign(seg_lo.size(), 0);
        if (!seg_lo.empty() && !be.crc((uint32_t)seg_lo.size(), seg_lo.data(), seg_hi.data(), raw.data())) return -1;
        for (size_t s = 0; s < seg_lo.size(); ++s) {
            const uint64_t len = seg_hi[s] - seg_lo[s];
            mem_raw = fl_gf2_mulmod(mem_raw, fl_crc32_shift(len)) ^ raw[s];
            mem_len += len;
            if (seg_end[s]) {
                const FlInfEvent &x = ev[seg_end[s] - 1];
                if (fl_crc32_finish(mem_raw, mem_len) != x.crc || (uint32_t)mem_len != x.isize) return 0;
                mem_raw = 0; mem_len = 0;
            }
        }
        if (total && !be.fetch(total, out + pos_out)) return -1;
        pos_out += total;
        pos_bit = ch[K - 1].stop_bit;
        pos_kind = ch[K - 1].stop_kind;
        if (pos_kind != FL_INF_END && pos_bit == (base << 3) && total == 0 && K == 1) return 0;   // no progress
    }
    if (open || pos_out == 0) return 0;
    *n_out = pos_out;
    return 1;
}

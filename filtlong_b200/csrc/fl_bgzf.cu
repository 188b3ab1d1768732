// filtlong_b200/csrc/fl_bgzf.cu -- BGZF (gzip members of at most 64 KiB with a 'BC' extra field, SAM specification
// section 4.1) compression on the device: what `| gzip` did at the end of the reference README's command lines.
//
// One CTA per 65,280-byte block (bgzip's block size), 512 threads, everything in shared memory:
//   1. candidates: positions are hashed four bytes at a time, 512 consecutive positions per step. A position's candidate
//      is the latest earlier lane of its warp with the same hash (__match_any_sync), else the latest position of an
//      earlier step (a hash table of positions updated with atomicMax after each step, so its content does not depend
//      on the order of the atomics), if the four bytes really agree and the distance is at most 32 KiB;
//   2. parse: thread t greedily parses bytes [128 t, 128 t + 128). A match is cut at the segment's end, or becomes a
//      literal when fewer than 3 bytes are left. The tokens overwrite the candidates in place (distance at the match's
//      first position, length at its second); the symbol histogram is counted; each thread also takes the CRC-32 of
//      its segment, shifted to the block's end (fl_bgzf.h), and the block's CRC is the XOR of those;
//   3. code: length-limited Huffman codes for literal/length and distance symbols and for the code lengths
//      (fl_bgzf.h), a dynamic-block header, the bit length of every thread's tokens and a block-wide scan of them;
//   4. emit: the member goes to a 64 KiB slot in global memory, every thread writing its own bits at its offset (words it
//      shares with a neighbour by atomicOr). A stored block is written instead when it is not larger.
// Then the member sizes are scanned and the members packed back to back into the caller's buffer.
#include "fl_internal.cuh"
#include "fl_bgzf.h"

namespace {

constexpr int BZ_THREADS = 512;
constexpr uint32_t BZ_SEG = 128;                     // bytes parsed by one thread: 512 x 128 >= 65,280
constexpr uint32_t BZ_BLOCK = FL_BGZF_BLOCK;
constexpr uint32_t BZ_SLOT = 65536;                  // bytes per member slot; a member never exceeds 65,311
constexpr uint32_t BZ_HASH_BITS = 13;
constexpr uint32_t BZ_WINDOW = 32768;
constexpr uint32_t BZ_HDR = 18;                      // gzip header with the 6-byte BC extra field
constexpr uint32_t BZ_STORED_MAX = BZ_HDR + 5 + BZ_BLOCK + 8;
constexpr int BZ_CHUNK_BLOCKS = 2048;                // blocks per launch: 128 MiB of member slots
static_assert(BZ_THREADS * BZ_SEG >= BZ_BLOCK, "segments must cover a block");
static_assert(BZ_STORED_MAX <= BZ_SLOT, "a stored member must fit a slot");

// shared memory: the block (zero-padded), one uint16 per position (candidate distance, then the parse), the hash table
constexpr uint32_t SM_IN = 0;
constexpr uint32_t SM_CAND = 65536;
constexpr uint32_t SM_TAB = SM_CAND + 2 * BZ_BLOCK;
constexpr uint32_t SM_BYTES = SM_TAB + (4u << BZ_HASH_BITS);

// what follows the candidate phase lives where the hash table was
struct Work {
    uint32_t crc_tab[256];
    uint32_t lhist[286], dhist[30], clhist[19];
    uint32_t lw[286], dw[30], clw[19];        // weights in ascending order, then code lengths in that order
    uint16_t lorder[286], dorder[30], clorder[19];
    uint8_t llen[288], dlen[32], cllen[20];
    uint16_t lcode[286], dcode[30], clcode[19];
    uint16_t rle[320];                        // code-length symbols of the header: symbol | extra bits << 5
    uint32_t bl[3][FL_BGZF_MAX_BITS + 2], nc[3][FL_BGZF_MAX_BITS + 2];
    uint32_t n_rle, n_lit_used, n_dist_used, hlit, hdist, hclen, hdr_bits;
    uint32_t warp_sum[BZ_THREADS / 32];
    uint32_t crc_part[BZ_THREADS / 32];
};
static_assert(sizeof(Work) <= (4u << BZ_HASH_BITS), "work area must fit the hash table's place");

__constant__ uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ uint32_t load4(const uint32_t *w, uint32_t p) {
    return __funnelshift_r(w[p >> 2], w[(p >> 2) + 1], (p & 3u) * 8u);
}

// bytes a and b agree for, up to lim (the block is zero-padded, lim keeps the result inside it)
__device__ __forceinline__ uint32_t match_len(const uint32_t *w, uint32_t a, uint32_t b, uint32_t lim) {
    uint32_t k = 0;
    while (k < lim) {
        const uint32_t x = load4(w, a + k) ^ load4(w, b + k);
        if (x) { k += (uint32_t)(__ffs(x) - 1) >> 3; break; }
        k += 4;
    }
    return k < lim ? k : lim;
}

// RFC 1951 3.2.5: length 3..258 -> symbol 257 + code, distance 1..32768 -> code, with their extra bits
__device__ __forceinline__ void len_sym(uint32_t L, uint32_t &code, uint32_t &ebits, uint32_t &eval) {
    const uint32_t x = L - 3;
    if (L == 258) { code = 28; ebits = 0; eval = 0; }
    else if (x < 8) { code = x; ebits = 0; eval = 0; }
    else {
        const uint32_t e = 29u - __clz(x);
        code = 4 * e + 4 + ((x >> e) & 3u); ebits = e; eval = x & ((1u << e) - 1u);
    }
}
__device__ __forceinline__ void dist_sym(uint32_t d, uint32_t &code, uint32_t &ebits, uint32_t &eval) {
    const uint32_t y = d - 1;
    if (y < 4) { code = y; ebits = 0; eval = 0; }
    else {
        const uint32_t k = 31u - __clz(y), e = k - 1;
        code = 2 * k + ((y >> e) & 1u); ebits = e; eval = y & ((1u << e) - 1u);
    }
}

// LSB-first bit writer into a zeroed member slot starting at bit `pos`. Words other threads may also touch (the first
// and the last) are combined with atomicOr; every word in between belongs to this thread alone.
struct BitOut {
    uint32_t *w;
    unsigned long long acc;
    uint32_t nb, word;
    bool first;
    __device__ BitOut(uint32_t *slot, uint32_t pos) : w(slot), acc(0), nb(pos & 31u), word(pos >> 5), first(true) {}
    __device__ __forceinline__ void put(uint32_t v, uint32_t n) {
        acc |= (unsigned long long)v << nb;
        nb += n;
        if (nb >= 32) {
            if (first) { atomicOr(w + word, (uint32_t)acc); first = false; }
            else w[word] = (uint32_t)acc;
            ++word;
            acc >>= 32;
            nb -= 32;
        }
    }
    __device__ __forceinline__ void finish() { if (nb) atomicOr(w + word, (uint32_t)acc); }
};

// ascending (frequency, symbol) order of the used symbols of h[0..ns), one thread per symbol
__device__ __forceinline__ void rank_symbol(const uint32_t *h, int ns, int sym, uint16_t *order, uint32_t *wts) {
    const uint32_t f = h[sym];
    if (!f) return;
    uint32_t r = 0;
    for (int j = 0; j < ns; ++j) {
        const uint32_t g = h[j];
        r += (g != 0) & ((g < f) | ((g == f) & (j < sym)));
    }
    order[r] = (uint16_t)sym;
    wts[r] = f;
}

__global__ void __launch_bounds__(BZ_THREADS, 1) k_bgzf_deflate(const uint8_t *__restrict__ in, unsigned long long n,
                                                               unsigned long long first_block, uint8_t *__restrict__ slots,
                                                               uint32_t *__restrict__ sizes) {
    extern __shared__ __align__(16) unsigned char sm[];
    uint8_t *IN = sm + SM_IN;
    const uint32_t *IN32 = reinterpret_cast<const uint32_t *>(IN);
    uint16_t *CAND = reinterpret_cast<uint16_t *>(sm + SM_CAND);
    uint32_t *TAB = reinterpret_cast<uint32_t *>(sm + SM_TAB);
    Work &W = *reinterpret_cast<Work *>(sm + SM_TAB);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const unsigned long long start = (first_block + blockIdx.x) * (unsigned long long)BZ_BLOCK;
    const uint32_t len = (uint32_t)(n - start < BZ_BLOCK ? n - start : BZ_BLOCK);
    uint8_t *slot = slots + (size_t)blockIdx.x * BZ_SLOT;
    uint32_t *slot32 = reinterpret_cast<uint32_t *>(slot);

    // ---- load the block, clear the hash table and the slot ----
    const uint8_t *src = in + start;
    if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
        const uint32_t nv = len >> 4;
        for (uint32_t i = tid; i < nv; i += BZ_THREADS) reinterpret_cast<uint4 *>(IN)[i] = __ldg(reinterpret_cast<const uint4 *>(src) + i);
        for (uint32_t i = (nv << 4) + tid; i < len; i += BZ_THREADS) IN[i] = src[i];
    } else {
        for (uint32_t i = tid; i < len; i += BZ_THREADS) IN[i] = src[i];
    }
    for (uint32_t i = len + tid; i < len + 16; i += BZ_THREADS) IN[i] = 0;
    for (uint32_t i = tid; i < (1u << BZ_HASH_BITS); i += BZ_THREADS) TAB[i] = 0;
    for (uint32_t i = tid; i < BZ_SLOT / 16; i += BZ_THREADS) reinterpret_cast<uint4 *>(slot)[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();

    // ---- 1. match candidates ----
    for (uint32_t base = 0; base < len; base += BZ_THREADS) {
        const uint32_t p = base + tid;
        const bool valid = p + 4 <= len;
        uint32_t x = 0, h = 0x10000u + lane;                       // never equal to a real hash
        if (valid) { x = load4(IN32, p); h = (x * 0x9E3779B1u) >> (32 - BZ_HASH_BITS); }
        const unsigned before = __match_any_sync(0xffffffffu, h) & ((1u << lane) - 1u);
        uint32_t d = 0;
        if (valid) {
            if (before) {
                const uint32_t q = base + (tid & ~31u) + (31u - __clz(before));
                if (load4(IN32, q) == x) d = p - q;
            }
            if (!d) {
                const uint32_t t = TAB[h];
                if (t && p - (t - 1) <= BZ_WINDOW && load4(IN32, t - 1) == x) d = p - (t - 1);
            }
        }
        if (p < len) CAND[p] = (uint16_t)d;
        __syncthreads();
        if (valid) atomicMax(&TAB[h], p + 1);
        __syncthreads();
    }

    // ---- 2. parse, histogram, CRC ----
    for (uint32_t i = tid; i < 256; i += BZ_THREADS) W.crc_tab[i] = fl_crc32_table_entry(i);
    for (uint32_t i = tid; i < 286; i += BZ_THREADS) W.lhist[i] = 0;
    if (tid < 30) W.dhist[tid] = 0;
    if (tid < 19) W.clhist[tid] = 0;
    __syncthreads();
    if (tid == 0) W.lhist[256] = 1;                                // end of block
    const uint32_t s = tid * BZ_SEG < len ? tid * BZ_SEG : len;
    const uint32_t e = s + BZ_SEG < len ? s + BZ_SEG : len;
    uint32_t crc = 0;
    for (uint32_t i = s; i < e; ++i) crc = W.crc_tab[(crc ^ IN[i]) & 0xffu] ^ (crc >> 8);
    if (s < e) crc = fl_gf2_mulmod(crc, fl_crc32_shift(len - e));
    for (uint32_t p = s; p < e;) {
        const uint32_t d = CAND[p];
        uint32_t L = 0;
        if (d && e - p >= 3) L = match_len(IN32, p - d, p, e - p < 258 ? e - p : 258);
        if (L >= 3) {
            uint32_t c, eb, ev;
            CAND[p + 1] = (uint16_t)L;
            len_sym(L, c, eb, ev);
            atomicAdd(&W.lhist[257 + c], 1u);
            dist_sym(d, c, eb, ev);
            atomicAdd(&W.dhist[c], 1u);
            p += L;
        } else {
            CAND[p] = 0;
            atomicAdd(&W.lhist[IN[p]], 1u);
            ++p;
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, o);
    if (lane == 0) W.crc_part[wid] = crc;
    __syncthreads();

    // ---- 3. codes ----
    if (tid < 64) {   // warp 0: literal/length symbols, warp 1: distances. Fewer than two used symbols: dummies up to two
        const bool lit = tid < 32;
        uint32_t *H = lit ? W.lhist : W.dhist;
        const int ns = lit ? 286 : 30;
        int cnt = 0, first = -1;
        for (int j0 = 0; j0 < ns; j0 += 32) {
            const int j = j0 + (int)lane;
            const unsigned b = __ballot_sync(0xffffffffu, j < ns && H[j] != 0);
            if (first < 0 && b) first = j0 + __ffs(b) - 1;
            cnt += __popc(b);
        }
        if (lane == 0) {
            if (cnt == 0) { H[0] = 1; H[1] = 1; }
            else if (cnt == 1) H[first == 0 ? 1 : 0] = 1;
            (lit ? W.n_lit_used : W.n_dist_used) = cnt < 2 ? 2u : (uint32_t)cnt;
        }
    }
    for (uint32_t i = tid; i < 288; i += BZ_THREADS) W.llen[i] = 0;
    if (tid < 32) W.dlen[tid] = 0;
    __syncthreads();
    if (tid < 286) rank_symbol(W.lhist, 286, (int)tid, W.lorder, W.lw);
    else if (tid < 286 + 30) rank_symbol(W.dhist, 30, (int)tid - 286, W.dorder, W.dw);
    __syncthreads();
    if (tid == 0) {
        fl_huff_lengths_sorted(W.lw, (int)W.n_lit_used, FL_BGZF_MAX_BITS);
        for (uint32_t i = 0; i < W.n_lit_used; ++i) W.llen[W.lorder[i]] = (uint8_t)W.lw[i];
    } else if (tid == 32) {
        fl_huff_lengths_sorted(W.dw, (int)W.n_dist_used, FL_BGZF_MAX_BITS);
        for (uint32_t i = 0; i < W.n_dist_used; ++i) W.dlen[W.dorder[i]] = (uint8_t)W.dw[i];
    }
    __syncthreads();
    if (tid == 0) {
        // the header: HLIT / HDIST, the run-length coded code lengths (RFC 1951 3.2.7) and their own code
        uint32_t hlit = 286, hdist = 30;
        while (hlit > 257 && !W.llen[hlit - 1]) --hlit;
        while (hdist > 1 && !W.dlen[hdist - 1]) --hdist;
        const uint32_t total = hlit + hdist;
        uint32_t nr = 0;
        for (uint32_t i = 0; i < total;) {
            const uint32_t v = i < hlit ? W.llen[i] : W.dlen[i - hlit];
            uint32_t run = 1;
            while (i + run < total && (i + run < hlit ? W.llen[i + run] : W.dlen[i + run - hlit]) == v) ++run;
            i += run;
            if (v == 0) {
                while (run >= 11) { const uint32_t k = run < 138 ? run : 138; W.rle[nr++] = (uint16_t)(18 | ((k - 11) << 5)); run -= k; }
                if (run >= 3) { W.rle[nr++] = (uint16_t)(17 | ((run - 3) << 5)); run = 0; }
                while (run) { W.rle[nr++] = 0; --run; }
            } else {
                W.rle[nr++] = (uint16_t)v;
                --run;
                while (run >= 3) { const uint32_t k = run < 6 ? run : 6; W.rle[nr++] = (uint16_t)(16 | ((k - 3) << 5)); run -= k; }
                while (run) { W.rle[nr++] = (uint16_t)v; --run; }
            }
        }
        for (uint32_t i = 0; i < nr; ++i) W.clhist[W.rle[i] & 31u]++;
        uint32_t used = 0;
        for (int i = 0; i < 19; ++i) used += W.clhist[i] != 0;
        if (used < 2) { for (int i = 0; i < 19 && used < 2; ++i) if (!W.clhist[i]) { W.clhist[i] = 1; ++used; } }
        uint32_t m = 0;
        for (int i = 0; i < 19; ++i) {            // insertion sort by (frequency, symbol)
            if (!W.clhist[i]) continue;
            int j = (int)m++;
            while (j > 0 && W.clw[j - 1] > W.clhist[i]) { W.clw[j] = W.clw[j - 1]; W.clorder[j] = W.clorder[j - 1]; --j; }
            W.clw[j] = W.clhist[i];
            W.clorder[j] = (uint16_t)i;
        }
        fl_huff_lengths_sorted(W.clw, (int)m, FL_BGZF_MAX_CL_BITS);
        for (int i = 0; i < 20; ++i) W.cllen[i] = 0;
        for (uint32_t i = 0; i < m; ++i) W.cllen[W.clorder[i]] = (uint8_t)W.clw[i];
        fl_huff_canonical(W.cllen, 19, FL_BGZF_MAX_CL_BITS, W.clcode, W.bl[2], W.nc[2]);
        uint32_t hclen = 19;
        while (hclen > 4 && !W.cllen[c_clen_order[hclen - 1]]) --hclen;
        uint32_t bits = 5 + 5 + 4 + 3 * hclen;
        for (uint32_t i = 0; i < nr; ++i) {
            const uint32_t sym = W.rle[i] & 31u;
            bits += W.cllen[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
        }
        W.n_rle = nr; W.hlit = hlit; W.hdist = hdist; W.hclen = hclen; W.hdr_bits = bits;
    } else if (tid == 32) {
        fl_huff_canonical(W.llen, 286, FL_BGZF_MAX_BITS, W.lcode, W.bl[0], W.nc[0]);
    } else if (tid == 64) {
        fl_huff_canonical(W.dlen, 30, FL_BGZF_MAX_BITS, W.dcode, W.bl[1], W.nc[1]);
    }
    __syncthreads();

    // ---- bit length of every thread's tokens, block-wide scan ----
    uint32_t mybits = 0;
    for (uint32_t p = s; p < e;) {
        const uint32_t d = CAND[p];
        if (!d) { mybits += W.llen[IN[p]]; ++p; continue; }
        const uint32_t L = CAND[p + 1];
        uint32_t c, eb, ev;
        len_sym(L, c, eb, ev);
        mybits += W.llen[257 + c] + eb;
        dist_sym(d, c, eb, ev);
        mybits += W.dlen[c] + eb;
        p += L;
    }
    if (tid == BZ_THREADS - 1) mybits += W.llen[256];
    uint32_t incl = mybits;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += v;
    }
    if (lane == 31) W.warp_sum[wid] = incl;
    __syncthreads();
    uint32_t before_warp = 0, all = 0;
    for (uint32_t k = 0; k < BZ_THREADS / 32; ++k) {
        if (k < wid) before_warp += W.warp_sum[k];
        all += W.warp_sum[k];
    }
    const uint32_t tok0 = BZ_HDR * 8 + 3 + W.hdr_bits;             // first token bit in the member
    const uint32_t dyn_bytes = (tok0 + all + 7) / 8 + 8;
    const bool stored = dyn_bytes >= BZ_HDR + 5 + len + 8;
    const uint32_t member = stored ? BZ_HDR + 5 + len + 8 : dyn_bytes;
    const uint32_t trailer = member - 8;

    // ---- 4. emit ----
    if (stored) {
        for (uint32_t i = tid; i < len; i += BZ_THREADS) slot[BZ_HDR + 5 + i] = IN[i];
    } else {
        BitOut bo(slot32, tok0 + before_warp + incl - mybits);
        for (uint32_t p = s; p < e;) {
            const uint32_t d = CAND[p];
            if (!d) { const uint32_t b = IN[p]; bo.put(W.lcode[b], W.llen[b]); ++p; continue; }
            const uint32_t L = CAND[p + 1];
            uint32_t c, eb, ev;
            len_sym(L, c, eb, ev);
            bo.put(W.lcode[257 + c], W.llen[257 + c]);
            if (eb) bo.put(ev, eb);
            dist_sym(d, c, eb, ev);
            bo.put(W.dcode[c], W.dlen[c]);
            if (eb) bo.put(ev, eb);
            p += L;
        }
        if (tid == BZ_THREADS - 1) bo.put(W.lcode[256], W.llen[256]);
        bo.finish();
    }
    if (tid == 0) {
        const uint8_t hdr[BZ_HDR] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0,
                                     (uint8_t)((member - 1) & 0xffu), (uint8_t)((member - 1) >> 8)};
        BitOut bo(slot32, 0);
        for (uint32_t i = 0; i < BZ_HDR; ++i) bo.put(hdr[i], 8);
        if (stored) {
            bo.put(1, 3);                                          // BFINAL, BTYPE 00, then pad to the byte
            bo.put(0, 5);
            bo.put(len & 0xffffu, 16);
            bo.put(~len & 0xffffu, 16);
        } else {
            bo.put(1 | (2 << 1), 3);                               // BFINAL, BTYPE 10
            bo.put(W.hlit - 257, 5);
            bo.put(W.hdist - 1, 5);
            bo.put(W.hclen - 4, 4);
            for (uint32_t i = 0; i < W.hclen; ++i) bo.put(W.cllen[c_clen_order[i]], 3);
            for (uint32_t i = 0; i < W.n_rle; ++i) {
                const uint32_t sym = W.rle[i] & 31u, x = W.rle[i] >> 5;
                bo.put(W.clcode[sym], W.cllen[sym]);
                if (sym == 16) bo.put(x, 2);
                else if (sym == 17) bo.put(x, 3);
                else if (sym == 18) bo.put(x, 7);
            }
        }
        bo.finish();
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t c = 0;
        for (uint32_t k = 0; k < BZ_THREADS / 32; ++k) c ^= W.crc_part[k];
        c = fl_crc32_finish(c, len);
        for (int i = 0; i < 4; ++i) { slot[trailer + i] = (uint8_t)(c >> (8 * i)); slot[trailer + 4 + i] = (uint8_t)(len >> (8 * i)); }
        sizes[blockIdx.x] = member;
    }
}

// exclusive scan of up to 2 x 1024 member sizes on top of the running output size state[0]; state[0] += total
__global__ void __launch_bounds__(1024) k_bgzf_offsets(const uint32_t *__restrict__ sizes, uint32_t m,
                                                      unsigned long long *__restrict__ offs, unsigned long long *state) {
    __shared__ unsigned long long warp_sums[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const uint32_t a = 2 * tid < m ? sizes[2 * tid] : 0u, b = 2 * tid + 1 < m ? sizes[2 * tid + 1] : 0u;
    unsigned long long v = (unsigned long long)a + b, incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += t;
    }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    unsigned long long pre = state[0], all = 0;
    for (uint32_t k = 0; k < 32; ++k) {
        if (k < wid) pre += warp_sums[k];
        all += warp_sums[k];
    }
    pre += incl - v;
    if (2 * tid < m) offs[2 * tid] = pre;
    if (2 * tid + 1 < m) offs[2 * tid + 1] = pre + a;
    __syncthreads();
    if (tid == 0) state[0] += all;
}

// members back to back; state[1] is set when one would end beyond cap (nothing of it is written then)
__global__ void __launch_bounds__(256) k_bgzf_gather(const uint8_t *__restrict__ slots, const uint32_t *__restrict__ sizes,
                                                    const unsigned long long *__restrict__ offs, uint8_t *__restrict__ out,
                                                    unsigned long long cap, unsigned long long *state) {
    const uint32_t size = sizes[blockIdx.x];
    const unsigned long long at = offs[blockIdx.x];
    if (at + size > cap) {
        if (threadIdx.x == 0) state[1] = 1;
        return;
    }
    const uint8_t *src = slots + (size_t)blockIdx.x * BZ_SLOT;
    uint8_t *dst = out + at;
    for (uint32_t i = threadIdx.x; i < size; i += blockDim.x) dst[i] = src[i];
}

// the empty member bgzip ends a file with (SAM specification 4.1.2)
const uint8_t kEof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};

int bgzf_run(fl_ctx *c, const uint8_t *din, uint64_t n, uint8_t *dout, uint64_t cap, int append_eof, uint64_t *n_out) {
    const uint64_t blocks = (n + BZ_BLOCK - 1) / BZ_BLOCK;
    const uint32_t chunk = (uint32_t)(blocks < (uint64_t)BZ_CHUNK_BLOCKS ? blocks : (uint64_t)BZ_CHUNK_BLOCKS);
    cudaStream_t s = c->stream;
    FL_CUDA(c, c->bz_state.reserve(2, 0, s));
    FL_CUDA(c, cudaMemsetAsync(c->bz_state.p, 0, 2 * sizeof(unsigned long long), s));
    if (chunk) {
        FL_CUDA(c, c->bz_slots.reserve((size_t)chunk * BZ_SLOT, 0, s));
        FL_CUDA(c, c->bz_sizes.reserve(chunk, 0, s));
        FL_CUDA(c, c->bz_offs.reserve(chunk, 0, s));
        if (!c->bgzf_attr_set) {
            FL_CUDA(c, cudaFuncSetAttribute(k_bgzf_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SM_BYTES));
            c->bgzf_attr_set = true;
        }
    }
    for (uint64_t b0 = 0; b0 < blocks; b0 += chunk) {
        KernelTimer kt(c, FL_KERNEL_BGZF);
        const uint32_t m = (uint32_t)(blocks - b0 < chunk ? blocks - b0 : chunk);
        k_bgzf_deflate<<<m, BZ_THREADS, SM_BYTES, s>>>(din, n, b0, c->bz_slots.p, c->bz_sizes.p);
        k_bgzf_offsets<<<1, 1024, 0, s>>>(c->bz_sizes.p, m, c->bz_offs.p, c->bz_state.p);
        k_bgzf_gather<<<m, 256, 0, s>>>(c->bz_slots.p, c->bz_sizes.p, c->bz_offs.p, dout, cap, c->bz_state.p);
        c->launches += 3;
        FL_CUDA(c, cudaGetLastError());
    }
    FL_CUDA(c, cudaMemcpyAsync(c->h_scalars + 48, c->bz_state.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    FL_CUDA(c, cudaStreamSynchronize(s));
    const uint64_t total = c->h_scalars[48] + (append_eof ? sizeof kEof : 0);
    *n_out = total;
    if (c->h_scalars[49] || total > cap) {
        c->set_error("fl_bgzf_compress: the output buffer holds " + std::to_string(cap) + " bytes, " + std::to_string(total) + " are needed");
        return FL_ERANGE;
    }
    if (append_eof) {
        FL_CUDA(c, cudaMemcpyAsync(dout + c->h_scalars[48], kEof, sizeof kEof, cudaMemcpyHostToDevice, s));
        FL_CUDA(c, cudaStreamSynchronize(s));
    }
    return FL_OK;
}

}  // namespace

extern "C" uint64_t fl_bgzf_bound(uint64_t n) {
    return (n + BZ_BLOCK - 1) / BZ_BLOCK * (uint64_t)BZ_STORED_MAX + sizeof kEof;
}

extern "C" int fl_bgzf_compress_device(fl_ctx *c, const void *dev_in, uint64_t n, void *dev_out, uint64_t cap, int append_eof,
                                       uint64_t *n_out) {
    FL_ENTER(c);
    if ((!dev_in && n) || !dev_out || !n_out) { c->set_error("fl_bgzf_compress_device: NULL buffer"); return FL_EINVAL; }
    return bgzf_run(c, static_cast<const uint8_t *>(dev_in), n, static_cast<uint8_t *>(dev_out), cap, append_eof, n_out);
}

extern "C" int fl_bgzf_compress(fl_ctx *c, const void *host_in, uint64_t n, void *host_out, uint64_t cap, int append_eof,
                                uint64_t *n_out) {
    FL_ENTER(c);
    if ((!host_in && n) || !host_out || !n_out) { c->set_error("fl_bgzf_compress: NULL buffer"); return FL_EINVAL; }
    cudaStream_t s = c->stream;
    const uint64_t bound = fl_bgzf_bound(n);
    const uint64_t dcap = cap < bound ? cap : bound;
    FL_CUDA(c, c->bz_hin.reserve((size_t)n + 16, 0, s));
    FL_CUDA(c, c->bz_hout.reserve((size_t)dcap + 16, 0, s));
    if (n) FL_CUDA(c, cudaMemcpyAsync(c->bz_hin.p, host_in, (size_t)n, cudaMemcpyHostToDevice, s));
    FL_TRY(bgzf_run(c, c->bz_hin.p, n, c->bz_hout.p, dcap, append_eof, n_out));
    FL_CUDA(c, cudaMemcpyAsync(host_out, c->bz_hout.p, (size_t)*n_out, cudaMemcpyDeviceToHost, s));
    FL_CUDA(c, cudaStreamSynchronize(s));
    return FL_OK;
}

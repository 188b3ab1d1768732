// filtlong_b200/csrc/fl_bam_mods.h -- `--keep_mods`: the base-modification tags (MM / ML / MN, SAMtags 1.7) of an
// unaligned BAM record, checked and re-based to a child [s, e) of the record. Plain arithmetic written once for the host
// (host/bam.cpp, bam_child_record) and the device (fl_bam.cu, k_bam_build), so that the rule exists in one place.
//
// MM:Z is a list of groups B[+-]CODES[.?]?(,delta)*; with B one of ACGTUN and CODES one or more of a-z or one ChEBI
// number. A group's calls are the running positions (delta + 1 each, from -1) among the SEQ bases equal to B: U counts
// T, N counts every base, the strand does not change what is counted. ML:B:C holds one value per call and code, group
// after group. The tags are valid when MM parses exactly so, every delta is an unsigned decimal below 2^32, no group's
// last call lies past the last base it counts, ML (if present) is B:C with exactly that many values, MN (if present) is
// an integer equal to l_seq, and none of the three tags appears twice.
//
// A child keeps every group, with the calls whose SEQ position lies in [s, e): the first kept delta becomes the call's
// index among the B bases less the B bases before s, the later deltas are copied as they are written; ML keeps the kept
// calls' values.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

// size of one value of an aux type ('B' arrays: of one element), 0 for a type that is not one
__host__ __device__ inline int fl_aux_size(uint8_t t) {
    switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    default: return 0;
    }
}

// the aux field at p (tag, type, value) ends at the returned pointer, not after `end`; nullptr if it does not parse
__host__ __device__ inline const uint8_t *fl_aux_next(const uint8_t *p, const uint8_t *end) {
    if (end - p < 3) return nullptr;
    const uint8_t t = p[2];
    p += 3;
    if (t == 'Z' || t == 'H') {
        for (; p < end; ++p)
            if (*p == 0) return p + 1;
        return nullptr;
    }
    if (t == 'B') {
        if (end - p < 5) return nullptr;
        const int s = fl_aux_size(p[0]);
        if (!s || p[0] == 'A') return nullptr;
        const uint64_t n = (uint64_t)p[1] | ((uint64_t)p[2] << 8) | ((uint64_t)p[3] << 16) | ((uint64_t)p[4] << 24);
        if ((uint64_t)(end - p - 5) < n * (uint64_t)s) return nullptr;
        return p + 5 + n * (uint64_t)s;
    }
    const int s = fl_aux_size(t);
    if (!s || end - p < s) return nullptr;
    return p + s;
}

__host__ __device__ inline uint32_t fl_rd32(const uint8_t *p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// The tags of one record's aux fields [aux, end) that a child keeps or checks. end - aux < 2^31 (bam_plan_chunks).
struct FlModTags {
    const uint8_t *rg_first = nullptr;    // RG fields are kept as they are: first one and the bytes of all of them
    uint32_t rg_bytes = 0;
    const uint8_t *mm = nullptr;          // the MM:Z value, without its NUL
    uint32_t mm_len = 0;
    const uint8_t *ml = nullptr;          // the ML:B:C values
    uint32_t ml_n = 0;
    bool has_mm = false, has_ml = false, ml_first = false, bad = false;
};

// Walks the aux fields (already checked to parse up to `end`) once.
__host__ __device__ inline void fl_mod_tags(const uint8_t *aux, const uint8_t *end, int64_t l_seq, FlModTags *t) {
    bool has_mn = false;
    for (const uint8_t *a = aux; a < end;) {
        const uint8_t *next = fl_aux_next(a, end);
        if (!next) { t->bad = true; return; }
        const uint8_t x = a[0], y = a[1], ty = a[2];
        if (x == 'R' && y == 'G') {
            if (!t->rg_first) t->rg_first = a;
            t->rg_bytes += (uint32_t)(next - a);
        } else if (x == 'M' && y == 'M') {
            if (t->has_mm || ty != 'Z') t->bad = true;
            t->has_mm = true;
            t->mm = a + 3;
            t->mm_len = (uint32_t)(next - a - 4);
        } else if (x == 'M' && y == 'L') {
            if (t->has_ml || ty != 'B' || a[3] != 'C') t->bad = true;
            t->ml_first = !t->has_mm;
            t->has_ml = true;
            t->ml = a + 8;
            t->ml_n = (uint32_t)(next - a - 8);
        } else if (x == 'M' && y == 'N') {
            int64_t v = 0;
            switch (ty) {
            case 'c': v = (int8_t)a[3]; break;
            case 'C': v = a[3]; break;
            case 's': v = (int16_t)(a[3] | (a[4] << 8)); break;
            case 'S': v = (uint16_t)(a[3] | (a[4] << 8)); break;
            case 'i': v = (int32_t)fl_rd32(a + 3); break;
            case 'I': v = fl_rd32(a + 3); break;
            default: t->bad = true;
            }
            if (has_mn || v != l_seq) t->bad = true;
            has_mn = true;
        }
        a = next;
    }
}

// which SEQ bases a group counts: A, C, G, T (and U) -> 0..3, N -> 4 (every base); -1 for any other letter
__host__ __device__ inline int fl_mm_base(uint8_t b) {
    switch (b) {
    case 'A': return 0;
    case 'C': return 1;
    case 'G': return 2;
    case 'T': case 'U': return 3;
    case 'N': return 4;
    default: return -1;
    }
}

// the 4-bit SEQ code ("=ACMGRSVTWYHKDBN") of bases 0..3
__host__ __device__ inline uint32_t fl_mm_code(int base) { return 1u << base; }

// The head B[+-]CODES[.?]? of the group at mm[p]: its length, base and number of codes. False if it does not parse.
__host__ __device__ inline bool fl_mm_head(const uint8_t *mm, uint32_t n, uint32_t p, uint32_t *head_len, int *base, uint32_t *n_codes) {
    const uint32_t p0 = p;
    if (n - p < 3) return false;
    *base = fl_mm_base(mm[p]);
    if (*base < 0 || (mm[p + 1] != '+' && mm[p + 1] != '-')) return false;
    p += 2;
    uint32_t letters = 0, digits = 0;
    for (; p < n && mm[p] >= 'a' && mm[p] <= 'z'; ++p) ++letters;
    if (!letters)
        for (; p < n && mm[p] >= '0' && mm[p] <= '9'; ++p) ++digits;
    if (!letters && !digits) return false;
    if (p < n && (mm[p] == '.' || mm[p] == '?')) ++p;
    if (p >= n || (mm[p] != ',' && mm[p] != ';')) return false;
    *head_len = p - p0;
    *n_codes = letters ? letters : 1;
    return true;
}

// The delta ",digits" at mm[p] (mm[p] == ','): its value and where it ends. False if it is not an unsigned decimal
// below 2^32.
__host__ __device__ inline bool fl_mm_delta(const uint8_t *mm, uint32_t n, uint32_t p, uint64_t *value, uint32_t *next) {
    uint64_t v = 0;
    uint32_t q = p + 1;
    for (; q < n && mm[q] >= '0' && mm[q] <= '9'; ++q) {
        v = v * 10 + (uint64_t)(mm[q] - '0');
        if (v > 0xFFFFFFFFull) return false;
    }
    if (q == p + 1) return false;
    *value = v;
    *next = q;
    return true;
}

// The tags are valid (see the top of this file). count[b]: the SEQ bases that base b counts (count[4] = l_seq).
__host__ __device__ inline bool fl_mods_valid(const FlModTags &t, const uint64_t count[5]) {
    if (!t.has_mm || t.bad) return false;
    const uint8_t *mm = t.mm;
    const uint32_t n = t.mm_len;
    uint64_t values = 0;
    for (uint32_t p = 0; p < n;) {
        uint32_t head, codes;
        int base;
        if (!fl_mm_head(mm, n, p, &head, &base, &codes)) return false;
        p += head;
        int64_t c = -1;
        uint64_t calls = 0;
        while (p < n && mm[p] == ',') {
            uint64_t d;
            if (!fl_mm_delta(mm, n, p, &d, &p)) return false;
            c += (int64_t)d + 1;
            ++calls;
        }
        if (p >= n || mm[p] != ';') return false;
        ++p;
        if (calls && c >= (int64_t)count[base]) return false;
        values += calls * codes;
    }
    return !t.has_ml || values == t.ml_n;
}

__host__ __device__ inline uint32_t fl_dec_digits(uint64_t v) {
    uint32_t d = 1;
    while (v >= 10) { v /= 10; ++d; }
    return d;
}

// writes v in decimal at out, returns its length
__host__ __device__ inline uint32_t fl_dec_write(uint64_t v, uint8_t *out) {
    const uint32_t d = fl_dec_digits(v);
    for (uint32_t i = d; i-- > 0; v /= 10) out[i] = (uint8_t)('0' + v % 10);
    return d;
}

// Where one group's walk stands: p at the ',' of the next call (or the group's ';'), c the index of the last call
// consumed among the bases the group counts (-1 before its first), k the calls consumed.
struct FlMMCursor {
    uint32_t start, p;
    int64_t c;
    uint64_t k;
};

__host__ __device__ inline FlMMCursor fl_mm_cursor(uint32_t after_head) { return FlMMCursor{after_head, after_head, -1, 0}; }

// One group of a child: the calls whose index among the counted bases lies in [before_s, before_e) (the counted bases
// before s and before e). Appends ",delta" per kept call to out (when not null) and returns those bytes; [*k0, *k1):
// the kept calls' ordinals in the group, for ML. The cursor moves past the kept calls, so children visited in the order
// of their starts walk the group once; a child that starts before a call already consumed walks it again from its start.
// The group is valid (fl_mods_valid).
__host__ __device__ inline uint32_t fl_mm_rebase(const uint8_t *mm, uint32_t n, FlMMCursor &cur, uint64_t before_s, uint64_t before_e,
                                                 uint8_t *out, uint64_t *k0, uint64_t *k1) {
    if (cur.c >= (int64_t)before_s) cur = fl_mm_cursor(cur.start);
    uint64_t d;
    uint32_t next;
    while (mm[cur.p] == ',') {
        fl_mm_delta(mm, n, cur.p, &d, &next);
        if (cur.c + (int64_t)d + 1 >= (int64_t)before_s) break;
        cur.c += (int64_t)d + 1;
        cur.p = next;
        ++cur.k;
    }
    *k0 = cur.k;
    uint32_t bytes = 0;
    while (mm[cur.p] == ',') {
        fl_mm_delta(mm, n, cur.p, &d, &next);
        const int64_t c = cur.c + (int64_t)d + 1;
        if (c >= (int64_t)before_e) break;
        if (cur.k == *k0) {
            const uint64_t first = (uint64_t)c - before_s;
            if (out) { out[bytes] = ','; fl_dec_write(first, out + bytes + 1); }
            bytes += 1 + fl_dec_digits(first);
        } else {
            if (out)
                for (uint32_t i = cur.p; i < next; ++i) out[bytes + i - cur.p] = mm[i];
            bytes += next - cur.p;
        }
        cur.c = c;
        cur.p = next;
        ++cur.k;
    }
    *k1 = cur.k;
    return bytes;
}

// position just after the ';' that ends the group the cursor is in; *calls: the group's calls
__host__ __device__ inline uint32_t fl_mm_group_end(const uint8_t *mm, const FlMMCursor &cur, uint64_t *calls) {
    uint32_t p = cur.p;
    uint64_t k = cur.k;
    for (; mm[p] != ';'; ++p) k += mm[p] == ',';
    *calls = k;
    return p + 1;
}

// A child's record before its aux fields: block_size, the fixed fields, read_name name_<s+1>-<e> with its NUL, SEQ, QUAL
__host__ __device__ inline uint32_t fl_child_name_bytes(uint32_t parent_name_len, int s, int e) {
    return parent_name_len + 1 + fl_dec_digits((uint64_t)s + 1) + 1 + fl_dec_digits((uint64_t)e) + 1;
}
__host__ __device__ inline uint64_t fl_child_core_bytes(uint32_t name_bytes, uint32_t n) { return 36 + name_bytes + (n + 1) / 2 + (uint64_t)n; }
// the kept modification fields: MM:Z with its NUL, ML:B:C (when the parent has one), MN:I
__host__ __device__ inline uint64_t fl_child_mods_bytes(const FlModTags &t, uint32_t mm_len, uint64_t ml_n) {
    return 4 + (uint64_t)mm_len + (t.has_ml ? 8 + ml_n : 0) + 7;
}

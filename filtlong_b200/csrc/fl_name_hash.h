// filtlong_b200/csrc/fl_name_hash.h -- the 64-bit hash of a read name that the duplicate-name check (reference
// src/main.cpp:113-117) keys its table on. One definition for the device text parser (fl_text.cu: k_text_records) and
// the host BAM walker (host/bam.cpp): the same name must give the same hash on either path.
//
// FNV-1a over the name's bytes, then a final mix (the upper bits of FNV-1a alone are poorly spread for short names).
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define FL_NAME_HASH_FN __host__ __device__ __forceinline__
#else
#define FL_NAME_HASH_FN inline
#endif

#define FL_NAME_HASH_INIT 0xCBF29CE484222325ull

FL_NAME_HASH_FN unsigned long long fl_name_hash_step(unsigned long long h, unsigned char c) { return (h ^ c) * 0x100000001B3ull; }

FL_NAME_HASH_FN unsigned long long fl_name_hash_final(unsigned long long h) {
    h ^= h >> 29;
    h *= 0xBF58476D1CE4E5B9ull;
    h ^= h >> 32;
    return h;
}

FL_NAME_HASH_FN unsigned long long fl_name_hash(const unsigned char *name, uint64_t n) {
    unsigned long long h = FL_NAME_HASH_INIT;
    for (uint64_t i = 0; i < n; ++i) h = fl_name_hash_step(h, name[i]);
    return fl_name_hash_final(h);
}

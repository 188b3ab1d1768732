// tests/bgzf_codes_dump.cpp -- test helper around the host/device arithmetic of the BGZF kernel (fl_bgzf.h).
//   huff <maxbits> <n> <f_0> ... <f_n-1>   -> the code lengths, then the bit-reversed canonical codes, one line each
//   crc <pieces> <file>                    -> the CRC-32 of the file from its raw per-piece CRCs, as the kernel combines them
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <fstream>
#include <iterator>
#include <vector>

#include "fl_bgzf.h"

int main(int argc, char **argv) {
    if (argc >= 4 && !strcmp(argv[1], "huff")) {
        const int maxbits = atoi(argv[2]), n = atoi(argv[3]);
        std::vector<uint32_t> f(n);
        for (int i = 0; i < n; ++i) f[i] = (uint32_t)strtoul(argv[4 + i], nullptr, 10);
        std::vector<int> order;
        for (int i = 0; i < n; ++i) if (f[i]) order.push_back(i);
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return f[a] < f[b]; });
        std::vector<uint32_t> w(order.size());
        for (size_t i = 0; i < order.size(); ++i) w[i] = f[order[i]];
        fl_huff_lengths_sorted(w.data(), (int)w.size(), maxbits);
        std::vector<uint8_t> len(n, 0);
        for (size_t i = 0; i < order.size(); ++i) len[order[i]] = (uint8_t)w[i];
        std::vector<uint16_t> code(n);
        std::vector<uint32_t> bl(maxbits + 2), nc(maxbits + 2);
        fl_huff_canonical(len.data(), n, maxbits, code.data(), bl.data(), nc.data());
        for (int i = 0; i < n; ++i) printf("%d%c", len[i], i + 1 < n ? ' ' : '\n');
        for (int i = 0; i < n; ++i) printf("%d%c", code[i], i + 1 < n ? ' ' : '\n');
        if (!n) printf("\n\n");
        return 0;
    }
    if (argc >= 4 && !strcmp(argv[1], "crc")) {
        const uint64_t pieces = strtoull(argv[2], nullptr, 10);
        std::ifstream in(argv[3], std::ios::binary);
        std::vector<unsigned char> d((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
        uint32_t tab[256];
        for (uint32_t b = 0; b < 256; ++b) tab[b] = fl_crc32_table_entry(b);
        const uint64_t n = d.size(), per = (n + pieces - 1) / (pieces ? pieces : 1);
        uint32_t x = 0;
        for (uint64_t s = 0; s < n; s += per) {
            const uint64_t e = std::min(n, s + per);
            uint32_t c = 0;
            for (uint64_t i = s; i < e; ++i) c = tab[(c ^ d[i]) & 0xffu] ^ (c >> 8);
            x ^= fl_gf2_mulmod(c, fl_crc32_shift(n - e));
        }
        printf("%u\n", fl_crc32_finish(x, n));
        return 0;
    }
    return 64;
}

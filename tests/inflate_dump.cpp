// tests/inflate_dump.cpp -- test helper: the parallel gzip inflater of fl_inflate.h run serially on the CPU, through the
// same fl_inf_run orchestration the device uses, with the same fl_inflate.h functions at every step.
//   inflate_dump run IN OUT CHUNK_BYTES MAX_DEVICE_BYTES CAP
//       prints "<rc> <members> <chunks> <redecoded> <rounds> <n_out>"; rc 1: OUT holds the bytes, 0: declined
//   inflate_dump finder IN LIMIT_BITS
//       decodes IN serially, recording every block and member header, checks the block-start test at every one of them
//       (missed: starts it rejects), then runs it at every bit offset below LIMIT_BITS to count false positives; prints
//       "<true starts> <missed> <false positives below LIMIT_BITS> <fixed blocks>"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <fstream>
#include <iterator>
#include <set>
#include <string>
#include <vector>

#include "fl_inflate.h"

namespace {

struct Cpu {
    const uint8_t *d;
    uint64_t n;
    uint64_t cap = 0, R = 0;
    std::vector<uint16_t> slots;
    std::vector<FlInfEvent> ev;
    std::vector<uint8_t> out, carry = std::vector<uint8_t>(FL_INF_WINDOW, 0);
    FlInfTables t;
    uint64_t free_bytes() { return ~0ull >> 2; }
    int upload() { return 1; }
    bool alloc(uint64_t r, uint64_t c) {
        R = r; cap = c;
        slots.assign(r * c, 0);
        ev.assign(r * FL_INF_MAXEV, FlInfEvent{});
        return true;
    }
    bool find(uint32_t m, const uint64_t *lo, const uint64_t *hi, uint64_t *bit, uint32_t *kind) {
        for (uint32_t j = 0; j < m; ++j) {
            kind[j] = 0xffffffffu;
            for (uint64_t b = lo[j]; b < hi[j]; ++b) {
                const int k = fl_inf_candidate(d, n, b, &t);
                if (k >= 0) { bit[j] = b; kind[j] = (uint32_t)k; break; }
            }
        }
        return true;
    }
    bool decode(FlInfChunk *ch, uint32_t, const uint32_t *idx, uint32_t m) {
        for (uint32_t i = 0; i < m; ++i)
            fl_inf_decode(d, n, &ch[idx[i]], slots.data() + (size_t)idx[i] * cap, cap, ev.data() + (size_t)idx[i] * FL_INF_MAXEV, &t);
        return true;
    }
    bool events(uint32_t K, FlInfEvent *dst) {
        memcpy(dst, ev.data(), (size_t)K * FL_INF_MAXEV * sizeof(FlInfEvent));
        return true;
    }
    bool resolve(const FlInfChunk *chunks, uint32_t K, const uint64_t *off, const uint32_t *win_lo, uint64_t total, uint8_t *bad) {
        out.assign(total, 0);
        std::vector<uint8_t> w = carry, nw(FL_INF_WINDOW);
        for (uint32_t k = 0; k < K; ++k) {
            const uint16_t *s = slots.data() + (size_t)k * cap;
            const uint64_t L = chunks[k].out_len;
            for (uint64_t i = 0; i < L; ++i) {
                if (s[i] >= FL_INF_MARKER && s[i] - FL_INF_MARKER < win_lo[k]) *bad = 1;
                out[off[k] + i] = fl_inf_resolve(s[i], w.data());
            }
            for (uint64_t j = 0; j < FL_INF_WINDOW; ++j) {        // the window of the next chunk
                const int64_t p = (int64_t)L - (int64_t)FL_INF_WINDOW + (int64_t)j;
                nw[j] = p >= 0 ? out[off[k] + (uint64_t)p] : w[(uint64_t)((int64_t)FL_INF_WINDOW + p)];
            }
            w.swap(nw);
        }
        carry = w;
        return true;
    }
    bool crc(uint32_t m, const uint64_t *lo, const uint64_t *hi, uint32_t *raw) {
        for (uint32_t s = 0; s < m; ++s) {
            uint32_t c = 0;
            for (uint64_t i = lo[s]; i < hi[s]; ++i) c = fl_crc32_table_entry((c ^ out[i]) & 0xffu) ^ (c >> 8);
            raw[s] = c;
        }
        return true;
    }
    bool fetch(uint64_t total, uint8_t *dst) {
        memcpy(dst, out.data(), (size_t)total);
        return true;
    }
};

struct Rec {
    std::vector<std::pair<uint64_t, uint32_t>> *v;
    void operator()(uint64_t bit, uint32_t type) const { v->push_back({bit, type}); }
};

}  // namespace

int main(int argc, char **argv) {
    if (argc < 3) return 64;
    std::ifstream in(argv[2], std::ios::binary);
    std::vector<uint8_t> data((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    const uint64_t n = data.size();
    // an exact-size copy, so that the sanitizer sees any read past the end
    uint8_t *d = (uint8_t *)malloc(n ? n : 1);
    if (n) memcpy(d, data.data(), n);
    if (!strcmp(argv[1], "run") && argc >= 7) {
        Cpu be;
        be.d = d; be.n = n;
        const uint64_t chunk = strtoull(argv[4], nullptr, 10), maxdev = strtoull(argv[5], nullptr, 10), cap = strtoull(argv[6], nullptr, 10);
        std::vector<uint8_t> out(cap ? cap : 1);
        uint64_t n_out = 0;
        FlInfStats st;
        const int rc = fl_inf_run(be, d, n, out.data(), cap, chunk, maxdev, &n_out, &st);
        if (rc == 1) {
            FILE *f = fopen(argv[3], "wb");
            fwrite(out.data(), 1, (size_t)n_out, f);
            fclose(f);
        }
        printf("%d %llu %llu %llu %llu %llu\n", rc, (unsigned long long)st.members, (unsigned long long)st.chunks,
               (unsigned long long)st.redecoded, (unsigned long long)st.rounds, (unsigned long long)n_out);
        free(d);
        return 0;
    }
    if (!strcmp(argv[1], "finder") && argc >= 4) {
        const uint64_t limit = strtoull(argv[3], nullptr, 10);
        std::vector<std::pair<uint64_t, uint32_t>> blocks;
        FlInfChunk c{};
        c.start_bit = 0; c.start_kind = FL_INF_HEADER; c.stop_at = ~0ull;
        const uint64_t cap = std::min<uint64_t>(n * 1100 + 65536, 1ull << 27);
        std::vector<uint16_t> slot(cap);
        std::vector<FlInfEvent> ev(FL_INF_MAXEV);
        FlInfTables t;
        uint64_t total_true = 0, missed = 0, fixed = 0;
        std::set<uint64_t> truth;
        fl_inf_decode(d, n, &c, slot.data(), cap, ev.data(), &t, Rec{&blocks});
        for (auto &b : blocks) {
            if (b.second == 1) { ++fixed; continue; }
            ++total_true;                                          // every start of the stream, whatever LIMIT_BITS is
            truth.insert(b.first);
            const int k = fl_inf_candidate(d, n, b.first, &t);
            const int want = b.second == 4 ? FL_INF_HEADER : FL_INF_BLOCK;
            if (k != want) ++missed;
        }
        uint64_t fp = 0;
        for (uint64_t b = 0; b < limit && b < n * 8; ++b)
            if (fl_inf_candidate(d, n, b, &t) >= 0 && !truth.count(b)) ++fp;
        printf("%llu %llu %llu %llu\n", (unsigned long long)total_true, (unsigned long long)missed, (unsigned long long)fp,
               (unsigned long long)fixed);
        free(d);
        return 0;
    }
    free(d);
    return 64;
}

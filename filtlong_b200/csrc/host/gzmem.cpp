// filtlong_b200/csrc/host/gzmem.cpp -- see gzmem.h.
#include "gzmem.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <thread>
#include <vector>

InflatedInput::~InflatedInput() { release(); }

void InflatedInput::release() {
    if (base) munmap(base, (size_t)reserved);
    base = nullptr;
    size = reserved = 0;
}

namespace {

uint64_t mem_available_bytes() {
    FILE *f = fopen("/proc/meminfo", "r");
    if (!f) return 0;
    char line[256];
    uint64_t kb = 0;
    while (fgets(line, sizeof line, f))
        if (strncmp(line, "MemAvailable:", 13) == 0) {
            kb = strtoull(line + 13, nullptr, 10);
            break;
        }
    fclose(f);
    return kb << 10;
}

uint64_t page_round(uint64_t n) {
    const uint64_t pg = (uint64_t)sysconf(_SC_PAGESIZE);
    return (n + pg - 1) / pg * pg;
}

char *reserve(uint64_t bytes) {
    void *p = mmap(nullptr, (size_t)bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) return nullptr;
    madvise(p, (size_t)bytes, MADV_HUGEPAGE);                          // fewer faults while the inflaters write; a hint only
    return (char *)p;
}

inline uint32_t le16(const unsigned char *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
inline uint32_t le32(const unsigned char *p) { return le16(p) | (le16(p + 2) << 16); }

struct Member {
    uint64_t off, csize, out_off;
    uint32_t isize;
};

// BGZF: every member is a complete gzip member whose extra field holds SI1='B', SI2='C', SLEN=2, BSIZE = size - 1
// (SAM specification, section 4.1). True only if the WHOLE file is such members, back to back.
bool scan_bgzf(const unsigned char *d, uint64_t n, std::vector<Member> &ms, uint64_t &total) {
    uint64_t pos = 0;
    total = 0;
    while (pos < n) {
        if (n - pos < 12 + 6 + 8) return false;
        const unsigned char *h = d + pos;
        if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) return false;
        const uint64_t xlen = le16(h + 10);
        if (pos + 12 + xlen + 8 > n) return false;
        int64_t bsize = -1;
        uint64_t q = 12;
        while (q + 4 <= 12 + xlen) {
            const uint32_t slen = le16(h + q + 2);
            if (h[q] == 'B' && h[q + 1] == 'C' && slen == 2 && q + 6 <= 12 + xlen) bsize = (int64_t)le16(h + q + 4);
            q += 4 + slen;
        }
        if (bsize < 0) return false;
        const uint64_t csize = (uint64_t)bsize + 1;
        if (csize < 12 + xlen + 8 || pos + csize > n) return false;
        const uint32_t isize = le32(h + csize - 4);
        ms.push_back(Member{pos, csize, total, isize});
        total += isize;
        pos += csize;
    }
    return !ms.empty();
}

bool inflate_members(const unsigned char *d, const std::vector<Member> &ms, size_t lo, size_t hi, char *out) {
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, 15 + 16) != Z_OK) return false;
    bool ok = true;
    unsigned char nothing[8];
    for (size_t i = lo; i < hi && ok; ++i) {
        const Member &m = ms[i];
        if (i > lo && inflateReset(&zs) != Z_OK) { ok = false; break; }
        zs.next_in = const_cast<unsigned char *>(d + m.off);
        zs.avail_in = (uInt)m.csize;                                    // <= 65536
        if (m.isize) {
            zs.next_out = reinterpret_cast<unsigned char *>(out + m.out_off);
            zs.avail_out = m.isize;
        } else {                                                        // the empty end-of-file block
            zs.next_out = nothing;
            zs.avail_out = sizeof nothing;
        }
        const int rc = inflate(&zs, Z_FINISH);
        ok = rc == Z_STREAM_END && zs.avail_in == 0 && zs.total_out == m.isize;   // zlib has checked CRC-32 and ISIZE
    }
    inflateEnd(&zs);
    return ok;
}

}  // namespace

uint64_t input_memory_budget() { return mem_available_bytes() / 10 * 6; }

bool inflate_gzip_memory(const unsigned char *d, uint64_t n, InflatedInput &out, int max_threads, uint64_t budget, std::string *why,
                         const GzipDeviceInflate &device) {
    auto fail = [&](const char *msg) {
        if (why) *why = msg;
        out.release();
        return false;
    };
    out.release();
    if (n < 18 || d[0] != 0x1f || d[1] != 0x8b) return fail("not a gzip file");
    if (budget == 0) budget = input_memory_budget();
    if (budget == 0) return fail("cannot tell how much memory is available");

    // ---- BGZF: sizes known, members independent ----
    std::vector<Member> ms;
    uint64_t total = 0;
    if (scan_bgzf(d, n, ms, total)) {
        if (total == 0) return fail("empty input");
        if (total > budget) return fail("inflated input would not fit the memory budget");
        out.reserved = page_round(total);
        out.base = reserve(out.reserved);
        if (!out.base) return fail("cannot reserve memory for the inflated input");
        int T = max_threads > 0 ? max_threads : (int)std::thread::hardware_concurrency();
        if (T > 32) T = 32;
        if ((size_t)T > ms.size() / 16 + 1) T = (int)(ms.size() / 16 + 1);
        if (T < 1) T = 1;
        // contiguous member ranges, balanced by compressed bytes
        std::vector<size_t> cut((size_t)T + 1, ms.size());
        cut[0] = 0;
        {
            size_t i = 0;
            for (int t = 1; t < T; ++t) {
                const uint64_t goal = n / (uint64_t)T * (uint64_t)t;
                while (i < ms.size() && ms[i].off < goal) ++i;
                cut[(size_t)t] = i;
            }
        }
        std::atomic<bool> ok(true);
        std::vector<std::thread> ts;
        int started = 1;                                               // ranges [0, started) have an owner
        for (int t = 1; t < T; ++t) {
            try {
                ts.emplace_back([&, t] {
                    if (!inflate_members(d, ms, cut[(size_t)t], cut[(size_t)t + 1], out.base)) ok.store(false);
                });
                started = t + 1;
            } catch (...) {                                            // no more threads to be had: this one does the rest
                break;
            }
        }
        if (!inflate_members(d, ms, cut[0], cut[1], out.base)) ok.store(false);
        if (started < T && !inflate_members(d, ms, cut[(size_t)started], cut[(size_t)T], out.base)) ok.store(false);
        for (auto &th : ts) th.join();
        if (!ok.load()) return fail("corrupt BGZF member");
        out.size = total;
        out.members = (int)ms.size();
        out.threads = T;
        out.bgzf = true;
        return true;
    }

    // ---- any other gzip file: one stream, members back to back (what gzread does) ----
    uint64_t want = n > (budget / 1032) ? budget : n * 1032 + 65536;     // deflate cannot expand by more than ~1032:1
    if (want > budget) want = budget;
    out.reserved = page_round(want);
    out.base = reserve(out.reserved);
    if (!out.base) return fail("cannot reserve memory for the inflated input");
    auto keep_used = [&](uint64_t used) {                              // give the unused tail of the reservation back
        const uint64_t keep = page_round(used);
        if (keep < out.reserved) {
            munmap(out.base + keep, (size_t)(out.reserved - keep));
            out.reserved = keep;
        }
    };
    if (device) {
        GzipDeviceResult r;
        const bool ok = device(d, n, out.base, out.reserved, &r);
        out.inflater = r.note;
        if (ok && r.n_out) {
            keep_used(r.n_out);
            out.size = r.n_out;
            out.members = (int)r.members;
            out.threads = 0;
            out.bgzf = false;
            return true;
        }
        // declined: the host path below, on the same reservation (an empty result is the host's "empty input" too)
    }
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, 15 + 16) != Z_OK) return fail("zlib: inflateInit2 failed");
    uint64_t ipos = 0, opos = 0;
    int members = 0;
    const char *err = nullptr;
    const uint64_t piece = 1ull << 30;
    for (;;) {
        const uint64_t in_now = std::min(n - ipos, piece), out_now = std::min(out.reserved - opos, piece);
        if (out_now == 0) { err = "inflated input would not fit the memory budget"; break; }
        zs.next_in = const_cast<unsigned char *>(d + ipos);
        zs.avail_in = (uInt)in_now;
        zs.next_out = reinterpret_cast<unsigned char *>(out.base + opos);
        zs.avail_out = (uInt)out_now;
        const int rc = inflate(&zs, Z_NO_FLUSH);
        ipos += in_now - zs.avail_in;
        opos += out_now - zs.avail_out;
        if (rc == Z_STREAM_END) {
            ++members;
            if (n - ipos < 2 || d[ipos] != 0x1f || d[ipos + 1] != 0x8b) break;    // end of file, or trailing bytes gzread ignores
            if (inflateReset(&zs) != Z_OK) { err = "zlib: inflateReset failed"; break; }
            continue;
        }
        if (rc == Z_OK) {
            if (ipos >= n) { err = "truncated gzip stream"; break; }
            continue;
        }
        err = rc == Z_BUF_ERROR ? "truncated gzip stream" : "corrupt gzip stream";
        break;
    }
    inflateEnd(&zs);
    if (err) return fail(err);
    if (opos == 0) return fail("empty input");
    keep_used(opos);
    out.size = opos;
    out.members = members;
    out.threads = 1;
    out.bgzf = false;
    return true;
}

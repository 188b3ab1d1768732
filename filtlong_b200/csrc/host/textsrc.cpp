// filtlong_b200/csrc/host/textsrc.cpp -- see textsrc.h.
#include "textsrc.h"

#include <fcntl.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "bam.h"
#include "gzmem.h"

bool MappedFile::open_plain(const std::string &path) {
    fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) return false;
    struct stat st;
    if (fstat(fd, &st) != 0 || !S_ISREG(st.st_mode) || st.st_size < 2) return false;
    size = map_bytes = (uint64_t)st.st_size;
    void *p = mmap(nullptr, (size_t)size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (p == MAP_FAILED) return false;
    base = (const char *)p;
    madvise(p, (size_t)size, MADV_SEQUENTIAL);
    const unsigned char b0 = (unsigned char)base[0], b1 = (unsigned char)base[1];
    gzip = b0 == 0x1f && b1 == 0x8b;
    return !gzip;
}

bool MappedFile::inflate(uint64_t budget, std::string *why, const GzipDeviceInflate &device) {
    if (!gzip || !base) return false;
    InflatedInput in;
    int threads = 0;
    if (const char *e = getenv("FL_INFLATE_THREADS")) threads = atoi(e);
    const bool ok = inflate_gzip_memory((const unsigned char *)base, size, in, threads, budget, why, device);
    inflater = in.inflater.empty() ? "host threads" : in.inflater;
    if (!ok) return false;
    munmap((void *)base, (size_t)map_bytes);
    if (fd >= 0) ::close(fd);
    fd = -1;
    size = in.size;
    map_bytes = in.reserved;
    base = in.take();
    return true;
}

bool MappedFile::open_any(const std::string &path, bool *inflated, std::string *why, const GzipDeviceInflate &device) {
    if (inflated) *inflated = false;
    if (open_plain(path)) return true;
    std::string w;
    if (!why) why = &w;
    if (!gzip) return false;                                           // not gzip either
    if (getenv("FL_GZ_HOST")) { *why = "FL_GZ_HOST is set"; return false; }
    if (!inflate(0, why, device)) return false;                        // declined (gzmem.h)
    if (inflated) *inflated = true;
    return true;
}

int MappedFile::format() const {
    if (!base || !size) return 0;
    if (base[0] == '@') return FL_TEXT_FASTQ;
    if (base[0] == '>') return FL_TEXT_FASTA;
    return fd < 0 && bam_magic(base, size) ? FL_FORMAT_BAM : 0;
}

MappedFile::~MappedFile() {
    if (base) munmap((void *)base, (size_t)map_bytes);
    if (fd >= 0) ::close(fd);
}

uint64_t chunk_target(uint64_t default_bytes) {
    uint64_t target = default_bytes;
    if (const char *e = getenv("FL_CHUNK_MB")) target = (uint64_t)atoll(e) << 20;
    return target < (1ull << 20) ? 1ull << 20 : target > (1024ull << 20) ? 1024ull << 20 : target;
}

namespace {

inline uint64_t eol(const char *b, uint64_t from, uint64_t size) {
    if (from >= size) return size;
    const void *p = memchr(b + from, '\n', (size_t)(size - from));
    return p ? (uint64_t)((const char *)p - b) : size;
}

// Is `p` the first byte of a record? FASTQ: '@' line, a sequence line that kseq takes for one (not empty, not led by
// '@', '>' or '+': kseq.h:199), a '+' line, a quality line as long as the sequence (a quality line that begins with '@'
// fails the '+' test two lines on). FASTA: any line starting with '>'. A cut the device then rejects costs only the
// fast path: the host reader takes over at the chunk's first byte.
bool record_starts_at(const char *b, uint64_t p, uint64_t size, int format) {
    if (p >= size) return false;
    if (format == FL_TEXT_FASTA) return b[p] == '>';
    if (b[p] != '@') return false;
    const uint64_t e0 = eol(b, p, size), s1 = e0 + 1, e1 = eol(b, s1, size), s2 = e1 + 1;
    if (e1 <= s1 || b[s1] == '@' || b[s1] == '>' || b[s1] == '+') return false;
    if (s2 >= size || b[s2] != '+') return false;
    const uint64_t e2 = eol(b, s2, size), s3 = e2 + 1, e3 = eol(b, s3, size);
    return s3 <= size && e3 - s3 == e1 - s1;
}

// Have the four lines of a FASTQ record starting at p all arrived? Only then does record_starts_at over the bytes so far
// answer what it answers over the whole input.
bool lines_arrived(const char *b, uint64_t p, uint64_t avail, bool ended, int format) {
    if (ended || format == FL_TEXT_FASTA) return true;
    for (int i = 0; i < 4; ++i) {
        const uint64_t e = eol(b, p, avail);
        if (e >= avail) return false;
        p = e + 1;
    }
    return true;
}

}  // namespace

int plan_next_chunk(const char *b, uint64_t avail, bool ended, int format, uint64_t target, uint64_t max_chunk, uint64_t pos, Chunk *out) {
    if (pos >= avail) return 0;
    uint64_t end = avail;
    if (avail - pos > target) {
        uint64_t p = pos + target;                             // last record start at or before pos + target
        bool found = false;
        while (p > pos) {
            const void *q = memrchr(b + pos, '\n', (size_t)(p - pos));
            if (!q) break;
            const uint64_t cand = (uint64_t)((const char *)q - b) + 1;
            if (!lines_arrived(b, cand, avail, ended, format)) return 0;
            if (cand > pos && record_starts_at(b, cand, avail, format)) { end = cand; found = true; break; }
            p = cand - 1;
            if (pos + target - p > (64ull << 20)) break;        // a single record this large: give up on the fast path
        }
        if (!found) return -1;
    } else if (!ended) {
        return 0;
    }
    if (end - pos > max_chunk) return -1;
    *out = Chunk{pos, end};
    return 1;
}

bool plan_chunks(const char *b, uint64_t size, int format, uint64_t target, uint64_t max_chunk, std::vector<Chunk> &out) {
    Chunk c;
    int r;
    for (uint64_t pos = 0; (r = plan_next_chunk(b, size, true, format, target, max_chunk, pos, &c)) == 1; pos = c.end) out.push_back(c);
    return r == 0;
}


// tests/bam_dump.cpp -- drives the BAM walker (filtlong_b200/csrc/host/bam.h) and the BAM side of the pass-2 writer
// (survivors.h) without a GPU.
//
//   bam_dump index FILE          the chunk plan (FL_CHUNK_MB, as the CLI reads it) and every record's index entry:
//                                "C begin end" per chunk, then "R name_off name_len seq_off qual_off len name_hash" per
//                                record, file offsets in the inflated input
//   bam_dump write FILE SPEC     the uncompressed BAM pass 2 writes for the results in SPEC: per read, in order,
//                                "n_child" and then one "start end passed" triple per row (a read without children has one)
//   bam_dump hash NAME...        fl_name_hash of each name, one per line
//
// Exit code: 0 done; 1 a check failed ("Error: ..." on stderr, as the CLI prints it); 2 bad usage; 3 FILE is not a
// BAM file that inflates into memory; 4 the writer failed.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "../filtlong_b200/csrc/fl_name_hash.h"
#include "../filtlong_b200/csrc/host/bam.h"
#include "../filtlong_b200/csrc/host/survivors.h"
#include "../filtlong_b200/csrc/host/textsrc.h"

namespace {

struct Indexed {
    uint64_t header = 0;
    std::vector<Chunk> plan;
    Records rec;
};

int index_file(const MappedFile &f, Indexed &out) {
    if (f.format() != FL_FORMAT_BAM) return 3;
    uint64_t target = 128ull << 20, max_chunk = 0;
    if (const char *e = getenv("FL_CHUNK_MB")) target = (uint64_t)atoll(e) << 20;
    std::string why;
    if (!bam_header(f.base, f.size, &out.header, &why) || !bam_plan_chunks(f.base, f.size, out.header, target, out.plan, &max_chunk, &why)) {
        std::cerr << "Error: " << why << "\n";
        return 1;
    }
    for (const Chunk &c : out.plan) {
        BamChunkIndex ix;
        if (!bam_index_chunk(f.base, c, ix)) {
            std::cerr << "Error: " << ix.error << "\n";
            return 1;
        }
        for (size_t j = 0; j < ix.rec.n; ++j) {
            out.rec.add(ix.rec.name_off[j] + c.begin, ix.rec.name_len[j], 0, ix.rec.seq_off[j] + c.begin, ix.rec.qual_off[j] + c.begin,
                        ix.rec.len[j]);
            out.rec.name_hash[out.rec.n - 1] = ix.rec.name_hash[j];
            if (ix.seq32[j] != ix.rec.seq_off[j] || ix.qual32[j] != ix.rec.qual_off[j]) return 5;
        }
    }
    return 0;
}

}  // namespace

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    const std::string mode = argv[1];
    if (mode == "hash") {
        for (int i = 2; i < argc; ++i) printf("%llu\n", fl_name_hash((const unsigned char *)argv[i], strlen(argv[i])));
        return 0;
    }
    if (argc < 3) return 2;
    MappedFile f;
    if (!f.open_any(argv[2])) return 3;
    Indexed ix;
    const int rc = index_file(f, ix);
    if (rc) return rc;
    if (mode == "index") {
        for (const Chunk &c : ix.plan) printf("C %llu %llu\n", (unsigned long long)c.begin, (unsigned long long)c.end);
        const Records &R = ix.rec;
        for (size_t i = 0; i < R.n; ++i)
            printf("R %llu %u %llu %llu %d %llu\n", (unsigned long long)R.name_off[i], R.name_len[i], (unsigned long long)R.seq_off[i],
                   (unsigned long long)R.qual_off[i], R.len[i], (unsigned long long)R.name_hash[i]);
        return 0;
    }
    if (mode != "write" || argc != 4) return 2;
    struct {
        std::vector<int32_t> n_child, row_s, row_e;
        std::vector<uint64_t> row_start;
        std::vector<uint8_t> row_pfinal;
    } res;
    std::ifstream spec(argv[3]);
    int32_t n_child;
    while (spec >> n_child) {
        res.n_child.push_back(n_child);
        res.row_start.push_back(res.row_s.size());
        for (int k = 0; k < (n_child ? n_child : 1); ++k) {
            int32_t s, e, passed;
            spec >> s >> e >> passed;
            res.row_s.push_back(s);
            res.row_e.push_back(e);
            res.row_pfinal.push_back((uint8_t)passed);
        }
    }
    if (res.n_child.size() != ix.rec.n) return 2;
    const Format fmt{'@', true, true, ix.header};
    return write_survivors(1, f.base, {Part{&ix.rec, Results::of(res)}}, fmt, nullptr) ? 0 : 4;
}

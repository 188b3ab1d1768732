// tests/bam_aligned_dump.cpp -- drives the aligned BAM walker (bam.h, --aligned), the follower join and the BAM side of the
// pass-2 writer (survivors.h) without a GPU.
//
//   bam_aligned_dump index FILE          the chunk plan (FL_CHUNK_MB) and the index: "C begin end" per chunk, then
//                                        "R name_off name_len seq_off qual_off len name_hash reverse" per read record and
//                                        "F off before name_hash owner" per follower (before and owner: indexes among all
//                                        read records; owner -1: an orphan), file offsets in the inflated input
//   bam_aligned_dump write FILE SPEC WANT the uncompressed BAM pass 2 writes for WANT (1: stdout, 0: --failed) when read i
//                                        has pass flag i of SPEC (whitespace-separated 0 / 1)
//
// With FL_DUMP_PARTS=k the chunks are dealt to k parts as contiguous ranges, as the CLI deals them to GPUs, and the join
// crosses parts. Exit code: 0 done; 1 a check failed ("Error: ..." on stderr, as the CLI prints it); 2 bad usage; 3 FILE is
// not a BAM file that inflates into memory; 4 the writer failed.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "../filtlong_b200/csrc/host/bam.h"
#include "../filtlong_b200/csrc/host/survivors.h"
#include "../filtlong_b200/csrc/host/textsrc.h"

namespace {

struct PartData {
    Records rec;
    std::vector<Follower> followers;
    std::vector<uint8_t> reverse;
    std::vector<int32_t> n_child, row_s, row_e;
    std::vector<uint64_t> row_start;
    std::vector<uint8_t> row_pfinal;
};

}  // namespace

int main(int argc, char **argv) {
    if (argc < 3) return 2;
    const std::string mode = argv[1];
    MappedFile f;
    if (!f.open_any(argv[2]) || f.format() != FL_FORMAT_BAM) return 3;
    uint64_t target = 128ull << 20, max_chunk = 0, header = 0;
    if (const char *e = getenv("FL_CHUNK_MB")) target = (uint64_t)atoll(e) << 20;
    size_t n_parts = 1;
    if (const char *e = getenv("FL_DUMP_PARTS")) n_parts = (size_t)atoll(e);
    std::string why;
    std::vector<Chunk> plan;
    if (!bam_header(f.base, f.size, &header, &why) || !bam_plan_chunks(f.base, f.size, header, target, plan, &max_chunk, &why)) {
        std::cerr << "Error: " << why << "\n";
        return 1;
    }
    std::vector<PartData> parts(n_parts);
    for (size_t ci = 0; ci < plan.size(); ++ci) {
        BamChunkIndex ix;
        if (!bam_index_chunk(f.base, plan[ci], ix, true)) {
            std::cerr << "Error: " << ix.error << "\n";
            return 1;
        }
        PartData &d = parts[ci * n_parts / plan.size()];
        bam_append_chunk(ix, plan[ci], d.rec, d.followers, &d.reverse);
    }
    std::vector<const Records *> tables;
    for (auto &d : parts) tables.push_back(&d.rec);
    NameIndex names;
    std::string dup;
    if (!names.build(tables, f.base, &dup)) {
        std::cerr << "Error: duplicate read name: " << dup << "\n";
        return 1;
    }
    uint64_t orphans = 0;
    for (auto &d : parts) orphans += bam_join_followers(f.base, names, d.followers);
    std::vector<uint64_t> first(n_parts + 1, 0);                 // parts' first reads among all
    for (size_t k = 0; k < n_parts; ++k) first[k + 1] = first[k] + parts[k].rec.n;
    if (mode == "index") {
        for (const Chunk &c : plan) printf("C %llu %llu\n", (unsigned long long)c.begin, (unsigned long long)c.end);
        for (size_t k = 0; k < n_parts; ++k) {
            const Records &R = parts[k].rec;
            for (size_t i = 0; i < R.n; ++i)
                printf("R %llu %u %llu %llu %d %llu %d\n", (unsigned long long)R.name_off[i], R.name_len[i], (unsigned long long)R.seq_off[i],
                       (unsigned long long)R.qual_off[i], R.len[i], (unsigned long long)R.name_hash[i], parts[k].reverse[i]);
        }
        for (size_t k = 0; k < n_parts; ++k)
            for (const Follower &x : parts[k].followers)
                printf("F %llu %llu %llu %lld\n", (unsigned long long)x.off, (unsigned long long)(first[k] + x.before),
                       (unsigned long long)x.name_hash, x.owner_part < 0 ? -1ll : (long long)(first[x.owner_part] + x.owner));
        fprintf(stderr, "orphans %llu\n", (unsigned long long)orphans);
        return 0;
    }
    if (mode != "write" || argc != 5) return 2;
    std::ifstream spec(argv[3]);
    int passed;
    size_t k = 0;
    while (spec >> passed) {
        while (k < n_parts && parts[k].row_pfinal.size() == parts[k].rec.n) ++k;
        if (k == n_parts) return 2;
        PartData &d = parts[k];
        d.n_child.push_back(0);
        d.row_start.push_back(d.row_s.size());
        d.row_s.push_back(0);
        d.row_e.push_back(d.rec.len[d.row_pfinal.size()]);
        d.row_pfinal.push_back((uint8_t)passed);
    }
    std::vector<Part> ps;
    for (auto &d : parts) {
        if (d.row_pfinal.size() != d.rec.n) return 2;
        ps.push_back(Part{&d.rec, Results::of(d), &d.followers});
    }
    const Format fmt{'@', true, true, header};
    return write_survivors(1, f.base, ps, fmt, nullptr, atoi(argv[4]) != 0) ? 0 : 4;
}

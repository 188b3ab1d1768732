// tests/bam_mods_dump.cpp -- the pass-2 writer (survivors.h) without a context and with --keep_mods, on a BAM file: the
// host's children, built by bam_child_record over fl_bam_mods.h.
//
//   bam_mods_dump FILE SPEC      the uncompressed BAM on stdout for the results in SPEC (per read, in order, "n_child"
//                                and then one "start end passed" triple per row; a read without children has one), then
//                                "kept invalid" on stderr
//
// Exit code: 0 done; 1 a check failed; 2 bad usage; 3 FILE is not BAM; 4 the writer failed.
#include <cstdio>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "../filtlong_b200/csrc/host/bam.h"
#include "../filtlong_b200/csrc/host/survivors.h"
#include "../filtlong_b200/csrc/host/textsrc.h"

int main(int argc, char **argv) {
    if (argc != 3) return 2;
    MappedFile f;
    if (!f.open_any(argv[1]) || f.format() != FL_FORMAT_BAM) return 3;
    uint64_t header = 0, max_chunk = 0, max_record = 0;
    std::vector<Chunk> plan;
    std::string why;
    if (!bam_header(f.base, f.size, &header, &why) || !bam_plan_chunks(f.base, f.size, header, 128ull << 20, plan, &max_chunk, &why, &max_record)) {
        std::cerr << "Error: " << why << "\n";
        return 1;
    }
    Records rec;
    for (const Chunk &c : plan) {
        BamChunkIndex ix;
        if (!bam_index_chunk(f.base, c, ix)) {
            std::cerr << "Error: " << ix.error << "\n";
            return 1;
        }
        for (size_t j = 0; j < ix.rec.n; ++j)
            rec.add(ix.rec.name_off[j] + c.begin, ix.rec.name_len[j], 0, ix.rec.seq_off[j] + c.begin, ix.rec.qual_off[j] + c.begin, ix.rec.len[j]);
    }
    struct {
        std::vector<int32_t> n_child, row_s, row_e;
        std::vector<uint64_t> row_start;
        std::vector<uint8_t> row_pfinal;
    } res;
    std::ifstream spec(argv[2]);
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
    if (res.n_child.size() != rec.n) return 2;
    Format fmt{'@', true, true, header, max_record, true};
    uint64_t counts[2] = {0, 0};
    const bool ok = write_survivors(1, f.base, {Part{&rec, Results::of(res)}}, fmt, nullptr, true, counts);
    std::cerr << counts[0] << " " << counts[1] << "\n";
    return ok ? 0 : 4;
}

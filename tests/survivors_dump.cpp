// tests/survivors_dump.cpp -- drives the CLI's pass-2 writer (filtlong_b200/csrc/host/survivors.h) without a GPU: the
// table of record offsets and the scoring results come from a spec file, the survivors go to stdout.
//
//   survivors_dump MODE fastq|fasta LEAD_CHECKED INPUT SPEC        MODE: auto, writev, pwrite or reparse
//
// SPEC is whitespace-separated: "P" starts a part (reparse takes exactly one); "R name_off name_len comment_len seq_off
// qual_off len n_child" is a read of the current part, and "W start end passed" one of its rows (a read without children
// has one row). Exit code: 0 written, 1 the writer reported a failure, 2 bad usage, 3 INPUT not mappable, 4 the table
// does not fit in INPUT.
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "../filtlong_b200/csrc/host/survivors.h"
#include "../filtlong_b200/csrc/host/textsrc.h"

struct PartData {
    Records rec;
    std::vector<int32_t> n_child, row_s, row_e;
    std::vector<uint64_t> row_start;
    std::vector<uint8_t> row_pfinal;
};

int main(int argc, char **argv) {
    if (argc != 6) return 2;
    const std::string mode = argv[1];
    const Format fmt = strcmp(argv[2], "fasta") == 0 ? Format{'>', false} : Format{'@', true};
    std::vector<PartData> data;
    std::ifstream spec(argv[5]);
    std::string tag;
    while (spec >> tag) {
        if (tag == "P") {
            data.emplace_back();
            data.back().rec.lead_checked = strcmp(argv[3], "1") == 0;
            continue;
        }
        if (data.empty()) return 2;
        PartData &d = data.back();
        if (tag == "R") {
            uint64_t name_off, seq_off, qual_off;
            uint32_t name_len, comment_len;
            int32_t len, n_child;
            spec >> name_off >> name_len >> comment_len >> seq_off >> qual_off >> len >> n_child;
            d.rec.add(name_off, name_len, comment_len, seq_off, qual_off, len);
            d.n_child.push_back(n_child);
            d.row_start.push_back(d.row_s.size());
        } else if (tag == "W") {
            int32_t s, e, passed;
            spec >> s >> e >> passed;
            d.row_s.push_back(s);
            d.row_e.push_back(e);
            d.row_pfinal.push_back((uint8_t)passed);
        } else {
            return 2;
        }
    }
    std::vector<Part> parts;
    for (auto &d : data) parts.push_back(Part{&d.rec, Results::of(d)});
    bool ok;
    if (mode == "reparse") {
        if (parts.size() != 1) return 2;
        ok = reparse_survivors(1, argv[4], parts[0].res, parts[0].rec->n, fmt, nullptr);
    } else {
        MappedFile f;
        if (!f.open_plain(argv[4])) return 3;
        for (auto &d : data)
            if (!d.rec.within(f.size, fmt.quality)) return 4;
        if (mode == "auto") ok = write_survivors(1, f.base, parts, fmt, nullptr);
        else if (mode == "writev") ok = write_survivors_writev(1, f.base, parts, fmt);
        else if (mode == "pwrite") ok = write_survivors_pwrite(1, f.base, parts, fmt);
        else return 2;
    }
    return ok ? 0 : 1;
}

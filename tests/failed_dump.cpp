// tests/failed_dump.cpp -- drives the CLI's pass-2 writer (filtlong_b200/csrc/host/survivors.h) with a second output, as
// `--failed FILE` uses it, without a GPU: the survivors go to stdout and the other rows to descriptor FAILED_FD.
//
//   failed_dump MODE fastq|fasta LEAD_CHECKED INPUT SPEC FAILED_FD   MODE: auto, writev, pwrite or reparse; SPEC as
//                                                                    tests/survivors_dump.cpp reads it
//   failed_dump auto bam - INPUT SPEC FAILED_FD                      INPUT a BAM file, indexed here; SPEC as
//                                                                    tests/bam_dump.cpp's write reads it; uncompressed
//
// On the random-access modes the second output is a second call with want = false after stdout's; reparse writes both
// from one parse. Exit code: 0 both written; 1 a writer reported a failure ("stdout" / "failed" on stderr says which); 2
// bad usage; 3 INPUT not mappable (or not BAM); 4 the table does not fit in INPUT.
#include <cstdio>
#include <cstdlib>
#include <cstring>
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
    std::vector<int32_t> n_child, row_s, row_e;
    std::vector<uint64_t> row_start;
    std::vector<uint8_t> row_pfinal;
    void row(int32_t s, int32_t e, int32_t passed) {
        row_s.push_back(s);
        row_e.push_back(e);
        row_pfinal.push_back((uint8_t)passed);
    }
};

bool read_text_spec(const char *path, bool lead_checked, std::vector<PartData> &data) {
    std::ifstream spec(path);
    std::string tag;
    while (spec >> tag) {
        if (tag == "P") {
            data.emplace_back();
            data.back().rec.lead_checked = lead_checked;
            continue;
        }
        if (data.empty()) return false;
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
            d.row(s, e, passed);
        } else {
            return false;
        }
    }
    return true;
}

// the records of a BAM file (bam.h, as the feeder indexes them) and the results in SPEC; 0, or an exit code
int read_bam(const MappedFile &f, const char *spec_path, uint64_t *header, PartData &d) {
    if (f.format() != FL_FORMAT_BAM) return 3;
    std::vector<Chunk> plan;
    uint64_t max_chunk = 0;
    std::string why;
    if (!bam_header(f.base, f.size, header, &why) || !bam_plan_chunks(f.base, f.size, *header, 128ull << 20, plan, &max_chunk, &why)) return 3;
    for (const Chunk &c : plan) {
        BamChunkIndex ix;
        if (!bam_index_chunk(f.base, c, ix)) return 3;
        for (size_t j = 0; j < ix.rec.n; ++j)
            d.rec.add(ix.rec.name_off[j] + c.begin, ix.rec.name_len[j], 0, ix.rec.seq_off[j] + c.begin, ix.rec.qual_off[j] + c.begin,
                      ix.rec.len[j]);
    }
    std::ifstream spec(spec_path);
    int32_t n_child;
    while (spec >> n_child) {
        d.n_child.push_back(n_child);
        d.row_start.push_back(d.row_s.size());
        for (int k = 0; k < (n_child ? n_child : 1); ++k) {
            int32_t s, e, passed;
            spec >> s >> e >> passed;
            d.row(s, e, passed);
        }
    }
    return d.n_child.size() == d.rec.n ? 0 : 2;
}

}  // namespace

int main(int argc, char **argv) {
    if (argc != 7) return 2;
    const std::string mode = argv[1], kind = argv[2];
    const int failed_fd = atoi(argv[6]);
    bool ok = true, failed_ok = true;
    if (kind == "bam") {
        if (mode != "auto") return 2;
        MappedFile f;
        if (!f.open_any(argv[4])) return 3;
        PartData d;
        Format fmt{'@', true, true, 0};
        if (const int rc = read_bam(f, argv[5], &fmt.bam_header, d)) return rc;
        const std::vector<Part> parts{Part{&d.rec, Results::of(d)}};
        ok = write_survivors(1, f.base, parts, fmt, nullptr);
        failed_ok = write_survivors(failed_fd, f.base, parts, fmt, nullptr, false);
    } else {
        const Format fmt = kind == "fasta" ? Format{'>', false} : Format{'@', true};
        std::vector<PartData> data;
        if (!read_text_spec(argv[5], strcmp(argv[3], "1") == 0, data)) return 2;
        std::vector<Part> parts;
        for (auto &d : data) parts.push_back(Part{&d.rec, Results::of(d)});
        if (mode == "reparse") {
            if (parts.size() != 1) return 2;
            ok = reparse_survivors(1, argv[4], parts[0].res, parts[0].rec->n, fmt, nullptr, failed_fd, &failed_ok);
        } else {
            MappedFile f;
            if (!f.open_plain(argv[4])) return 3;
            for (auto &d : data)
                if (!d.rec.within(f.size, fmt.quality)) return 4;
            for (bool want : {true, false}) {
                const int fd = want ? 1 : failed_fd;
                bool &r = want ? ok : failed_ok;
                if (mode == "auto") r = write_survivors(fd, f.base, parts, fmt, nullptr, want);
                else if (mode == "writev") r = write_survivors_writev(fd, f.base, parts, fmt, want);
                else if (mode == "pwrite") r = write_survivors_pwrite(fd, f.base, parts, fmt, want);
                else return 2;
            }
        }
    }
    if (!ok) std::cerr << "stdout\n";
    if (!failed_ok) std::cerr << "failed\n";
    return ok && failed_ok ? 0 : 1;
}

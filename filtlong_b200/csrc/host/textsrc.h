// filtlong_b200/csrc/host/textsrc.h -- an input file as ONE byte range cut into record-aligned chunks: what the device-text
// entry points (fl_reads_push_text for the reads, fl_kmers_add_text for the -1/-2/-a references) are fed from.
// A plain file is mapped; a gzip file is inflated once into memory (gzmem.h). Replaces, for the common record layout,
// the gzopen / kseq_init / kseq_read loops of reference src/main.cpp:70-75 and src/kmers.cpp:76-89.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../../include/filtlong_b200.h"
#include "gzmem.h"

struct MappedFile {
    const char *base = nullptr;
    uint64_t size = 0;
    uint64_t map_bytes = 0;                                         // what munmap() gets
    int fd = -1;                                                    // < 0: `base` is memory (an inflated gzip file), not a file mapping
    bool gzip = false;                                              // the file on disk starts with the gzip magic
    std::string inflater;                                           // which inflater ran on it (gzmem.h), for FL_CLI_TIMING
    bool open_plain(const std::string &path);
    // gzip: inflate the whole of [base, base + size) ONCE into memory (gzmem.h), give the compressed bytes back and carry
    // on as if it were a mapped plain file; the reference inflates it once per pass (main.cpp:70-75, 263-269). budget:
    // the most the inflated bytes may take (0: input_memory_budget()). false: *why says why, and the compressed bytes stay. device:
    // tried first on gzip that is not BGZF (gzmem.h).
    bool inflate(uint64_t budget, std::string *why, const GzipDeviceInflate &device = GzipDeviceInflate());
    // plain file, or gzip inflated into memory (unless FL_GZ_HOST is set); false: use the streaming host reader (*why:
    // why a gzip file was not inflated)
    bool open_any(const std::string &path, bool *inflated = nullptr, std::string *why = nullptr,
                  const GzipDeviceInflate &device = GzipDeviceInflate());
    // FL_TEXT_FASTQ, FL_TEXT_FASTA, FL_FORMAT_BAM (bam.h: an inflated input that starts with the BAM magic), or 0
    int format() const;
    MappedFile() = default;
    MappedFile(const MappedFile &) = delete;
    MappedFile &operator=(const MappedFile &) = delete;
    ~MappedFile();
};

struct Chunk { uint64_t begin, end; };

// The chunk size to cut at: default_bytes, or FL_CHUNK_MB MiB when it is set, within [1 MiB, 1 GiB]
uint64_t chunk_target(uint64_t default_bytes);

// record-aligned chunks of about `target` bytes; false if no boundary can be found (then the host parser runs)
bool plan_chunks(const char *b, uint64_t size, int format, uint64_t target, uint64_t max_chunk, std::vector<Chunk> &out);

// One step of plan_chunks over an input that is still arriving: the chunk that starts at `pos`, given the bytes [0, avail)
// so far (`ended`: no more will come). 1: *out is that chunk; 0: wait for more bytes (or, once ended, nothing is left);
// -1: no record start to cut at. A candidate cut is judged only once its record's four lines have arrived, so the chunks
// cut while the input arrives are the ones plan_chunks cuts from the whole of it.
int plan_next_chunk(const char *b, uint64_t avail, bool ended, int format, uint64_t target, uint64_t max_chunk, uint64_t pos, Chunk *out);

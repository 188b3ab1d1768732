// filtlong_b200/csrc/host/gzmem.h -- gzip input for the device-text feeder (SURVEY 8f-1).
//
// The reference reads .gz input through zlib's gzread inside kseq, one record at a time, and does so twice (reference
// src/main.cpp:70-125 and 263-313). The feeder wants the input as one byte range it can cut into record-aligned chunks
// and later write survivors from, so a gzip file is inflated ONCE into anonymous memory and then treated exactly like a
// mapped plain file (the parse, the duplicate check and pass 2 never see the difference):
//   * BGZF (bgzip: every member carries its compressed size in a 'BC' extra field and its inflated size in the
//     trailer): the members are located without inflating anything, the output size is known up front, and the
//     members are inflated in parallel by a few host threads, each straight into its final place;
//   * any other gzip file (one member, or several concatenated): the caller's device inflater when it takes the file,
//     else one thread, one z_stream, members back to back -- what gzread does, including "bytes after the last member
//     that do not start a gzip header are ignored".
// A file that is not gzip, is truncated or corrupt, or whose inflated size would not fit the memory budget (a share of
// MemAvailable) yields `false` and leaves nothing behind: the caller then runs the kseq-compatible host reader, which
// reports errors the way the reference does.
#pragma once
#include <cstdint>
#include <functional>
#include <string>

struct InflatedInput {
    char *base = nullptr;        // anonymous mapping holding the inflated bytes
    uint64_t size = 0;           // inflated bytes
    uint64_t reserved = 0;       // bytes of address space behind `base`
    int members = 0;             // gzip members inflated
    int threads = 1;             // host threads that inflated them
    bool bgzf = false;
    std::string inflater;        // which inflater ran, for FL_CLI_TIMING: empty for the host threads
    InflatedInput() = default;
    InflatedInput(const InflatedInput &) = delete;
    InflatedInput &operator=(const InflatedInput &) = delete;
    ~InflatedInput();
    void release();              // give the memory back
    char *take() {               // hand the mapping to a new owner (who munmap()s `reserved` bytes)
        char *p = base;
        base = nullptr;
        return p;
    }
};

// How much memory an input held in memory may take: 60 % of MemAvailable (0 when it cannot be told).
uint64_t input_memory_budget();

// An inflater tried before the host z_stream on a gzip file that is not BGZF (the CLI binds fl_gzip_inflate to its
// scoring context). It writes out[0, cap) and returns true only when out[0, r->n_out) is exactly what zlib inflates from
// data[0, n); false declines, and the host path then runs exactly as it would without it. r->note says what ran either
// way (FL_CLI_TIMING). This file never calls into the CUDA library itself.
struct GzipDeviceResult {
    uint64_t n_out = 0, members = 0;
    std::string note;
};
using GzipDeviceInflate = std::function<bool(const unsigned char *data, uint64_t n, char *out, uint64_t cap, GzipDeviceResult *r)>;

// `data`/`n`: the compressed file's bytes (e.g. a read-only mapping). max_threads <= 0: pick from the machine.
// budget_bytes == 0: input_memory_budget(). device: see GzipDeviceInflate (empty: the host path only).
bool inflate_gzip_memory(const unsigned char *data, uint64_t n, InflatedInput &out, int max_threads, uint64_t budget_bytes,
                         std::string *why, const GzipDeviceInflate &device = GzipDeviceInflate());

// filtlong_b200/csrc/host/bgzf_out.h -- `--bgzip`: the CLI's output compressed as BGZF on the GPU.
//
// The reference prints plain FASTQ / FASTA and its README pipes it through `gzip`. BgzfOut is an output sink with the
// interface of the CLI's other sinks (put / put_owned): the bytes are copied into pinned batches of whole 65,280-byte
// blocks, each batch is compressed by fl_bgzf_compress and the members are written to the descriptor in order. Filling
// the next batch (the caller's thread), compressing one (a compressor thread) and writing the one before (a writer
// thread) overlap. finish() writes the last batch and the EOF member. The context must not be used by anyone else
// until finish() returns, except by other BgzfOut: all of them in the process share one lock around fl_bgzf_compress, so
// two sinks on one context (stdout and `--failed` in one re-parse) compress one batch at a time, in turn, on the same
// GPU, while their fills and writes still overlap.
//
// BAM output (the BamOut options): the batches hold BAM bytes and a list of items (fl_bam_item): raw pieces of the
// stream (put) and children of records copied into the batch once (put_child), and the compressor thread builds the
// records on the device and compresses them there (fl_bam_writer), which holds back the last partial block, so that the
// members are cut every FL_BGZF_BLOCK bytes of the stream as they are for a stream put() whole.
#pragma once
#include <condition_variable>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../../include/filtlong_b200.h"

struct BamOut {
    uint64_t max_record;               // the largest record of the input: a batch holds at least one
    bool keep_mods;
};

class BgzfOut {
public:
    BgzfOut(fl_ctx *ctx, int fd, const BamOut *bam = nullptr);
    ~BgzfOut();                        // without finish(): stops the threads, writes no EOF member
    BgzfOut(const BgzfOut &) = delete;
    BgzfOut &operator=(const BgzfOut &) = delete;

    void put(const void *p, size_t n);
    void put_owned(std::string s) { put(s.data(), s.size()); }
    // BAM output only: the child [s, e) of the record at rec (bam.h), built on the device
    void put_child(const char *rec, int s, int e);
    // BAM output: children that kept modification tags, children of parents with invalid ones (after finish())
    const uint64_t *mods_counts() const { return counts_; }
    // Compresses and writes what is left, then the EOF member. False if a compression or a write failed.
    bool finish();
    // why a compression failed (empty when it was a write that failed)
    const std::string &error() const { return error_; }

private:
    static constexpr int NIN = 3, NOUT = 2;
    void submit();
    void compress_loop();
    void write_loop();
    void stop();
    void fail(const std::string &why);

    fl_ctx *ctx_;
    int fd_;
    uint64_t in_cap_ = 0, out_cap_ = 0;
    char *in_[NIN] = {nullptr, nullptr, nullptr};
    uint64_t in_len_[NIN] = {0, 0, 0};
    bool in_busy_[NIN] = {false, false, false};
    // BAM output
    bool bam_ = false, keep_mods_ = false;
    std::vector<fl_bam_item> items_[NIN];
    uint64_t out_bound_ = 0, out_limit_ = 0;        // the batch being filled: a bound on its records' bytes, and its limit
    const char *parent_ = nullptr;                  // the record copied last into the batch being filled
    uint64_t parent_at_ = 0;
    bool last_[NIN] = {false, false, false};
    fl_bam_writer *writer_bam_ = nullptr;
    uint64_t counts_[2] = {0, 0};
    char *out_[NOUT] = {nullptr, nullptr};
    uint64_t out_len_[NOUT] = {0, 0};
    bool out_busy_[NOUT] = {false, false};
    int fill_ = 0, next_out_ = 0;
    std::deque<int> to_compress_, to_write_;
    bool closing_ = false, compress_done_ = false, failed_ = false, finished_ = false;
    std::string error_;
    std::mutex m_;
    std::condition_variable cv_;
    std::thread compressor_, writer_;
};

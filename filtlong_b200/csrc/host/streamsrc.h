// filtlong_b200/csrc/host/streamsrc.h -- input reads that can be read only once: standard input ("-"), a FIFO, /dev/stdin
// on a pipe, /dev/fd/N from a shell's <(...). The reference opens its input twice (src/main.cpp:70 and :265), so on a
// pipe its second pass finds nothing. Here the stream is read ONCE into memory and the rest of the CLI works from there,
// as it does from an inflated gzip file (textsrc.h, gzmem.h):
//   * address space for the whole memory budget (input_memory_budget()) is reserved up front, so the bytes never move; one
//     reader thread read()s into it and publishes how many bytes have arrived;
//   * plain FASTQ / FASTA can be cut into chunks (plan_next_chunk) and scored while the rest still arrives;
//   * a stream that starts with the gzip magic (gzip, BGZF, BAM) is buffered whole, then inflated by inflate_gzip_memory
//     and the compressed bytes are given back. Compressed and inflated bytes both count against the budget.
// A stream larger than the budget is an error: there is no second pass to fall back to.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <string>
#include <thread>

#include "textsrc.h"

// `path` is a FIFO, a character device or a socket: something that can be read only once
bool is_stream_file(const std::string &path);
// The input reads `*path` names are a stream: "-" (unless standard input is a regular file), or a FIFO, a character
// device or a socket. "-" on a regular file becomes "/dev/stdin", which is then mapped like any named file.
bool stream_input(std::string *path);

class StreamInput {
public:
    // Opens `path` ("-": descriptor 0) and starts reading it. budget == 0: input_memory_budget(). Throws when the stream
    // cannot be opened or the memory cannot be reserved.
    void start(const std::string &path, uint64_t budget = 0);
    // Blocks until at least `need` bytes have arrived or the stream has ended; returns the bytes that have arrived, all at
    // base(). *ended: no more will come (broken(): because of an error, which finish() reports). One waiter at a time:
    // the reader wakes it only once `need` is reached, not at every read().
    uint64_t wait_for(uint64_t need, bool *ended);
    bool ended();
    bool broken();
    const char *base() const { return file_.base; }
    // Waits for the end of the stream and inflates a gzip stream. false: *why says what went wrong (the stream did not fit
    // in memory, could not be read, or is a damaged gzip stream). Then file() is the whole input, in memory (fd < 0).
    bool finish(std::string *why, const GzipDeviceInflate &device = GzipDeviceInflate());
    const MappedFile &file() const { return file_; }
    bool inflated() const { return inflated_; }
    uint64_t stream_bytes();                                    // bytes read from the stream so far (compressed, for gzip)
    // what the feeder reports under FL_CLI_TIMING: chunks scored, and how many of them before the stream ended
    std::atomic<size_t> chunks{0}, chunks_before_end{0};
    StreamInput() = default;
    StreamInput(const StreamInput &) = delete;
    StreamInput &operator=(const StreamInput &) = delete;
    ~StreamInput();

private:
    void read_all();
    std::string name_;
    int fd_ = -1, stop_[2] = {-1, -1};
    bool own_fd_ = false;
    char *buf_ = nullptr;               // the reservation the reader writes to (owned by file_ from start() on)
    uint64_t budget_ = 0;
    std::mutex m_;
    std::condition_variable cv_;
    uint64_t got_ = 0, need_ = 0;
    bool ended_ = false, overflow_ = false;
    int errno_ = 0;
    std::thread reader_;
    bool finished_ = false, finish_ok_ = false, inflated_ = false;
    std::string finish_why_;
    MappedFile file_;
};

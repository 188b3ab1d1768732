// filtlong_b200/csrc/host/fastx.h -- FASTA/FASTQ record reader (plain or gzip through zlib).
//
// Written from scratch to the parsing rules the reference gets from klib's kseq (reference
// src/kseq.h:161-224), because record boundaries, names, comments and the error codes are part of
// the drop-in surface (main.cpp:76-88, SURVEY 8f I/O KATs):
//   - a record starts at the next '>' or '@' character; the name runs to the first whitespace, the
//     comment is the rest of that line (one trailing '\r' dropped);
//   - sequence lines are concatenated until a line starts with '>', '@' or '+'; blank lines are
//     skipped and one trailing '\r' per line is dropped;
//   - after '+', the rest of that line is ignored and quality lines are concatenated until they
//     are at least as long as the sequence;
//   - next() returns the sequence length, or -1 at end of file, -2 for a truncated / mismatching
//     quality string, -3 on a stream error.
// One rule comes from the reference's use of kseq rather than kseq itself: `name` ends at its first NUL
// byte, because the reference only ever reads it as a C string. The comment, the sequence and the quality
// keep every byte (the reference scores seq.l bases); pass 2 prints them up to their first NUL.
#pragma once
#include <zlib.h>

#include <cstdint>
#include <memory>
#include <string>

class FastxReader {
public:
    explicit FastxReader(const std::string &path);
    // the same parser over bytes already in memory (a mapped plain file or an inflated gzip file, from any record
    // boundary on): what a device-text caller falls back to in the middle of a file
    FastxReader(const char *mem, uint64_t n_bytes);
    ~FastxReader();
    bool ok() const { return fp_ != nullptr || mem_ != nullptr; }
    int64_t next();
    std::string name, comment, seq, qual;
    bool is_fastq = false;

    // Where the last record sits in the (uncompressed) byte stream, for writers that want to copy
    // slices of the input instead of parsing it a second time (main.cpp:263-313 re-reads the file).
    // Valid after next() >= 0. `simple` says the sequence and the quality each came from exactly one
    // line with nothing stripped, i.e. input[seq_off, seq_off + length) IS the sequence (and likewise
    // for the name, the quality and the comment, none of which holds a NUL); otherwise the offsets
    // must not be used.
    bool simple = false;
    uint64_t name_off = 0, comment_off = 0, seq_off = 0, qual_off = 0;
    // true when the offsets are those of the bytes given: a file that is not compressed, or memory
    bool plain() const { return mem_ != nullptr || (fp_ && gzdirect(fp_) != 0); }

private:
    int getc();
    // appends the rest of the current line to s (without the newline); returns false at EOF with
    // nothing read
    bool get_line(std::string &s, bool append);
    int refill();                      // the next bytes of the stream into buf_: > 0 bytes, 0 at the end, < 0 on a stream error
    gzFile fp_ = nullptr;
    const char *mem_ = nullptr;
    uint64_t mem_n_ = 0, mem_pos_ = 0;
    static constexpr int kBuf = 1 << 16;
    unsigned char *buf_;
    int begin_ = 0, end_ = 0;
    uint64_t buf_base_ = 0;            // stream offset of buf_[0]
    bool stripped_cr_ = false;         // the last get_line dropped a '\r'
    uint64_t pos() const { return buf_base_ + (uint64_t)begin_; }
    bool eof_ = false, err_ = false;
    int last_char_ = 0;
};

// Where a FastxReader reads its records from: a file by its path (plain or gzip, streamed through zlib), or bytes already
// in memory. A path converts to one, so a caller that has only a path passes it as it is.
struct FastxInput {
    std::string path;
    const char *mem = nullptr;
    uint64_t n_bytes = 0;
    bool in_memory = false;
    FastxInput(const std::string &p) : path(p) {}
    FastxInput(const char *p) : path(p) {}
    FastxInput(const char *m, uint64_t n) : mem(m), n_bytes(n), in_memory(true) {}
    // a reader at the first record
    std::unique_ptr<FastxReader> open() const {
        return std::unique_ptr<FastxReader>(in_memory ? new FastxReader(mem, n_bytes) : new FastxReader(path));
    }
};

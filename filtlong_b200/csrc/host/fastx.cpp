// filtlong_b200/csrc/host/fastx.cpp -- see fastx.h
#include "fastx.h"

#include <cctype>
#include <cstring>

FastxReader::FastxReader(const std::string &path) : buf_(new unsigned char[kBuf]) { fp_ = gzopen(path.c_str(), "r"); }

FastxReader::FastxReader(const char *mem, uint64_t n_bytes) : mem_(mem), mem_n_(n_bytes), buf_(new unsigned char[kBuf]) {}

int FastxReader::refill() {
    if (!mem_) return gzread(fp_, buf_, kBuf);
    const uint64_t left = mem_n_ - mem_pos_;
    const int n = left < (uint64_t)kBuf ? (int)left : kBuf;
    memcpy(buf_, mem_ + mem_pos_, (size_t)n);
    mem_pos_ += (uint64_t)n;
    return n;
}

FastxReader::~FastxReader() {
    if (fp_) gzclose(fp_);
    delete[] buf_;
}

// pass 2 prints the comment, the sequence and the quality as C strings (main.cpp:273-305): a record with a NUL is
// not a slice of the input
static bool has_nul(const std::string &s) { return !s.empty() && memchr(s.data(), 0, s.size()) != nullptr; }

int FastxReader::getc() {
    if (err_) return -3;
    if (eof_ && begin_ >= end_) return -1;
    if (begin_ >= end_) {
        buf_base_ += (uint64_t)end_;
        begin_ = 0;
        end_ = refill();
        if (end_ == 0) { eof_ = true; return -1; }
        if (end_ < 0) { eof_ = true; err_ = true; end_ = 0; return -3; }
    }
    return (int)buf_[begin_++];
}

bool FastxReader::get_line(std::string &s, bool append) {
    bool gotany = false;
    if (!append) s.clear();
    for (;;) {
        if (err_) return false;
        if (begin_ >= end_) {
            if (eof_) break;
            buf_base_ += (uint64_t)end_;
            begin_ = 0;
            end_ = refill();
            if (end_ == 0) { eof_ = true; break; }
            if (end_ < 0) { eof_ = true; err_ = true; end_ = 0; return false; }
        }
        const unsigned char *nl = (const unsigned char *)memchr(buf_ + begin_, '\n', end_ - begin_);
        int i = nl ? (int)(nl - buf_) : end_;
        gotany = true;
        s.append((const char *)buf_ + begin_, i - begin_);
        begin_ = i + 1;
        if (i < end_) break;   // newline consumed
    }
    if (!gotany && eof_) return false;
    stripped_cr_ = false;
    if (s.size() > 1 && s.back() == '\r') { s.pop_back(); stripped_cr_ = true; }
    return true;
}

int64_t FastxReader::next() {
    int c;
    if (last_char_ == 0) {
        while ((c = getc()) >= 0 && c != '>' && c != '@') {}
        if (c < 0) return c;
        last_char_ = c;
    }
    comment.clear();
    seq.clear();
    qual.clear();
    // name: up to the first whitespace character
    name.clear();
    name_off = pos();
    bool got = false;
    for (;;) {
        c = getc();
        if (c < 0) break;
        got = true;
        if (isspace(c)) break;
        name.push_back((char)c);
    }
    if (!got) return c == -3 ? -3 : -1;
    simple = true;
    // the reference uses the name only as a C string (main.cpp:81,90,99,114,268,273): it ends at the first NUL
    const size_t nul = name.find('\0');
    if (nul != std::string::npos) {
        name.resize(nul);
        simple = false;
    }
    comment_off = pos();
    if (c >= 0 && c != '\n') {
        get_line(comment, false);
        if (stripped_cr_) simple = false;
    }
    int seq_lines = 0;
    while ((c = getc()) >= 0 && c != '>' && c != '+' && c != '@') {
        if (c == '\n') continue;
        if (seq_lines++ == 0) seq_off = pos() - 1;
        seq.push_back((char)c);
        get_line(seq, true);
        if (stripped_cr_) simple = false;
    }
    if (seq_lines != 1) simple = false;
    if (c == '>' || c == '@') last_char_ = c;
    is_fastq = (c == '+');
    if (!is_fastq) {
        if (c != '>' && c != '@') last_char_ = 0;   // end of file
        if (has_nul(comment) || has_nul(seq)) simple = false;
        return (int64_t)seq.size();
    }
    while ((c = getc()) >= 0 && c != '\n') {}
    if (c == -1) return -2;
    qual_off = pos();
    int qual_lines = 0;
    while (get_line(qual, true)) {
        ++qual_lines;
        if (stripped_cr_) simple = false;
        if (qual.size() >= seq.size()) break;
    }
    if (qual_lines != 1) simple = false;
    // a stream error while reading the quality string: kseq's operator precedence (kseq.h:213-216) reports it as a
    // truncated quality string (-2, "incorrect FASTQ format"), not as -3; same here
    if (err_) return -2;
    last_char_ = 0;
    if (seq.size() != qual.size()) return -2;
    if (has_nul(comment) || has_nul(seq) || has_nul(qual)) simple = false;
    return (int64_t)seq.size();
}

// filtlong_b200/csrc/host/bgzf_out.cpp -- see bgzf_out.h.
#include "bgzf_out.h"

#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <stdexcept>

#include "bam.h"

namespace {

// the empty member that ends a BGZF file (SAM specification 4.1.2)
const unsigned char kEof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};

// held around every fl_bgzf_compress call of every BgzfOut: a context takes one host thread at a time, and the re-parse
// path of pass 2 runs two BgzfOut (stdout and --failed) on one context
std::mutex g_compress;

bool write_all(int fd, const char *p, uint64_t n) {
    while (n) {
        const ssize_t w = write(fd, p, (size_t)n);
        if (w <= 0) return false;
        p += w;
        n -= (uint64_t)w;
    }
    return true;
}

}  // namespace

BgzfOut::BgzfOut(fl_ctx *ctx, int fd, const BamOut *bam) : ctx_(ctx), fd_(fd) {
    in_cap_ = 1028ull * FL_BGZF_BLOCK;                     // 64 MiB of input per batch
    out_cap_ = fl_bgzf_bound(in_cap_);
    if (bam) {
        // a child's record is smaller than its parent's plus 300 bytes (a longer name, MN:I), so one fits any batch
        bam_ = true;
        keep_mods_ = bam->keep_mods;
        in_cap_ = std::max<uint64_t>(in_cap_, bam->max_record + 16);
        out_limit_ = in_cap_ + (1u << 20);
        out_cap_ = fl_bgzf_bound(out_limit_ + FL_BGZF_BLOCK);
        if (fl_bam_writer_create(ctx_, &writer_bam_) != FL_OK) throw std::runtime_error(std::string("fl_bam_writer_create: ") + fl_last_error(ctx_));
    }
    for (int i = 0; i < NIN; ++i) {
        void *p = nullptr;
        if (fl_host_alloc(in_cap_, &p) != FL_OK) { stop(); throw std::runtime_error("--bgzip: cannot allocate pinned host memory"); }
        in_[i] = (char *)p;
    }
    for (int i = 0; i < NOUT; ++i) {
        void *p = nullptr;
        if (fl_host_alloc(out_cap_, &p) != FL_OK) { stop(); throw std::runtime_error("--bgzip: cannot allocate pinned host memory"); }
        out_[i] = (char *)p;
    }
    in_busy_[0] = true;                                    // the batch being filled
    compressor_ = std::thread([this] { compress_loop(); });
    writer_ = std::thread([this] { write_loop(); });
}

BgzfOut::~BgzfOut() { stop(); }

// why: empty for a failed write, which the caller reports like one of plain output (by its exit code only)
void BgzfOut::fail(const std::string &why) {
    if (!failed_) error_ = why;
    failed_ = true;
}

void BgzfOut::put(const void *p, size_t n) {
    const char *s = (const char *)p;
    while (bam_ && n) {                                    // raw items, at most 1 GiB each
        uint64_t k = std::min<uint64_t>({n, in_cap_ - in_len_[fill_], out_limit_ - out_bound_, 1ull << 30});
        if (k == 0) { submit(); continue; }
        items_[fill_].push_back(fl_bam_item{in_len_[fill_], -1, (int32_t)k});
        memcpy(in_[fill_] + in_len_[fill_], s, (size_t)k);
        in_len_[fill_] += k;
        out_bound_ += k;
        s += k;
        n -= (size_t)k;
    }
    while (n) {
        const uint64_t k = std::min<uint64_t>(n, in_cap_ - in_len_[fill_]);
        memcpy(in_[fill_] + in_len_[fill_], s, (size_t)k);
        in_len_[fill_] += k;
        s += k;
        n -= (size_t)k;
        if (in_len_[fill_] == in_cap_) submit();
    }
}

void BgzfOut::put_child(const char *rec, int s, int e) {
    if (!bam_) throw std::logic_error("BgzfOut::put_child on an output that is not BAM");
    const uint64_t rb = bam_record_bytes(rec), n = (uint64_t)(e - s);
    const uint64_t bound = rb - (uint64_t)bam_l_seq(rec) * 3 / 2 + n + n / 2 + 300;
    if (out_bound_ + bound > out_limit_) submit();
    if (rec != parent_) {
        if (in_len_[fill_] + rb > in_cap_) submit();
        parent_at_ = in_len_[fill_];
        memcpy(in_[fill_] + parent_at_, rec, (size_t)rb);
        in_len_[fill_] += rb;
        parent_ = rec;
    }
    items_[fill_].push_back(fl_bam_item{parent_at_, s, e});
    out_bound_ += bound;
}

// hands the batch being filled to the compressor and waits for a free one
void BgzfOut::submit() {
    std::unique_lock<std::mutex> lk(m_);
    to_compress_.push_back(fill_);
    cv_.notify_all();
    const int next = (fill_ + 1) % NIN;
    cv_.wait(lk, [&] { return !in_busy_[next]; });
    fill_ = next;
    in_busy_[fill_] = true;
    in_len_[fill_] = 0;
    items_[fill_].clear();
    last_[fill_] = false;
    out_bound_ = 0;
    parent_ = nullptr;
}

void BgzfOut::compress_loop() {
    for (;;) {
        int i, o;
        {
            std::unique_lock<std::mutex> lk(m_);
            cv_.wait(lk, [&] { return !to_compress_.empty() || closing_; });
            if (to_compress_.empty()) break;
            i = to_compress_.front();
            to_compress_.pop_front();
            o = next_out_;
            next_out_ = (next_out_ + 1) % NOUT;
            cv_.wait(lk, [&] { return !out_busy_[o]; });
            out_busy_[o] = true;
        }
        uint64_t n = 0;
        bool ok;
        {
            std::lock_guard<std::mutex> lk(m_);
            ok = !failed_;
        }
        if (ok) {
            std::unique_lock<std::mutex> gl(g_compress);
            const int rc = bam_ ? fl_bam_writer_push(writer_bam_, in_[i], in_len_[i], items_[i].data(), items_[i].size(), keep_mods_, last_[i],
                                                     out_[o], out_cap_, &n, counts_)
                                : fl_bgzf_compress(ctx_, in_[i], in_len_[i], out_[o], out_cap_, 0, &n);
            if (rc != FL_OK) {
                const std::string why = bam_ ? std::string(fl_last_error(ctx_)) : std::string("fl_bgzf_compress: ") + fl_last_error(ctx_);
                gl.unlock();
                std::lock_guard<std::mutex> lk(m_);
                fail(why);
                ok = false;
            }
        }
        std::lock_guard<std::mutex> lk(m_);
        in_busy_[i] = false;
        out_len_[o] = ok ? n : 0;
        to_write_.push_back(o);
        cv_.notify_all();
    }
    std::lock_guard<std::mutex> lk(m_);
    compress_done_ = true;
    cv_.notify_all();
}

void BgzfOut::write_loop() {
    for (;;) {
        int o;
        bool ok;
        {
            std::unique_lock<std::mutex> lk(m_);
            cv_.wait(lk, [&] { return !to_write_.empty() || compress_done_; });
            if (to_write_.empty()) break;
            o = to_write_.front();
            to_write_.pop_front();
            ok = !failed_;
        }
        if (ok && !write_all(fd_, out_[o], out_len_[o])) {
            std::lock_guard<std::mutex> lk(m_);
            fail("");
        }
        std::lock_guard<std::mutex> lk(m_);
        out_busy_[o] = false;
        cv_.notify_all();
    }
}

void BgzfOut::stop() {
    {
        std::lock_guard<std::mutex> lk(m_);
        closing_ = true;
        cv_.notify_all();
    }
    if (compressor_.joinable()) compressor_.join();
    if (writer_.joinable()) writer_.join();
    for (int i = 0; i < NIN; ++i) if (in_[i]) { fl_host_free(in_[i]); in_[i] = nullptr; }
    for (int i = 0; i < NOUT; ++i) if (out_[i]) { fl_host_free(out_[i]); out_[i] = nullptr; }
    if (writer_bam_) { fl_bam_writer_destroy(writer_bam_); writer_bam_ = nullptr; }
}

bool BgzfOut::finish() {
    if (finished_) return !failed_;
    finished_ = true;
    if (in_len_[fill_] || bam_) {                          // BAM: the last batch also compresses the bytes held back
        std::lock_guard<std::mutex> lk(m_);
        last_[fill_] = true;
        to_compress_.push_back(fill_);
        cv_.notify_all();
    }
    stop();
    if (!failed_ && !write_all(fd_, (const char *)kEof, sizeof kEof)) fail("");
    return !failed_;
}

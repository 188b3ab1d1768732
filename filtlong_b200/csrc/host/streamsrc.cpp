// filtlong_b200/csrc/host/streamsrc.cpp -- see streamsrc.h.
#include "streamsrc.h"

#include <errno.h>
#include <fcntl.h>
#include <poll.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <stdexcept>

#include "gzmem.h"

bool is_stream_file(const std::string &path) {
    struct stat st;
    return stat(path.c_str(), &st) == 0 && (S_ISFIFO(st.st_mode) || S_ISCHR(st.st_mode) || S_ISSOCK(st.st_mode));
}

bool stream_input(std::string *path) {
    struct stat st;
    if (*path == "-") {
        if (fstat(0, &st) == 0 && S_ISREG(st.st_mode)) {
            *path = "/dev/stdin";
            return false;
        }
        return true;
    }
    return is_stream_file(*path);
}

void StreamInput::start(const std::string &path, uint64_t budget) {
    name_ = path == "-" || path == "/dev/stdin" ? "standard input" : path;
    budget_ = budget ? budget : input_memory_budget();
    if (budget_ == 0) throw std::runtime_error("cannot tell how much memory is available to hold " + name_);
    const uint64_t pg = (uint64_t)sysconf(_SC_PAGESIZE), reserved = (budget_ + pg - 1) / pg * pg;
    void *p = mmap(nullptr, (size_t)reserved, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (p == MAP_FAILED) throw std::runtime_error("cannot reserve memory to hold " + name_);
    madvise(p, (size_t)reserved, MADV_HUGEPAGE);                      // fewer faults while the reader writes; a hint only
    buf_ = (char *)p;
    file_.base = buf_;
    file_.map_bytes = reserved;
    if (path == "-") fd_ = 0;
    else {
        fd_ = ::open(path.c_str(), O_RDONLY | O_CLOEXEC);
        if (fd_ < 0) throw std::runtime_error("cannot open " + path + ": " + strerror(errno));
        own_fd_ = true;
    }
    struct stat st;
    if (fstat(fd_, &st) == 0 && S_ISFIFO(st.st_mode)) (void)fcntl(fd_, F_SETPIPE_SZ, 1 << 20);   // fewer, larger reads; a hint only
    if (pipe2(stop_, O_CLOEXEC) != 0) throw std::runtime_error(std::string("pipe2: ") + strerror(errno));
    reader_ = std::thread([this] { read_all(); });
}

// read() into the reservation until the end of the stream, an error, the budget, or a stop from the destructor
void StreamInput::read_all() {
    const uint64_t piece = 4ull << 20;
    uint64_t n = 0;
    bool overflow = false;
    int err = 0;
    for (;;) {
        struct pollfd pf[2] = {{fd_, POLLIN, 0}, {stop_[0], POLLIN, 0}};
        if (poll(pf, 2, -1) < 0) {
            if (errno == EINTR) continue;
            err = errno;
            break;
        }
        if (pf[1].revents) { err = ECANCELED; break; }
        ssize_t r;
        if (n < budget_) {
            r = read(fd_, buf_ + n, (size_t)std::min(piece, budget_ - n));
        } else {                                                       // full: is there more?
            char c;
            r = read(fd_, &c, 1);
            if (r > 0) { overflow = true; break; }
        }
        if (r < 0) {
            if (errno == EINTR || errno == EAGAIN) continue;
            err = errno;
            break;
        }
        if (r == 0) break;
        n += (uint64_t)r;
        bool wake;
        {
            std::lock_guard<std::mutex> lk(m_);
            got_ = n;
            wake = need_ && n >= need_;
        }
        if (wake) cv_.notify_all();
    }
    {
        std::lock_guard<std::mutex> lk(m_);
        got_ = n;
        ended_ = true;
        overflow_ = overflow;
        errno_ = err;
    }
    cv_.notify_all();
}

uint64_t StreamInput::wait_for(uint64_t need, bool *ended) {
    std::unique_lock<std::mutex> lk(m_);
    need_ = need;
    cv_.wait(lk, [&] { return got_ >= need || ended_; });
    need_ = 0;
    *ended = ended_;
    return got_;
}

bool StreamInput::ended() {
    std::lock_guard<std::mutex> lk(m_);
    return ended_;
}

bool StreamInput::broken() {
    std::lock_guard<std::mutex> lk(m_);
    return ended_ && (overflow_ || errno_ != 0);
}

uint64_t StreamInput::stream_bytes() {
    std::lock_guard<std::mutex> lk(m_);
    return got_;
}

bool StreamInput::finish(std::string *why, const GzipDeviceInflate &device) {
    if (!finished_) {
        finished_ = true;
        if (reader_.joinable()) reader_.join();
        const uint64_t n = file_.size = got_;
        file_.gzip = n >= 2 && (unsigned char)buf_[0] == 0x1f && (unsigned char)buf_[1] == 0x8b;
        std::string &w = finish_why_;
        if (overflow_) {
            w = name_ + " did not fit in memory (more than " + std::to_string(budget_) + " bytes; the limit is 60 % of MemAvailable)";
        } else if (errno_) {
            w = "cannot read " + name_ + ": " + strerror(errno_);
        } else if (file_.gzip) {
            std::string iw;
            if (n >= budget_) {
                w = name_ + " did not fit in memory once inflated";
            } else if (file_.inflate(budget_ - n, &iw, device)) {
                buf_ = nullptr;                                        // file_ gave the compressed bytes back
                inflated_ = true;
                finish_ok_ = true;
            } else if (iw == "empty input") {                          // like an empty file
                file_.size = 0;
                finish_ok_ = true;
            } else {
                w = name_ + ": " + iw;
            }
        } else {
            finish_ok_ = true;
        }
    }
    if (!finish_ok_ && why) *why = finish_why_;
    return finish_ok_;
}

StreamInput::~StreamInput() {
    if (reader_.joinable()) {                                          // an early way out: stop reading, whatever is left
        if (stop_[1] >= 0) (void)!write(stop_[1], "x", 1);
        reader_.join();
    }
    if (stop_[0] >= 0) close(stop_[0]);
    if (stop_[1] >= 0) close(stop_[1]);
    if (own_fd_) close(fd_);
}

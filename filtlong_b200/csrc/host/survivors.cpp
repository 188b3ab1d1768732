// filtlong_b200/csrc/host/survivors.cpp -- see survivors.h.
#include "survivors.h"

#include <fcntl.h>
#include <sys/stat.h>
#include <sys/uio.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <memory>
#include <thread>

#include "bam.h"
#include "bgzf_out.h"
#include "fastx.h"
#include "misc.h"

bool Records::within(uint64_t file_size, bool quality) const {
    for (size_t i = 0; i < n; ++i) {
        const uint64_t L = (uint64_t)len[i];
        if (name_off[i] + name_len[i] + 1 + comment_len[i] > file_size || seq_off[i] + L > file_size ||
            (quality && qual_off[i] + L > file_size))
            return false;
    }
    return true;
}

bool NameIndex::build(const std::vector<const Records *> &tables, const char *base, std::string *dup) {
    tables_ = tables;
    base_ = base;
    size_t n = 0;
    for (const Records *t : tables) n += t->n;
    size_t cap = 16;
    while (cap < 2 * n + 16) cap <<= 1;
    keys_.assign(cap, 0);
    at_.assign(cap, 0);
    mask_ = cap - 1;
    for (size_t t = 0; t < tables.size(); ++t) {
        const Records &R = *tables[t];
        for (size_t i = 0; i < R.n; ++i) {
            const uint64_t h = R.name_hash[i];
            size_t slot = (size_t)(h * 0x9E3779B97F4A7C15ull) & mask_;
            for (; at_[slot]; slot = (slot + 1) & mask_) {
                if (keys_[slot] != h) continue;
                const Records &O = *tables[(at_[slot] - 1) >> 56];
                const uint64_t j = (at_[slot] - 1) & ((1ull << 56) - 1);
                if (O.name_len[j] == R.name_len[i] && memcmp(base + O.name_off[j], base + R.name_off[i], R.name_len[i]) == 0) {
                    dup->assign(base + R.name_off[i], R.name_len[i]);
                    return false;
                }
            }
            keys_[slot] = h;
            at_[slot] = ((uint64_t)t << 56 | i) + 1;
        }
    }
    return true;
}

bool NameIndex::find(uint64_t h, const char *name, uint32_t len, int32_t *table, uint64_t *index) const {
    for (size_t slot = (size_t)(h * 0x9E3779B97F4A7C15ull) & mask_; at_[slot]; slot = (slot + 1) & mask_) {
        if (keys_[slot] != h) continue;
        const uint64_t t = (at_[slot] - 1) >> 56, i = (at_[slot] - 1) & ((1ull << 56) - 1);
        const Records &R = *tables_[t];
        if (R.name_len[i] == len && memcmp(base_ + R.name_off[i], name, len) == 0) {
            *table = (int32_t)t;
            *index = i;
            return true;
        }
    }
    return false;
}

namespace {

struct RecordText {               // one input record's bytes
    const char *name;
    size_t name_len;
    const char *comment;
    size_t comment_len;
    const char *seq, *qual;
    size_t len;
    bool lead_before_name;        // name[-1] is the format's lead character
    // The reference prints the comment when it has any byte, but prints it, the sequence and the quality as C strings
    // (main.cpp:274-305). These are the printed lengths: up to the first NUL (all of it when there is none).
    bool has_comment;
    size_t comment_print, seq_print, qual_print;
};

RecordText text_of(const Records &R, const char *base, size_t i) {
    const char *name = base + R.name_off[i];
    const size_t L = (size_t)R.len[i], C = R.comment_len[i];
    return RecordText{name, R.name_len[i], name + R.name_len[i] + 1, C, base + R.seq_off[i], base + R.qual_off[i], L, R.lead_checked,
                      C > 0, C, L, L};
}

// bytes [start, start + length) of a C string of n bytes, as std::string(s).substr(start, length) gives them. Past its
// end the reference's substr throws; here nothing is printed (DESIGN 5).
size_t c_substr(size_t n, size_t start, size_t length) { return start >= n ? 0 : std::min(length, n - start); }

// Read i's output: the read if its pass flag is `want` and it has no children, else each child longer than 0 whose flag
// is `want` (stdout: the survivors, want = true; --failed: the rest, want = false). put()'s bytes must stay valid until
// the sink is flushed; put_owned() keeps its string alive until then.
template <class Sink>
void emit_survivors(Sink &sink, const Format &fmt, const RecordText &r, const Results &res, size_t i, bool want) {
    auto pass = [&](size_t row) { return (res.row_pfinal[row] != 0) == want; };
    if (fmt.bam) {                                                        // the record as it is, or new ones for the children
        const char *rec = bam_record_of(r.name);
        const size_t rs = (size_t)res.row_start[i];
        if (res.n_child[i] == 0) {
            if (pass(rs)) sink.put(rec, bam_record_bytes(rec));
            return;
        }
        for (size_t row = rs; row < rs + (size_t)res.n_child[i]; ++row) {
            const int start = res.row_s[row], end = res.row_e[row];
            if (!pass(row) || end - start <= 0 || (size_t)end > r.len) continue;
            sink.put_child(rec, start, end);
        }
        return;
    }
    const char *lead = fmt.lead == '>' ? ">" : "@";
    auto rest = [&](size_t start, size_t length) {
        if (r.has_comment) { sink.put(" ", 1); sink.put(r.comment, r.comment_print); }
        sink.put("\n", 1);
        sink.put(r.seq + start, c_substr(r.seq_print, start, length));
        sink.put("\n", 1);
        if (fmt.quality) { sink.put("+\n", 2); sink.put(r.qual + start, c_substr(r.qual_print, start, length)); sink.put("\n", 1); }
    };
    const size_t rs = (size_t)res.row_start[i];
    if (res.n_child[i] == 0) {
        if (!pass(rs)) return;
        if (r.lead_before_name) sink.put(r.name - 1, 1 + r.name_len);
        else { sink.put(lead, 1); sink.put(r.name, r.name_len); }
        rest(0, r.len);
        return;
    }
    for (size_t row = rs; row < rs + (size_t)res.n_child[i]; ++row) {
        const int start = res.row_s[row], end = res.row_e[row];
        // (a row past the record's end can only come from an input that changed since pass 1)
        if (!pass(row) || end - start <= 0 || (size_t)end > r.len) continue;
        std::string nm(lead, 1);
        append_child_name(nm, r.name, r.name_len, start, end);
        sink.put_owned(std::move(nm));
        rest((size_t)start, (size_t)(end - start));
    }
}

// Reads [lo, hi) of part pi. BAM --aligned: with each read, in file order, the followers just before it, and after the
// part's last read those after it; a follower is written when its read's pass flag is `want`, an orphan when want is
// false.
template <class Sink>
void emit_range(Sink &sink, const char *base, const std::vector<Part> &parts, size_t pi, size_t lo, size_t hi, const Format &fmt, bool want) {
    const Part &p = parts[pi];
    if (!p.followers) {
        for (size_t i = lo; i < hi; ++i) emit_survivors(sink, fmt, text_of(*p.rec, base, i), p.res, i, want);
        return;
    }
    const std::vector<Follower> &F = *p.followers;
    auto f = std::lower_bound(F.begin(), F.end(), lo, [](const Follower &x, size_t i) { return x.before < i; });
    const bool last = hi == p.rec->n;                                   // the part's last range also takes those after its reads
    for (size_t i = lo; i < hi || (last && i == hi); ++i) {
        for (; f != F.end() && f->before == i; ++f) {
            bool kept = false;
            if (f->owner_part >= 0) {
                const Results &r = parts[(size_t)f->owner_part].res;
                kept = r.row_pfinal[r.row_start[f->owner]] != 0;
            }
            if (kept == want) sink.put(base + f->off, bam_record_bytes(base + f->off));
        }
        if (i < hi) emit_survivors(sink, fmt, text_of(*p.rec, base, i), p.res, i, want);
    }
}

// the host sinks build a child's BAM record with bam_child_record
struct HostChildren {
    bool keep_mods = false;
    uint64_t counts[2] = {0, 0};
    std::string child(const char *rec, int s, int e) {
        std::string c;
        const int st = bam_child_record(rec, s, e, c, keep_mods);
        if (st) ++counts[st == FL_BAM_MODS_KEPT ? 0 : 1];
        return c;
    }
};

// iovecs into the mapping, written with writev()
struct Writer : HostChildren {
    static constexpr int MAXV = 1000;
    int fd;
    struct iovec v[MAXV];
    int nv = 0;
    std::vector<std::string> small;            // child names: must stay alive (and in place: short strings live inside the object) until the flush
    bool failed = false;
    explicit Writer(int f) : fd(f) { small.reserve(256); }
    void flush() {
        int done = 0;
        while (done < nv && !failed) {
            ssize_t w = writev(fd, v + done, nv - done);
            if (w < 0) { failed = true; break; }
            while (done < nv && (size_t)w >= v[done].iov_len) { w -= (ssize_t)v[done].iov_len; ++done; }
            if (done < nv && w > 0) { v[done].iov_base = (char *)v[done].iov_base + w; v[done].iov_len -= (size_t)w; }
        }
        nv = 0;
        small.clear();
    }
    void put(const void *p, size_t n) {
        if (n == 0) return;
        if (nv == MAXV) flush();
        v[nv].iov_base = const_cast<void *>(p);
        v[nv].iov_len = n;
        ++nv;
    }
    void put_owned(std::string s) {
        if (nv == MAXV || small.size() >= 200) flush();
        small.push_back(std::move(s));
        put(small.back().data(), small.back().size());
    }
    void put_child(const char *rec, int s, int e) { put_owned(child(rec, s, e)); }
};

struct Sizer : HostChildren {
    uint64_t n = 0;
    void put(const void *, size_t k) { n += k; }
    void put_owned(std::string s) { n += s.size(); }
    void put_child(const char *rec, int s, int e) { n += child(rec, s, e).size(); }
};

// copies into a buffer of about 8 MiB; flush() writes it with pwrite() at `pos`, or with write() when pos < 0
struct Copier : HostChildren {
    int fd;
    int64_t pos;
    std::string buf;
    bool failed = false;
    Copier(int f, int64_t p) : fd(f), pos(p) { buf.reserve((8u << 20) + (2u << 20)); }
    void flush() {
        size_t done = 0;
        while (done < buf.size() && !failed) {
            const ssize_t w = pos < 0 ? write(fd, buf.data() + done, buf.size() - done)
                                      : pwrite(fd, buf.data() + done, buf.size() - done, (off_t)(pos + (int64_t)done));
            if (w <= 0) { failed = true; break; }
            done += (size_t)w;
        }
        if (pos >= 0) pos += (int64_t)buf.size();
        buf.clear();
    }
    void put(const void *p, size_t k) { buf.append((const char *)p, k); if (buf.size() >= (8u << 20)) flush(); }
    void put_owned(std::string s) { put(s.data(), s.size()); }
    void put_child(const char *rec, int s, int e) { put_owned(child(rec, s, e)); }
};

bool finish(BgzfOut &z) {
    if (z.finish()) return true;
    if (!z.error().empty()) std::cerr << "Error: " << z.error() << "\n";
    return false;
}

}  // namespace

bool write_survivors_writev(int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, bool want) {
    Writer w(fd);
    for (size_t pi = 0; pi < parts.size(); ++pi) emit_range(w, base, parts, pi, 0, parts[pi].rec->n, fmt, want);
    w.flush();
    return !w.failed;
}

// contiguous groups of reads are sized, then written with pwrite() by a few threads
bool write_survivors_pwrite(int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, bool want) {
    struct Group { size_t part, lo, hi; uint64_t bytes = 0, at = 0; };
    std::vector<Group> groups;
    size_t n_reads = 0;
    for (const Part &p : parts) n_reads += p.rec->n;
    const size_t per = n_reads / 32 + 1;
    for (size_t pi = 0; pi < parts.size(); ++pi)
        for (size_t lo = 0; lo < parts[pi].rec->n; lo += per) groups.push_back(Group{pi, lo, std::min(lo + per, parts[pi].rec->n), 0, 0});
    const off_t base_pos = lseek(fd, 0, SEEK_CUR);
    auto work = [&](bool write_pass) {
        std::vector<std::thread> ts;
        std::atomic<size_t> next(0);
        std::atomic<bool> bad(false);
        const unsigned nt = std::min<size_t>(8, groups.size());
        for (unsigned t = 0; t < nt; ++t)
            ts.emplace_back([&] {
                for (size_t g = next.fetch_add(1); g < groups.size(); g = next.fetch_add(1)) {
                    Group &G = groups[g];
                    if (!write_pass) {
                        Sizer z;
                        emit_range(z, base, parts, G.part, G.lo, G.hi, fmt, want);
                        G.bytes = z.n;
                    } else {
                        Copier c(fd, (int64_t)base_pos + (int64_t)G.at);
                        emit_range(c, base, parts, G.part, G.lo, G.hi, fmt, want);
                        c.flush();
                        if (c.failed) bad.store(true);
                    }
                }
            });
        for (auto &t : ts) t.join();
        return !bad.load();
    };
    work(false);
    uint64_t total_out = 0;
    for (auto &G : groups) { G.at = total_out; total_out += G.bytes; }
    if (base_pos < 0 || !work(true)) return false;
    return lseek(fd, base_pos + (off_t)total_out, SEEK_SET) >= 0;
}

bool write_survivors(int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, fl_ctx *bgzf, bool want,
                     uint64_t *mods_counts) {
    fflush(stdout);
    if (bgzf) {
        // compressed offsets are not known in advance: pipe or file, the members are written in order
        const BamOut bam{fmt.bam_max_record, fmt.keep_mods};
        BgzfOut z(bgzf, fd, fmt.bam ? &bam : nullptr);
        if (fmt.bam) z.put(base, (size_t)fmt.bam_header);
        for (size_t pi = 0; pi < parts.size(); ++pi) emit_range(z, base, parts, pi, 0, parts[pi].rec->n, fmt, want);
        const bool ok = finish(z);
        if (mods_counts) { mods_counts[0] = z.mods_counts()[0]; mods_counts[1] = z.mods_counts()[1]; }
        return ok;
    }
    if (fmt.bam) {
        Copier c(fd, -1);
        c.keep_mods = fmt.keep_mods;
        c.put(base, (size_t)fmt.bam_header);
        for (size_t pi = 0; pi < parts.size(); ++pi) emit_range(c, base, parts, pi, 0, parts[pi].rec->n, fmt, want);
        c.flush();
        if (mods_counts) { mods_counts[0] = c.counts[0]; mods_counts[1] = c.counts[1]; }
        return !c.failed;
    }
    struct stat st;
    const int flags = fcntl(fd, F_GETFL);
    if (fstat(fd, &st) == 0 && S_ISREG(st.st_mode) && flags >= 0 && !(flags & O_APPEND))
        return write_survivors_pwrite(fd, base, parts, fmt, want);
    return write_survivors_writev(fd, base, parts, fmt, want);
}

bool write_outputs(const Arguments &args, int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, fl_ctx *bgzf) {
    uint64_t mods[2] = {0, 0};
    bool ok = write_survivors(fd, base, parts, fmt, bgzf, true, mods);
    if (args.failed_fd >= 0 && !report_failed_write(args, write_survivors(args.failed_fd, base, parts, fmt, bgzf, false))) ok = false;
    if (fmt.keep_mods)
        std::cerr << "  modification tags: re-based on " << int_to_string((long long)mods[0]) << " child reads, dropped from "
                  << int_to_string((long long)mods[1]) << " whose parent's MM/ML/MN tags are invalid\n";
    return ok;
}

// One walk over the input feeds both outputs: stdout's sink, and failed's when there is one (a null pointer otherwise)
bool reparse_survivors(int fd, const FastxInput &input, const Results &res, size_t n_reads, const Format &fmt, fl_ctx *bgzf,
                       int failed_fd, bool *failed_ok) {
    const std::unique_ptr<FastxReader> reader = input.open();
    FastxReader &in = *reader;
    fflush(stdout);
    auto run = [&](auto &sink, auto *failed) {
        for (size_t i = 0; in.ok() && in.next() >= 0 && i < n_reads; ++i) {
            const RecordText r{in.name.data(), in.name.size(), in.comment.data(), in.comment.size(), in.seq.data(), in.qual.data(),
                               in.seq.size(), false, !in.comment.empty(), strnlen(in.comment.data(), in.comment.size()),
                               strnlen(in.seq.data(), in.seq.size()), strnlen(in.qual.data(), in.qual.size())};
            emit_survivors(sink, fmt, r, res, i, true);
            if (failed) emit_survivors(*failed, fmt, r, res, i, false);
        }
    };
    bool ok, second_ok = true;
    if (bgzf) {                                   // two BgzfOut on one context: bgzf_out.h serialises their compressions
        BgzfOut z(bgzf, fd);
        std::unique_ptr<BgzfOut> zf(failed_fd >= 0 ? new BgzfOut(bgzf, failed_fd) : nullptr);
        run(z, zf.get());
        ok = finish(z);
        if (zf) second_ok = finish(*zf);
    } else {
        Copier c(fd, -1);
        std::unique_ptr<Copier> cf(failed_fd >= 0 ? new Copier(failed_fd, -1) : nullptr);
        run(c, cf.get());
        c.flush();
        ok = !c.failed;
        if (cf) { cf->flush(); second_ok = !cf->failed; }
    }
    if (failed_ok) *failed_ok = second_ok;
    return ok;
}

bool report_failed_write(const Arguments &args, bool ok) {
    if (!ok) std::cerr << "Error: cannot write to file: " << args.failed << "\n";
    return ok;
}

void log_after_trim_split(const Arguments &args, uint64_t n_rows, const fl_summary &summary) {
    if (args.trim || args.split_set) {
        if (args.trim && args.split_set) std::cerr << "  after trimming and splitting: ";
        else if (args.trim) std::cerr << "  after trimming: ";
        else std::cerr << "  after splitting: ";
        std::cerr << int_to_string((long long)n_rows) << " reads (" << int_to_string(summary.rows_bases) << " bp)\n";
    }
    std::cerr << "\n";
}

void log_filtering(const Arguments &args, const fl_summary &summary) {
    if (!args.target_bases_set && !args.keep_percent_set) return;
    std::cerr << "Filtering long reads\n";
    std::cerr << "  target: " << int_to_string(summary.target) << " bp\n";
    if (summary.status == 1) std::cerr << "  not enough reads to reach target\n";
    else if (summary.status == 2) std::cerr << "  reads already fall below target after filtering\n";
    else std::cerr << "  keeping " << int_to_string(summary.keeping) << " bp\n";
    std::cerr << "\n";
}

// filtlong_b200/csrc/host/feeder.cpp -- see feeder.h.
#include "feeder.h"

#include <fcntl.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/uio.h>
#include <unistd.h>

#include <stdlib.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <iostream>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "bgzf_out.h"
#include "misc.h"
#include "read.h"
#include "textsrc.h"

namespace {

// The records go to the descriptor stdout had at start-up. With more than one GPU, fd 1 itself is pointed at stderr while the
// run lasts: NCCL (NCCL_DEBUG=VERSION/WARN/INFO) and other libraries print to "stdout", which here is the data stream.
int g_out_fd = 1;
struct StdoutGuard {
    bool on = false;
    void engage() {
        if (on) return;
        fflush(stdout);
        const int d = dup(1);
        if (d < 0) return;
        if (dup2(2, 1) < 0) { close(d); return; }
        g_out_fd = d;
        on = true;
    }
    void release() {                 // the host parser (std::cout) takes over: give it the real stdout back
        if (!on) return;
        fflush(stdout);
        dup2(g_out_fd, 1);
        close(g_out_fd);
        g_out_fd = 1;
        on = false;
    }
};

// ---------------------------------------------------------------------------------------------
// one shard = one GPU = one context = one pusher thread + a ring of pinned chunks filled by copy threads
// ---------------------------------------------------------------------------------------------
struct Records {                      // per shard, in file order; offsets are FILE offsets
    std::vector<uint64_t> name_off, seq_off, qual_off, name_hash;
    std::vector<uint32_t> name_len, comment_len;
    std::vector<int32_t> len;
    size_t n = 0;
    void ensure(size_t cap) {
        if (name_off.size() >= cap) return;
        const size_t c = cap + cap / 2;
        name_off.resize(c); seq_off.resize(c); qual_off.resize(c); name_hash.resize(c);
        name_len.resize(c); comment_len.resize(c); len.resize(c);
    }
};

struct Shard {
    int index = 0, device = 0;
    fl_ctx *ctx = nullptr;
    bool owns_ctx = false;
    size_t chunk_lo = 0, chunk_hi = 0;          // chunks [lo, hi) of the plan
    Records rec;
    // results needed by the writer
    std::vector<int32_t> n_child, row_s, row_e;
    std::vector<uint64_t> row_start;
    std::vector<uint8_t> row_pfinal;
    uint64_t n_rows = 0;
    fl_summary summary{};
    std::string error;
    bool fallback = false;
};

struct Ring {
    static constexpr int KMAX = 32;
    int K = 8;                                  // slots = reader threads per shard (FL_READERS)
    char *slot[KMAX] = {nullptr};
    bool registered[KMAX] = {false};
    int state[KMAX] = {0};                      // 0 free, 1 filled, -1 the reader failed
    std::mutex m;
    std::condition_variable cv;
};

void check(fl_ctx *c, int rc, const char *what) {
    if (rc != FL_OK) throw std::runtime_error(std::string(what) + ": " + fl_last_error(c));
}

// get_ctx0: the caller's context for shard 0 (creating it may take the second or so the CUDA driver needs: the
// readers below are already filling the ring by then)
void run_shard(Shard &sh, const MappedFile &f, const std::vector<Chunk> &plan, int format, const fl_params &params, int nranks,
               const unsigned char *comm_id, const std::function<fl_ctx *()> &get_ctx0, std::atomic<bool> &abort_all, uint64_t slot_bytes,
               bool share_kmers) {
    Ring ring;
    if (const char *e = getenv("FL_READERS")) {
        const int k = atoi(e);
        ring.K = k < 1 ? 1 : (k > ring.KMAX ? ring.KMAX : k);
    }
    std::vector<std::thread> readers;
    try {
        // reader threads first: pread() from the page cache needs neither CUDA nor page faults on a mapping.
        // Chunk i of the shard goes through slot i % K.
        const size_t n_chunks = sh.chunk_hi - sh.chunk_lo;
        for (int k = 0; k < ring.K; ++k) {
            void *p = nullptr;
            if (posix_memalign(&p, 2u << 20, (size_t)slot_bytes + 4096) != 0) throw std::runtime_error("chunk ring: out of memory");
            ring.slot[k] = (char *)p;
        }
        for (int k = 0; k < ring.K; ++k)
            readers.emplace_back([&, k] {
                for (size_t i = (size_t)k; i < n_chunks; i += ring.K) {
                    {
                        std::unique_lock<std::mutex> lk(ring.m);
                        ring.cv.wait(lk, [&] { return ring.state[k] == 0 || abort_all.load(); });
                        if (abort_all.load()) return;
                    }
                    const Chunk &c = plan[sh.chunk_lo + i];
                    uint64_t done = 0;
                    const uint64_t want = c.end - c.begin;
                    bool ok = true;
                    if (f.fd < 0) {                                    // inflated gzip input: already in memory
                        memcpy(ring.slot[k], f.base + c.begin, (size_t)want);
                        done = want;
                    }
                    while (done < want) {
                        const ssize_t r = pread(f.fd, ring.slot[k] + done, (size_t)(want - done), (off_t)(c.begin + done));
                        if (r <= 0) { ok = false; break; }
                        done += (uint64_t)r;
                    }
                    {
                        std::lock_guard<std::mutex> lk(ring.m);
                        ring.state[k] = ok ? 1 : -1;
                    }
                    ring.cv.notify_all();
                    if (!ok) return;
                }
            });
        if (sh.index == 0) sh.ctx = get_ctx0();
        else {
            if (fl_ctx_create(&params, sh.device, &sh.ctx) != FL_OK) throw std::runtime_error(std::string("fl_ctx_create: ") + fl_last_error(nullptr));
            sh.owns_ctx = true;
        }
        check(sh.ctx, fl_ctx_set_params(sh.ctx, &params), "fl_ctx_set_params");
        for (int k = 0; k < ring.K; ++k) ring.registered[k] = fl_host_register(ring.slot[k], slot_bytes + 4096) == FL_OK;
        if (nranks > 1) {
            check(sh.ctx, fl_comm_init(sh.ctx, comm_id, sh.index, nranks), "fl_comm_init");
            if (share_kmers) {
                check(sh.ctx, fl_kmers_broadcast(sh.ctx, 0), "fl_kmers_broadcast");   // Kmers built once (main.cpp:53-59), used by every shard
                uint64_t nk = 0;
                check(sh.ctx, fl_kmers_finalize(sh.ctx, &nk), "fl_kmers_finalize");
            }
        }
        size_t guess = 1024;
        for (size_t i = 0; i < n_chunks && !abort_all.load(); ++i) {
            const int k = (int)(i % ring.K);
            {
                std::unique_lock<std::mutex> lk(ring.m);
                ring.cv.wait(lk, [&] { return ring.state[k] != 0 || abort_all.load(); });
                if (abort_all.load()) break;
                if (ring.state[k] < 0) throw std::runtime_error("Error reading the input file");
            }
            const Chunk &c = plan[sh.chunk_lo + i];
            const uint64_t nb = c.end - c.begin;
            const bool last = sh.chunk_lo + i + 1 == plan.size();
            if (i == 0) guess = (size_t)(nb / 256) + 1024;
            for (;;) {
                Records &R = sh.rec;
                R.ensure(R.n + guess);
                fl_text_records out{};
                out.cap = guess;
                out.name_off = R.name_off.data() + R.n; out.name_len = R.name_len.data() + R.n; out.comment_len = R.comment_len.data() + R.n;
                out.seq_off = R.seq_off.data() + R.n; out.qual_off = R.qual_off.data() + R.n; out.len = R.len.data() + R.n;
                out.name_hash = R.name_hash.data() + R.n;
                uint64_t n_rec = 0, used = 0;
                int status = 0;
                const int rc = fl_reads_push_text(sh.ctx, ring.slot[k], nb, format, last ? 1 : 0, &out, &n_rec, &used, &status);
                if (rc == FL_ERANGE && n_rec > guess) { guess = (size_t)n_rec + 16; continue; }
                check(sh.ctx, rc, "fl_reads_push_text");
                if (status != FL_TEXT_OK || used != nb) { sh.fallback = true; abort_all.store(true); break; }
                for (size_t j = R.n; j < R.n + n_rec; ++j) {            // chunk offsets -> file offsets
                    R.name_off[j] += c.begin; R.seq_off[j] += c.begin; R.qual_off[j] += c.begin;
                }
                R.n += (size_t)n_rec;
                guess = (size_t)n_rec + (size_t)n_rec / 4 + 1024;
                break;
            }
            {
                std::lock_guard<std::mutex> lk(ring.m);
                ring.state[k] = 0;
            }
            ring.cv.notify_all();
        }
    } catch (const std::exception &e) {
        sh.error = e.what();
        abort_all.store(true);
    }
    ring.cv.notify_all();
    for (auto &t : readers) t.join();
    for (int k = 0; k < ring.K; ++k) {
        if (ring.registered[k]) fl_host_unregister(ring.slot[k]);
        free(ring.slot[k]);
    }
}

// main.cpp:169-261 on every shard (collective over NCCL when there are several), then the arrays the writer needs
void finalize_shard(Shard &sh) {
    try {
        check(sh.ctx, fl_finalize(sh.ctx, -1, &sh.summary), "fl_finalize");
        uint64_t nr = 0, nw = 0;
        check(sh.ctx, fl_reads_count(sh.ctx, &nr, &nw, nullptr), "fl_reads_count");
        sh.n_rows = nw;
        sh.n_child.resize(nr); sh.row_start.resize(nr);
        sh.row_s.resize(nw); sh.row_e.resize(nw); sh.row_pfinal.resize(nw);
        fl_read_results rr{};
        rr.n_child = sh.n_child.data(); rr.row_start = sh.row_start.data();
        check(sh.ctx, fl_results_reads(sh.ctx, &rr), "fl_results_reads");
        fl_row_results wr{};
        wr.start = sh.row_s.data(); wr.end = sh.row_e.data(); wr.passed_final = sh.row_pfinal.data();
        check(sh.ctx, fl_results_rows(sh.ctx, &wr), "fl_results_rows");
    } catch (const std::exception &e) {
        sh.error = e.what();
    }
}

// ---------------------------------------------------------------------------------------------
// duplicate names (main.cpp:113-117) at scale: a flat open-addressing table over the 64-bit hashes the
// device computed, names compared byte for byte in the mapping only when two hashes agree
// ---------------------------------------------------------------------------------------------
struct NameRef { uint64_t off; uint32_t len; };

bool find_duplicate(const std::vector<Shard> &shards, const char *base, std::string *dup) {
    size_t n = 0;
    for (auto &s : shards) n += s.rec.n;
    size_t cap = 16;
    while (cap < 2 * n + 16) cap <<= 1;
    std::vector<uint64_t> keys(cap, 0);
    std::vector<NameRef> vals(cap);
    std::vector<uint8_t> used(cap, 0);
    for (auto &s : shards)
        for (size_t i = 0; i < s.rec.n; ++i) {
            const uint64_t h = s.rec.name_hash[i];
            size_t slot = (size_t)(h * 0x9E3779B97F4A7C15ull) & (cap - 1);
            for (;;) {
                if (!used[slot]) {
                    used[slot] = 1; keys[slot] = h; vals[slot] = NameRef{s.rec.name_off[i], s.rec.name_len[i]};
                    break;
                }
                if (keys[slot] == h && vals[slot].len == s.rec.name_len[i] &&
                    memcmp(base + vals[slot].off, base + s.rec.name_off[i], s.rec.name_len[i]) == 0) {
                    dup->assign(base + s.rec.name_off[i], s.rec.name_len[i]);
                    return true;
                }
                slot = (slot + 1) & (cap - 1);
            }
        }
    return false;
}

// ---------------------------------------------------------------------------------------------
// pass 2: the survivors, in input order, straight out of the mapping (main.cpp:263-313)
// ---------------------------------------------------------------------------------------------
struct Writer {
    static constexpr int MAXV = 1000;
    struct iovec v[MAXV];
    int nv = 0;
    std::vector<std::string> small;            // child names: must stay alive (and in place: short strings live inside the object) until the flush
    bool failed = false;
    Writer() { small.reserve(256); }
    void flush() {
        int done = 0;
        while (done < nv && !failed) {
            ssize_t w = writev(g_out_fd, v + done, nv - done);
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
};

}  // namespace

FeederOutcome run_text_feeder(Arguments &args, Kmers &kmers, const std::function<void(const char *)> &mark) {
    FeederOutcome res;
    if (args.verbose || getenv("FL_HOST_PARSER")) return res;           // per-read dumps come from the host path
    MappedFile f;
    bool inflated = false;
    if (!f.open_any(args.input_reads, &inflated)) return res;           // neither plain nor gzip that fits in memory: the host reader
    if (inflated) mark("gzip input inflated into memory");
    const int format = f.format();
    if (!format) return res;
    const bool kmers_empty = kmers.empty();
    if (format == FL_TEXT_FASTA && kmers_empty) return res;             // main.cpp:103-106: the host path prints the error
    uint64_t target = 128ull << 20;
    if (const char *e = getenv("FL_CHUNK_MB")) target = (uint64_t)atoll(e) << 20;
    if (target < (1ull << 20)) target = 1ull << 20;
    if (target > (1024ull << 20)) target = 1024ull << 20;
    const uint64_t max_chunk = target;                                   // plan_chunks never cuts later than `target` bytes after a chunk's start
    int nranks = args.gpus;
    std::vector<Chunk> plan;
    if (!plan_chunks(f.base, f.size, format, target, max_chunk, plan) || plan.empty()) return res;
    if ((size_t)nranks > plan.size()) nranks = (int)plan.size();         // tiny inputs: fewer shards than GPUs asked for

    const fl_params params = params_from_arguments(args);
    unsigned char comm_id[FL_COMM_ID_BYTES] = {0};
    StdoutGuard guard;
    if (nranks > 1) guard.engage();
    if (nranks > 1 && fl_comm_unique_id(comm_id) != FL_OK) throw std::runtime_error("NCCL is not available: cannot shard across GPUs");
    // contiguous chunk ranges, balanced by bytes (file order is kept: shard r holds the records before shard r + 1's)
    std::vector<Shard> shards((size_t)nranks);
    {
        size_t c = 0;
        for (int r = 0; r < nranks; ++r) {
            shards[r].index = r;
            shards[r].device = r;
            shards[r].chunk_lo = c;
            const uint64_t goal = f.size / (uint64_t)nranks * (uint64_t)(r + 1);
            while (c < plan.size() && (r + 1 == nranks || plan[c].end <= goal || c == shards[r].chunk_lo)) ++c;
            shards[r].chunk_hi = c;
        }
        shards.back().chunk_hi = plan.size();
    }
    std::atomic<bool> abort_all(false);
    fl_ctx *ctx0 = nullptr;
    const std::function<fl_ctx *()> get_ctx0 = [&]() { ctx0 = kmers.context(); return ctx0; };
    {
        std::vector<std::thread> ts;
        for (int r = 1; r < nranks; ++r)
            ts.emplace_back(run_shard, std::ref(shards[r]), std::cref(f), std::cref(plan), format, std::cref(params), nranks, comm_id,
                            std::cref(get_ctx0), std::ref(abort_all), max_chunk, !kmers_empty);
        run_shard(shards[0], f, plan, format, params, nranks, comm_id, get_ctx0, abort_all, max_chunk, !kmers_empty);
        for (auto &t : ts) t.join();
    }
    auto cleanup = [&]() {
        for (auto &s : shards) {
            if (s.ctx && nranks > 1) fl_comm_destroy(s.ctx);
            if (s.owns_ctx && s.ctx) fl_ctx_destroy(s.ctx);
        }
    };
    for (auto &s : shards)
        if (!s.error.empty()) { cleanup(); throw std::runtime_error(s.error); }
    if (abort_all.load()) {                                             // not the simple layout after all: start over on the host
        if (ctx0) fl_reads_reset(ctx0);
        cleanup();
        guard.release();
        return res;
    }
    mark("pass 1 (device parse + score)");
    res.handled = true;
    std::cerr << "Scoring long reads\n";
    long long n_reads = 0, total_bases = 0;
    for (auto &s : shards) {
        n_reads += (long long)s.rec.n;
        for (size_t i = 0; i < s.rec.n; ++i) total_bases += s.rec.len[i];
    }
    {
        std::string dup;
        if (find_duplicate(shards, f.base, &dup)) {
            std::cerr << "Error: duplicate read name: " << dup << "\n";       // main.cpp:113-116
            cleanup();
            res.exit_code = 1;
            return res;
        }
    }
    print_read_score_progress(n_reads, total_bases);
    std::cerr << "\n";
    mark("duplicate-name check");
    // ---- normalise, final score, target (main.cpp:136-261) ----
    {
        std::vector<std::thread> ts;
        for (int r = 1; r < nranks; ++r) ts.emplace_back(finalize_shard, std::ref(shards[r]));
        finalize_shard(shards[0]);
        for (auto &t : ts) t.join();
    }
    for (auto &s : shards)
        if (!s.error.empty()) { cleanup(); throw std::runtime_error(s.error); }
    mark("finalize + download");
    const fl_summary &summary = shards[0].summary;
    uint64_t n_rows = 0;
    for (auto &s : shards) n_rows += s.n_rows;
    if (args.trim || args.split_set) {
        if (args.trim && args.split_set) std::cerr << "  after trimming and splitting: ";
        else if (args.trim) std::cerr << "  after trimming: ";
        else std::cerr << "  after splitting: ";
        std::cerr << int_to_string((long long)n_rows) << " reads (" << int_to_string(summary.rows_bases) << " bp)\n";
    }
    std::cerr << "\n";
    if (args.target_bases_set || args.keep_percent_set) {
        std::cerr << "Filtering long reads\n";
        std::cerr << "  target: " << int_to_string(summary.target) << " bp\n";
        if (summary.status == 1) std::cerr << "  not enough reads to reach target\n";
        else if (summary.status == 2) std::cerr << "  reads already fall below target after filtering\n";
        else std::cerr << "  keeping " << int_to_string(summary.keeping) << " bp\n";
        std::cerr << "\n";
    }
    // ---- pass 2 ----
    std::cerr << "Outputting passed long reads\n";
    fflush(stdout);
    const char lead = format == FL_TEXT_FASTA ? '>' : '@';
    // one output record; Sink is a Writer (iovecs into the mapping) or a Sizer / Copier (below)
    auto emit_read = [&](auto &sink, const Shard &s, size_t i) {
        static const char plus_nl[] = "+\n", nl[] = "\n", sp[] = " ";
        const Records &R = s.rec;
        const size_t rs = (size_t)s.row_start[i];
        const int nc = s.n_child[i];
        if (nc == 0) {
            if (!s.row_pfinal[rs]) return;
            sink.put(f.base + R.name_off[i] - 1, 1 + (size_t)R.name_len[i]);                        // '@' / '>' + name
            if (R.comment_len[i]) { sink.put(sp, 1); sink.put(f.base + R.name_off[i] + R.name_len[i] + 1, R.comment_len[i]); }
            sink.put(nl, 1);
            sink.put(f.base + R.seq_off[i], (size_t)R.len[i]);
            sink.put(nl, 1);
            if (format == FL_TEXT_FASTQ) { sink.put(plus_nl, 2); sink.put(f.base + R.qual_off[i], (size_t)R.len[i]); sink.put(nl, 1); }
            return;
        }
        for (int c = 0; c < nc; ++c) {
            const size_t row = rs + (size_t)c;
            if (!s.row_pfinal[row]) continue;
            const int start = s.row_s[row], length = s.row_e[row] - s.row_s[row];
            if (length <= 0) continue;
            std::string nm(1, lead);
            nm.append(f.base + R.name_off[i], R.name_len[i]);
            nm += "_" + std::to_string(start + 1) + "-" + std::to_string(s.row_e[row]);              // read.cpp:135-136
            sink.put_owned(std::move(nm));
            if (R.comment_len[i]) { sink.put(sp, 1); sink.put(f.base + R.name_off[i] + R.name_len[i] + 1, R.comment_len[i]); }
            sink.put(nl, 1);
            sink.put(f.base + R.seq_off[i] + start, (size_t)length);
            sink.put(nl, 1);
            if (format == FL_TEXT_FASTQ) { sink.put(plus_nl, 2); sink.put(f.base + R.qual_off[i] + start, (size_t)length); sink.put(nl, 1); }
        }
    };
    bool out_failed = false;
    struct stat ost;
    const int oflags = fcntl(g_out_fd, F_GETFL);
    const bool to_file = !args.bgzip && fstat(g_out_fd, &ost) == 0 && S_ISREG(ost.st_mode) && oflags >= 0 && !(oflags & O_APPEND) && !getenv("FL_SERIAL_OUTPUT");
    if (to_file) {
        // stdout is a regular file: contiguous groups of reads are sized, then written with pwrite() by a few threads
        struct Sizer {
            uint64_t n = 0;
            void put(const void *, size_t k) { n += k; }
            void put_owned(std::string s) { n += s.size(); }
        };
        struct Copier {
            int fd; uint64_t pos; std::string buf; bool failed = false;
            void flush() {
                size_t done = 0;
                while (done < buf.size() && !failed) {
                    const ssize_t w = pwrite(fd, buf.data() + done, buf.size() - done, (off_t)(pos + done));
                    if (w < 0) { failed = true; break; }
                    done += (size_t)w;
                }
                pos += buf.size();
                buf.clear();
            }
            void put(const void *p, size_t k) { buf.append((const char *)p, k); if (buf.size() >= (8u << 20)) flush(); }
            void put_owned(std::string s) { put(s.data(), s.size()); }
        };
        struct Group { size_t shard, lo, hi; uint64_t bytes = 0, at = 0; };
        std::vector<Group> groups;
        const size_t per = (size_t)(n_reads / 32) + 1;
        for (size_t si = 0; si < shards.size(); ++si)
            for (size_t lo = 0; lo < shards[si].rec.n; lo += per) groups.push_back(Group{si, lo, std::min(lo + per, shards[si].rec.n), 0, 0});
        const off_t base_pos = lseek(g_out_fd, 0, SEEK_CUR);
        std::atomic<size_t> next(0);
        auto work = [&](bool write_pass) {
            std::vector<std::thread> ts;
            next.store(0);
            std::atomic<bool> bad(false);
            const unsigned nt = std::min<size_t>(8, groups.size());
            for (unsigned t = 0; t < nt; ++t)
                ts.emplace_back([&] {
                    for (size_t g = next.fetch_add(1); g < groups.size(); g = next.fetch_add(1)) {
                        Group &G = groups[g];
                        if (!write_pass) {
                            Sizer z;
                            for (size_t i = G.lo; i < G.hi; ++i) emit_read(z, shards[G.shard], i);
                            G.bytes = z.n;
                        } else {
                            Copier c{g_out_fd, (uint64_t)base_pos + G.at, std::string()};
                            c.buf.reserve((8u << 20) + (2u << 20));
                            for (size_t i = G.lo; i < G.hi; ++i) emit_read(c, shards[G.shard], i);
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
        if (base_pos < 0 || !work(true)) out_failed = true;
        else if (lseek(g_out_fd, base_pos + (off_t)total_out, SEEK_SET) < 0) out_failed = true;
    } else if (args.bgzip) {
        // compressed offsets are not known in advance: pipe or file, the members are written in order (GPU 0 compresses)
        BgzfOut z(ctx0, g_out_fd);
        for (auto &s : shards)
            for (size_t i = 0; i < s.rec.n; ++i) emit_read(z, s, i);
        out_failed = !z.finish();
        if (out_failed && !z.error().empty()) std::cerr << "Error: " << z.error() << "\n";
    } else {
        Writer w;
        for (auto &s : shards)
            for (size_t i = 0; i < s.rec.n; ++i) emit_read(w, s, i);
        w.flush();
        out_failed = w.failed;
    }
    mark("pass 2 (slices of the mapped input)");
    std::cerr << "\n";
    cleanup();
    res.exit_code = out_failed ? 1 : 0;
    return res;
}

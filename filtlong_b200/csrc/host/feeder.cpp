// filtlong_b200/csrc/host/feeder.cpp -- see feeder.h.
#include "feeder.h"

#include <string.h>
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

#include "bam.h"
#include "misc.h"
#include "read.h"
#include "streamsrc.h"
#include "survivors.h"
#include "textsrc.h"

namespace {

// The records go to the descriptor stdout had at start-up. With more than one GPU, fd 1 itself is pointed at stderr while the
// run lasts: NCCL (NCCL_DEBUG=VERSION/WARN/INFO) and other libraries print to "stdout", which here is the data stream.
int g_out_fd = 1;

// ---------------------------------------------------------------------------------------------
// one shard = one GPU = one context = one pusher thread + a ring of pinned chunks filled by copy threads
// ---------------------------------------------------------------------------------------------
struct Shard {
    int index = 0, device = 0;
    fl_ctx *ctx = nullptr;
    bool owns_ctx = false;
    size_t chunk_lo = 0, chunk_hi = 0;          // chunks [lo, hi) of the plan
    Records rec;                                // lead_checked: fl_reads_push_text checks every record's '@' / '>'
    std::vector<Follower> followers;            // BAM --aligned: the records that follow a read of rec (or no read)
    // results needed by the writer
    std::vector<int32_t> n_child, row_s, row_e;
    std::vector<uint64_t> row_start;
    std::vector<uint8_t> row_pfinal;
    uint64_t n_rows = 0;
    fl_contam_counts contam{};                  // --contam: what the shard's reads lost
    fl_summary summary{};
    std::string error;
    bool fallback = false;
};

// The shards of one run: contiguous chunk ranges of the plan, balanced by bytes (file order is kept: shard r holds the
// records before shard r + 1's). A tiny input gets fewer shards than GPUs asked for; a growing stream's one shard takes
// every chunk that comes. With more than one shard, fd 1 points at stderr while they live. Going away, it destroys their
// NCCL communicators and the contexts they created (shard 0 scores on the caller's), then gives stdout back.
struct ShardSet {
    std::vector<Shard> v;
    ShardSet(const std::vector<Chunk> &cs, uint64_t size, int gpus, bool growing) {
        const int nranks = growing || (size_t)gpus <= cs.size() ? gpus : cs.empty() ? 1 : (int)cs.size();
        v.resize((size_t)nranks);
        size_t c = 0;
        for (int r = 0; r < nranks; ++r) {
            Shard &sh = v[r];
            sh.index = sh.device = r;
            sh.chunk_lo = c;
            sh.rec.lead_checked = true;
            const uint64_t goal = size / (uint64_t)nranks * (uint64_t)(r + 1);
            while (c < cs.size() && (r + 1 == nranks || cs[c].end <= goal || c == sh.chunk_lo)) ++c;
            sh.chunk_hi = c;
        }
        v.back().chunk_hi = growing ? SIZE_MAX : cs.size();
        if (nranks == 1) return;
        fflush(stdout);
        const int d = dup(1);
        if (d >= 0 && dup2(2, 1) >= 0) g_out_fd = d;
        else if (d >= 0) close(d);
    }
    ShardSet(const ShardSet &) = delete;
    ~ShardSet() {
        for (auto &s : v) {
            if (s.ctx && v.size() > 1) fl_comm_destroy(s.ctx);
            if (s.owns_ctx && s.ctx) fl_ctx_destroy(s.ctx);
        }
        if (g_out_fd == 1) return;
        fflush(stdout);
        dup2(g_out_fd, 1);
        close(g_out_fd);
        g_out_fd = 1;
    }
};

struct Ring {
    static constexpr int KMAX = 32;
    int K = 8;                                  // slots = reader threads per shard (FL_READERS)
    char *slot[KMAX] = {nullptr};
    bool registered[KMAX] = {false};
    int state[KMAX] = {0};                      // 0 free, 1 filled, -1 the reader failed
    bool stop = false;                          // the shard stopped on its own (an error in the input): readers stop too
    std::mutex m;
    std::condition_variable cv;
};

void check(fl_ctx *c, int rc, const char *what) {
    if (rc != FL_OK) throw std::runtime_error(std::string(what) + ": " + fl_last_error(c));
}

// A record of the input that fails a check. Only the shard that met it stops: the shards after it hold later records,
// and the one before it may still meet an earlier one, whose message is the one printed.
struct InputError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

// The chunks of the input, in order. A file's plan is whole before the first push (done()); a stream's grows while the
// stream arrives (add(), then close()), and the shard's readers and pusher wait for the chunks they need.
class Plan {
public:
    std::vector<Chunk> chunks;              // a whole plan: set before any shard runs, read-only afterwards
    void done() { complete_ = true; }
    // `final`: c is the input's last chunk (the plan is complete with it, in the same step)
    void add(const Chunk &c, bool final) {
        {
            std::lock_guard<std::mutex> lk(m_);
            chunks.push_back(c);
            complete_ = complete_ || final;
        }
        cv_.notify_all();
    }
    bool failed() {
        std::lock_guard<std::mutex> lk(m_);
        return failed_;
    }
    // ok == false: no boundary to cut at, or the stream broke; or cancel(): a shard stopped
    void close(bool ok) {
        { std::lock_guard<std::mutex> lk(m_); complete_ = true; failed_ = failed_ || !ok; }
        cv_.notify_all();
    }
    void cancel() { close(false); }
    // Chunk i and whether it is the input's last. 1: *c, *last set; 0: the plan ended before chunk i; -1: it failed first.
    // A chunk cut while the stream still arrives is never the last: bytes after it have arrived.
    int get(size_t i, Chunk *c, bool *last) {
        std::unique_lock<std::mutex> lk(m_);
        cv_.wait(lk, [&] { return i < chunks.size() || complete_; });
        if (i < chunks.size() && !failed_) {
            *c = chunks[i];
            *last = complete_ && i + 1 == chunks.size();
            return 1;
        }
        return failed_ ? -1 : 0;
    }

private:
    std::mutex m_;
    std::condition_variable cv_;
    bool complete_ = false, failed_ = false;
};

// How the chunks of one input reach the device. fill (may be empty): on a reader thread, once chunk ci (c) of the plan
// is in its ring slot. push: on the shard's thread, scores chunk ci and appends its records to sh.rec as file offsets;
// false when the chunk is not the layout the device parses (the host parser then reads the whole input). `guess` is the
// shard's own scratch, 0 before its first chunk.
struct ChunkPush {
    std::function<void(size_t ci, const Chunk &c, const char *slot)> fill;
    std::function<bool(Shard &sh, size_t ci, const Chunk &c, bool last, const char *slot, size_t &guess)> push;
};

// FASTQ / FASTA text: the device finds the records (fl_reads_push_text)
ChunkPush text_push(int format) {
    ChunkPush p;
    p.push = [format](Shard &sh, size_t, const Chunk &c, bool last, const char *slot, size_t &guess) {
        const uint64_t nb = c.end - c.begin;
        if (guess == 0) guess = (size_t)(nb / 256) + 1024;
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
            const int rc = fl_reads_push_text(sh.ctx, slot, nb, format, last ? 1 : 0, &out, &n_rec, &used, &status);
            if (rc == FL_ERANGE && n_rec > guess) { guess = (size_t)n_rec + 16; continue; }
            check(sh.ctx, rc, "fl_reads_push_text");
            if (status != FL_TEXT_OK || used != nb) return false;
            for (size_t j = R.n; j < R.n + n_rec; ++j) {            // chunk offsets -> file offsets
                R.name_off[j] += c.begin; R.seq_off[j] += c.begin; R.qual_off[j] += c.begin;
            }
            R.n += (size_t)n_rec;
            guess = (size_t)n_rec + (size_t)n_rec / 4 + 1024;
            return true;
        }
    };
    return p;
}

// BAM: a reader thread checks and indexes the chunk's records (bam.h) while the shard's thread pushes the one before;
// the device only gathers and scores (fl_reads_push_bam_strand). aligned: the reads' strands go with them, and the
// followers into the shard's list.
ChunkPush bam_push(const char *base, std::vector<BamChunkIndex> &idx, bool aligned) {
    ChunkPush p;
    p.fill = [base, &idx, aligned](size_t ci, const Chunk &c, const char *) { bam_index_chunk(base, c, idx[ci], aligned); };
    p.push = [&idx, aligned](Shard &sh, size_t ci, const Chunk &c, bool, const char *slot, size_t &) {
        BamChunkIndex &ix = idx[ci];
        if (!ix.error.empty()) throw InputError(ix.error);
        const Records &X = ix.rec;
        check(sh.ctx, fl_reads_push_bam_strand(sh.ctx, slot, c.end - c.begin, X.n, ix.seq32.data(), ix.qual32.data(), X.len.data(),
                                               aligned ? ix.reverse.data() : nullptr),
              "fl_reads_push_bam_strand");
        bam_append_chunk(ix, c, sh.rec, sh.followers);
        ix = BamChunkIndex();
        return true;
    };
    return p;
}

// get_ctx0: the caller's context for shard 0 (creating it may take the second or so the CUDA driver needs: the
// readers below are already filling the ring by then)
void run_shard(Shard &sh, const MappedFile &f, Plan &plan, const ChunkPush &push, const fl_params &params, int nranks,
               const unsigned char *comm_id, const std::function<fl_ctx *()> &get_ctx0, std::atomic<bool> &abort_all, uint64_t slot_bytes,
               bool share_kmers, const Kmers *share_contam, StreamInput *stream) {
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
                        ring.cv.wait(lk, [&] { return ring.state[k] == 0 || abort_all.load() || ring.stop; });
                        if (abort_all.load() || ring.stop) return;
                    }
                    Chunk c;
                    bool last;
                    if (plan.get(sh.chunk_lo + i, &c, &last) != 1) return;    // a stream's plan ended (the pusher sees it too)
                    uint64_t done = 0;
                    const uint64_t want = c.end - c.begin;
                    bool ok = true;
                    if (f.fd < 0) {                                    // inflated gzip input or a stream: already in memory
                        memcpy(ring.slot[k], f.base + c.begin, (size_t)want);
                        done = want;
                    }
                    while (done < want) {
                        const ssize_t r = pread(f.fd, ring.slot[k] + done, (size_t)(want - done), (off_t)(c.begin + done));
                        if (r <= 0) { ok = false; break; }
                        done += (uint64_t)r;
                    }
                    if (ok && push.fill) push.fill(sh.chunk_lo + i, c, ring.slot[k]);
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
            if (share_contam) {
                if (sh.index != 0 && share_contam->contam_k() > 16)   // the table's bytes go as they are: the same size everywhere
                    check(sh.ctx, fl_contam_configure(sh.ctx, share_contam->contam_k(), share_contam->contam_max_kmers()), "fl_contam_configure");
                check(sh.ctx, fl_contam_broadcast(sh.ctx, 0), "fl_contam_broadcast");
                uint64_t nk = 0;
                check(sh.ctx, fl_contam_finalize(sh.ctx, &nk), "fl_contam_finalize");
            }
        }
        size_t guess = 0;
        for (size_t i = 0; i < n_chunks && !abort_all.load(); ++i) {
            const int k = (int)(i % ring.K);
            Chunk c;
            bool last;
            const int got = plan.get(sh.chunk_lo + i, &c, &last);
            if (got == 0) break;                                       // the end of a stream
            if (got < 0) { sh.fallback = true; abort_all.store(true); break; }
            {
                std::unique_lock<std::mutex> lk(ring.m);
                ring.cv.wait(lk, [&] { return ring.state[k] != 0 || abort_all.load(); });
                if (abort_all.load()) break;
                if (ring.state[k] < 0) throw std::runtime_error("Error reading the input file");
            }
            if (!push.push(sh, sh.chunk_lo + i, c, last, ring.slot[k], guess)) { sh.fallback = true; abort_all.store(true); break; }
            if (stream) {
                ++stream->chunks;
                if (!stream->ended()) ++stream->chunks_before_end;
            }
            {
                std::lock_guard<std::mutex> lk(ring.m);
                ring.state[k] = 0;
            }
            ring.cv.notify_all();
        }
    } catch (const InputError &e) {
        sh.error = e.what();
        std::lock_guard<std::mutex> lk(ring.m);
        ring.stop = true;
    } catch (const std::exception &e) {
        sh.error = e.what();
        abort_all.store(true);
    }
    if (abort_all.load()) plan.cancel();                               // readers waiting for a stream's next chunk
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
        check(sh.ctx, fl_results_contam(sh.ctx, nullptr, nullptr, &sh.contam), "fl_results_contam");
    } catch (const std::exception &e) {
        sh.error = e.what();
    }
}

struct NameRef { uint64_t off; uint32_t len; };

// the first shard's error, if one failed
void throw_shard_error(const std::vector<Shard> &shards) {
    for (auto &s : shards)
        if (!s.error.empty()) throw std::runtime_error(s.error);
}

// ---- the steps of run_device_feeder, in the order they run ----
using Mark = std::function<void(const char *)>;

// The input as the device reads it: one byte range and its format
struct Source {
    const MappedFile *file = nullptr;       // nullptr: the device declines the input, and the host path reads it
    int format = 0;
    StreamInput *stream = nullptr;          // the input reads are a stream
    bool growing = false;                   // ... scored while it still arrives (plain text, one GPU)
};

// How the input is cut into chunks
struct Cuts {
    uint64_t target = chunk_target(128ull << 20);
    uint64_t max_chunk = target;            // no chunk is longer (plan_chunks never cuts later than `target` bytes on)
    uint64_t bam_header = 0;                // BAM: bytes [0, bam_header) of the input are its header
    uint64_t bam_max_record = 0;            // BAM: its largest record
};

// A stream's plain text goes to the device while it arrives; any other stream is read to its end first, then goes as a
// file does: mapped, or gzip inflated into `own`. The host parser (the per-read dumps come from the host path, which reads
// text only) leaves only BAM here: a file needs the BAM magic to be opened at all. Then a stream under two bytes, BAM with
// --verbose (an error) and FASTA without k-mers decline.
Source choose_source(const Arguments &args, Kmers &kmers, StreamInput *stream, MappedFile &own, const Mark &mark) {
    const bool host_parser = args.verbose || getenv("FL_HOST_PARSER");
    Source src;
    std::string why;
    bool inflated = false;
    if (stream) {
        bool ended = false;
        const uint64_t head = stream->wait_for(2, &ended);
        const char b0 = head ? stream->base()[0] : 0;
        src.growing = !host_parser && args.gpus == 1 && head >= 2 && (b0 == '@' || b0 == '>');
        if (src.growing) src.format = b0 == '@' ? FL_TEXT_FASTQ : FL_TEXT_FASTA;
        else if (!stream->finish(&why, kmers.device_inflater())) throw std::runtime_error(why);
        src.file = &stream->file();
        src.stream = stream;
        inflated = stream->inflated();
    } else {
        if (host_parser && !bam_file_magic(args.input_reads)) return Source();
        if (!own.open_any(args.input_reads, &inflated, &why, kmers.device_inflater())) {   // neither plain nor gzip in memory: the host reader
            if (own.gzip && bam_file_magic(args.input_reads)) throw std::runtime_error("cannot read BAM input " + args.input_reads + ": " + why);
            return Source();
        }
        src.file = &own;
    }
    if (inflated) mark(("gzip input inflated into memory (" + src.file->inflater + ")").c_str());   // FL_CLI_TIMING: and by what
    if (stream && !src.growing && src.file->size < 2 && !inflated) return Source();   // as MappedFile::open_plain declines a file that small
    if (!src.growing) src.format = src.file->format();
    if (!src.format) return Source();
    const bool bam = src.format == FL_FORMAT_BAM;
    if (bam && args.verbose) throw std::runtime_error("--verbose is not supported with BAM input");
    if (!bam && host_parser) return Source();
    if (src.format == FL_TEXT_FASTA && kmers.empty()) return Source();   // main.cpp:103-106: the host path prints the error
    return src;
}

// The chunks of a file or an ended stream, all cut here; a growing stream's are cut by plan_stream while it arrives.
// false: text with no record start to cut at, left to the host path. A BAM input's records are known here or never: a
// broken header or block_size chain is an error.
bool plan_input(const Source &src, Plan &plan, Cuts &cuts, const Mark &mark) {
    if (src.growing) return true;
    const MappedFile &f = *src.file;
    std::string why;
    if (src.format == FL_FORMAT_BAM) {
        if (!bam_header(f.base, f.size, &cuts.bam_header, &why) ||
            !bam_plan_chunks(f.base, f.size, cuts.bam_header, cuts.target, plan.chunks, &cuts.max_chunk, &why, &cuts.bam_max_record))
            throw std::runtime_error(why);
        mark("BAM block_size chain");
    } else if (!plan_chunks(f.base, f.size, src.format, cuts.target, cuts.max_chunk, plan.chunks) || plan.chunks.empty()) {
        return false;
    }
    plan.done();
    return true;
}

// A growing stream's chunks, cut as its bytes arrive: the same cuts plan_chunks makes of the whole (textsrc.h). Runs on a
// thread of its own beside the shard.
void plan_stream(StreamInput &stream, int format, const Cuts &cuts, Plan &plan) {
    uint64_t pos = 0, avail = 0;
    for (;;) {
        bool ended = false;
        avail = stream.wait_for(std::max(avail + 1, pos + cuts.target + 1), &ended);   // what plan_next_chunk needs to cut
        if (ended && stream.broken()) { plan.close(false); return; }
        Chunk c;
        int r;
        while ((r = plan_next_chunk(stream.base(), avail, ended, format, cuts.target, cuts.max_chunk, pos, &c)) == 1) {
            pos = c.end;
            plan.add(c, ended && pos == avail);
        }
        if (r < 0 || plan.failed()) { plan.close(false); return; }
        if (ended) { plan.close(true); return; }
    }
}

// Runs every shard, shard 0 on this thread, and a growing stream's planner beside them. true: a shard handed a chunk back,
// or a stream's plan failed; the host path is then to read the whole input.
bool score(std::vector<Shard> &shards, const Source &src, const Cuts &cuts, Plan &plan, const ChunkPush &push, const Arguments &args,
           Kmers &kmers, bool share_kmers, bool share_contam) {
    const int nranks = (int)shards.size();
    unsigned char comm_id[FL_COMM_ID_BYTES] = {0};
    if (nranks > 1 && fl_comm_unique_id(comm_id) != FL_OK) throw std::runtime_error("NCCL is not available: cannot shard across GPUs");
    const fl_params params = params_from_arguments(args);
    std::atomic<bool> abort_all(false);
    const std::function<fl_ctx *()> get_ctx0 = [&]() { return kmers.context(); };
    const Kmers *contam = share_contam ? &kmers : nullptr;
    std::thread planner;
    if (src.growing) planner = std::thread(plan_stream, std::ref(*src.stream), src.format, std::cref(cuts), std::ref(plan));
    std::vector<std::thread> ts;
    for (int r = 1; r < nranks; ++r)
        ts.emplace_back(run_shard, std::ref(shards[r]), std::cref(*src.file), std::ref(plan), std::cref(push), std::cref(params), nranks, comm_id,
                        std::cref(get_ctx0), std::ref(abort_all), cuts.max_chunk, share_kmers, contam, src.stream);
    run_shard(shards[0], *src.file, plan, push, params, nranks, comm_id, get_ctx0, abort_all, cuts.max_chunk, share_kmers, contam,
              src.stream);
    for (auto &t : ts) t.join();
    if (planner.joinable()) planner.join();
    return abort_all.load();
}

// The checks main.cpp makes while it parses, over the records the shards found: the message to print, or "" when they
// pass. A BAM input's FASTQ equivalent holds a FASTA record wherever the quality is missing: a mix of the two is an error,
// and so is FASTA without k-mers. Then duplicate names (main.cpp:113-117), in an index of the read names that then
// finds each follower's read (BAM --aligned); *orphans: the followers without one.
std::string check_records(std::vector<Shard> &shards, const char *base, bool bam, bool kmers_empty, uint64_t *orphans) {
    if (bam) {
        NameRef first_q{}, first_f{};
        long long nq = -1, nf = -1, k = 0;
        for (auto &s : shards)
            for (size_t i = 0; i < s.rec.n && (nq < 0 || nf < 0); ++i, ++k) {
                const bool fasta = bam_no_quality(base + s.rec.qual_off[i]);
                if (fasta && nf < 0) { nf = k; first_f = NameRef{s.rec.name_off[i], s.rec.name_len[i]}; }
                if (!fasta && nq < 0) { nq = k; first_q = NameRef{s.rec.name_off[i], s.rec.name_len[i]}; }
            }
        if (nf >= 0 && kmers_empty && (nq < 0 || nf < nq)) return "\n\nError: FASTA input not supported without an external reference\n";
        const NameRef at = nf > nq ? first_f : first_q;
        if (nf >= 0 && nq >= 0) return "\n\nError: could not parse input reads\n  problem occurred at read " + std::string(base + at.off, at.len) + "\n";
    }
    std::vector<const Records *> tables;
    for (auto &s : shards) tables.push_back(&s.rec);
    NameIndex names;
    std::string dup;
    if (!names.build(tables, base, &dup)) return "Error: duplicate read name: " + dup + "\n";     // main.cpp:113-116
    *orphans = 0;
    for (auto &s : shards) *orphans += bam_join_followers(base, names, s.followers);
    return "";
}

// normalise, final score, target (main.cpp:136-261) on every shard, collective over NCCL when there are several; then
// the log that follows
void finalize(std::vector<Shard> &shards, const Arguments &args, const Mark &mark) {
    std::vector<std::thread> ts;
    for (size_t r = 1; r < shards.size(); ++r) ts.emplace_back(finalize_shard, std::ref(shards[r]));
    finalize_shard(shards[0]);
    for (auto &t : ts) t.join();
    throw_shard_error(shards);
    mark("finalize + download");
    uint64_t n_rows = 0;
    long long removed_reads = 0, removed_bases = 0;
    for (auto &s : shards) {
        n_rows += s.n_rows - s.contam.rows;
        removed_reads += (long long)s.contam.reads;
        removed_bases += (long long)s.contam.bases;
    }
    log_after_trim_split(args, n_rows, shards[0].summary);
    if (args.contam_set) print_contam_removal(args.max_contam, removed_reads, removed_bases, args.contam_k);
    log_filtering(args, shards[0].summary);
}

}  // namespace

FeederOutcome run_device_feeder(Arguments &args, Kmers &kmers, StreamInput *stream, const Mark &mark) {
    FeederOutcome res;
    MappedFile own;
    const Source src = choose_source(args, kmers, stream, own, mark);
    if (args.keep_mods && src.format != FL_FORMAT_BAM) throw std::runtime_error("--keep_mods needs BAM input");
    if (args.aligned && src.format != FL_FORMAT_BAM) throw std::runtime_error("--aligned needs BAM input");
    if (!src.file) return res;
    const MappedFile &f = *src.file;
    const bool bam = src.format == FL_FORMAT_BAM;
    Cuts cuts;
    Plan plan;
    if (!plan_input(src, plan, cuts, mark)) return res;
    std::vector<BamChunkIndex> bam_idx(bam ? plan.chunks.size() : 0);
    const ChunkPush push = bam ? bam_push(f.base, bam_idx, args.aligned) : text_push(src.format);
    ShardSet shards(plan.chunks, f.size, args.gpus, src.growing);
    const bool kmers_empty = kmers.empty();
    const bool declined = score(shards.v, src, cuts, plan, push, args, kmers, !kmers_empty, kmers.contam_size() > 0);
    std::string why;
    if (src.growing && !stream->finish(&why)) throw std::runtime_error(why);
    throw_shard_error(shards.v);
    if (declined) {                                                     // not the simple layout after all: start over on the host
        if (shards.v[0].ctx) fl_reads_reset(shards.v[0].ctx);
        return res;
    }
    mark(bam ? "pass 1 (BAM records + score)" : "pass 1 (device parse + score)");
    res.handled = true;
    std::cerr << "Scoring long reads\n";
    uint64_t orphans = 0;
    const std::string error = check_records(shards.v, f.base, bam, kmers_empty, &orphans);
    if (!error.empty()) {
        std::cerr << error;
        res.exit_code = 1;
        return res;
    }
    long long n_reads = 0, total_bases = 0;
    for (auto &s : shards.v) {
        n_reads += (long long)s.rec.n;
        for (size_t i = 0; i < s.rec.n; ++i) total_bases += s.rec.len[i];
    }
    print_read_score_progress(n_reads, total_bases);
    std::cerr << "\n";
    mark("duplicate-name check");
    finalize(shards.v, args, mark);
    // ---- pass 2 ----
    std::cerr << "Outputting passed long reads\n";
    std::vector<Part> parts;
    for (auto &s : shards.v) parts.push_back(Part{&s.rec, Results::of(s), args.aligned ? &s.followers : nullptr});
    const Format fmt{src.format == FL_TEXT_FASTA ? '>' : '@', src.format == FL_TEXT_FASTQ, bam, cuts.bam_header, cuts.bam_max_record, args.keep_mods};
    fl_ctx *bgzf = args.bgzip || bam ? shards.v[0].ctx : nullptr;      // BAM in, BAM out: always BGZF (--bgzip changes nothing)
    res.exit_code = write_outputs(args, g_out_fd, f.base, parts, fmt, bgzf) ? 0 : 1;
    if (orphans)
        std::cerr << "  secondary or supplementary records without their read in the input: " << int_to_string((long long)orphans)
                  << " (not written to stdout)\n";
    mark("pass 2 (slices of the mapped input)");
    std::cerr << "\n";
    return res;
}

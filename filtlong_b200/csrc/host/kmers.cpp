// filtlong_b200/csrc/host/kmers.cpp -- see kmers.h. Log lines follow reference src/kmers.cpp:50-72.
#include "kmers.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <iostream>
#include <memory>
#include <stdexcept>

#include "arena.h"
#include "fastx.h"
#include "misc.h"
#include "textsrc.h"

void Kmers::check(fl_ctx *ctx, int rc, const char *what) {
    if (rc == FL_OK) return;
    throw std::runtime_error(std::string(what) + ": " + fl_last_error(ctx));
}

Kmers::Kmers() : Kmers(0) {}

Kmers::Kmers(int device) : device_(device) {}

fl_ctx *Kmers::context() {
    if (!ctx_) {
        fl_params p{};
        p.window_size = 250;
        p.length_weight = p.mean_q_weight = p.window_q_weight = 1.0;
        int rc = fl_ctx_create(&p, device_, &ctx_);
        if (rc != FL_OK) throw std::runtime_error(std::string("fl_ctx_create: ") + fl_last_error(nullptr));
    }
    return ctx_;
}

// The threshold is DESIGN §7's CLI sweep on an H100 (`filtlong -p 90` on one member of C2-like FASTQ at level 1, wall-clock,
// best and median of 3 alternated runs): from 64 MiB compressed both favour the GPU inflater (256 MiB: 2.0 s against
// 4.0 s); at 16 MiB and below the two are within the runs' spread, so the host z_stream keeps those files.
// FL_GUNZIP_HOST=1 keeps every file on the host z_stream; FL_GUNZIP_MIN_BYTES=N moves the threshold (measurement only:
// the bytes are the same either way).
GzipDeviceInflate Kmers::device_inflater() {
    return [this](const unsigned char *d, uint64_t n, char *out, uint64_t cap, GzipDeviceResult *r) {
        uint64_t min_bytes = kDeviceGunzipMinBytes;
        if (const char *e = getenv("FL_GUNZIP_MIN_BYTES")) min_bytes = strtoull(e, nullptr, 10);
        if (n < min_bytes) { r->note = "host zlib (under the GPU inflater's threshold)"; return false; }
        if (getenv("FL_GUNZIP_HOST")) { r->note = "host zlib (FL_GUNZIP_HOST)"; return false; }
        fl_ctx *c = nullptr;
        try {
            c = context();
        } catch (const std::exception &) {
            r->note = "host zlib (no CUDA context)";
            return false;
        }
        uint64_t got = 0;
        int status = FL_GUNZIP_DECLINED;
        fl_gunzip_stats st{};
        const int rc = fl_gzip_inflate(c, d, n, out, cap, 0, 0, &got, &status, &st);
        char buf[200];
        if (rc != FL_OK) {
            snprintf(buf, sizeof buf, "host zlib (GPU inflater failed: %.120s)", fl_last_error(c));
            r->note = buf;
            return false;
        }
        snprintf(buf, sizeof buf, "%s: %llu chunks, %llu re-decoded, %llu rounds",
                 status == FL_GUNZIP_OK ? "GPU inflater" : "host zlib (GPU inflater declined)", (unsigned long long)st.chunks,
                 (unsigned long long)st.redecoded, (unsigned long long)st.rounds);
        r->note = buf;
        if (status != FL_GUNZIP_OK) return false;
        r->n_out = got;
        r->members = st.members;
        return true;
    };
}

Kmers::~Kmers() {
    if (ctx_) fl_ctx_destroy(ctx_);
}

uint64_t Kmers::size() {
    if (!ctx_) return 0;                                               // nothing was ever added
    uint64_t n = 0;
    check(ctx_, fl_kmers_finalize(ctx_, &n), "fl_kmers_finalize");
    return n;
}

void Kmers::add_read_fastqs(std::vector<std::string> filenames) {
    std::cerr << "Hashing 16-mers from short reads\n";
    int sequence_count = 0;
    for (auto &filename : filenames) sequence_count += add_reference(filename, true);
    const long long n_kmers = (long long)size();                      // resolves the multiple-copy rule (kmers.cpp:142-166)
    // the 49 GiB of transient counting state are not needed for scoring (the reference's count map is
    // likewise dead after hashing, it just never frees it: kmers.h:48-49)
    if (ctx_) check(ctx_, fl_kmers_release_build_state(ctx_), "fl_kmers_release_build_state");
    std::cerr << "  " << int_to_string(sequence_count) << " reads, " << int_to_string(n_kmers) << " 16-mers\n\n";
}

void Kmers::add_assembly_fasta(std::string filename) {
    std::cerr << "Hashing 16-mers from assembly\n";
    std::cerr << "  " << filename << "\n";
    int sequence_count = add_reference(filename, false);
    std::cerr << "  " << int_to_string(sequence_count) << " " << (sequence_count == 1 ? "contig" : "contigs") << ", "
              << int_to_string((long long)size()) << " 16-mers\n\n";
}

uint64_t Kmers::contam_size() {
    if (!ctx_) return 0;
    uint64_t n = 0;
    check(ctx_, fl_contam_finalize(ctx_, &n), "fl_contam_finalize");
    return n;
}

// The same block as add_assembly_fasta's (kmers.cpp:61-72), then the chance that a base of random sequence lies in one
// of the set's k-mers: 1 - (1 - n / 4^k)^k. The 16-mers of a genome the size of a human one cover almost every base, which
// removes everything; its 31-mers cover about one base in 2^26.
void Kmers::add_contaminant_fasta(const std::string &filename, int k) {
    contam_k_ = k;
    std::cerr << "Hashing " << k << "-mers from contaminant sequences\n";
    std::cerr << "  " << filename << "\n";
    const int sequence_count = add_reference(filename, false, true);
    const uint64_t n = contam_size();
    std::cerr << "  " << int_to_string(sequence_count) << " " << (sequence_count == 1 ? "contig" : "contigs") << ", "
              << int_to_string((long long)n) << " " << k << "-mers\n";
    const double covered = -expm1((double)k * log1p(-(double)n / ldexp(1.0, 2 * k)));
    char buf[96];
    snprintf(buf, sizeof buf, "  a random base lies in one of them with probability %.3g\n\n", covered);
    std::cerr << buf;
}

// The reference's loop (kmers.cpp:75-134) parses one record at a time through kseq on the calling thread. Here the file
// is one byte range (mapped, or a gzip file inflated once: textsrc.h) whose record-aligned chunks go to the device as
// TEXT (fl_kmers_add_text): records (4-line FASTQ; FASTA with one sequence line or evenly wrapped), validation, 2-bit
// packing and the non-ACGT mask all happen there. The first chunk that is not in that layout (CR LF, ragged or blank
// lines, a broken record ...) -- and everything after it -- is parsed
// by the kseq-compatible host reader from that chunk's first byte, so the adds stay in file order and the reader stops
// where the reference's would (a parse error silently ends hashing: kmers.cpp:90-94).
int Kmers::add_reference(const std::string &filename, bool multi, bool contam) {
    int sequence_count = 0;
    long long base_count = 0, last_progress = 0;
    auto progress = [&](bool force) {
        if (force || base_count - last_progress >= 483611) {           // the reference's progress cadence (kmers.cpp:123-126)
            last_progress = base_count;
            print_hash_progress(filename, base_count);
        }
    };
    // A contaminant set of k > 16 is a hash table sized before its first add (fl_contam_configure): by the file's bytes
    // (after inflation), which bound its bases, when the file is in memory; otherwise by its bases, read once by the host
    // parser into packed batches that are held until the whole input is in (a pipe cannot be read twice).
    const bool sized = contam && contam_k_ > 16;
    auto configure = [&](uint64_t bound) {
        contam_max_kmers_ = bound > 0 ? bound : 1;
        check(context(), fl_contam_configure(context(), contam_k_, contam_max_kmers_), "fl_contam_configure");
    };
    // the host parser over `in`, feeding packed batches (fl_kmers_add_batch); hold_all: size the set first (see above)
    auto host_parse = [&](FastxReader &in, bool hold_all) {
        const uint64_t kBatchBases = 256ull << 20;
        std::vector<std::unique_ptr<HostArena>> held;
        auto arena = std::make_unique<HostArena>(true, false, true);
        auto add = [&](const HostArena &a) {
            fl_batch b = a.batch();
            fl_ctx *c = context();
            if (contam) check(c, fl_contam_add_batch(c, &b), "fl_contam_add_batch");
            else check(c, fl_kmers_add_batch(c, &b, multi ? 1 : 0), "fl_kmers_add_batch");
        };
        auto flush = [&]() {
            if (arena->empty()) return;
            if (hold_all) {
                held.push_back(std::move(arena));
                arena = std::make_unique<HostArena>(true, false, true);
                return;
            }
            add(*arena);
            arena->clear();
        };
        while (in.ok() && in.next() >= 0) {        // a parse error silently ends hashing (kmers.cpp:90-94)
            ++sequence_count;
            if (in.seq.size() < 16) continue;      // kmers.cpp:99-100
            base_count += (long long)in.seq.size();
            arena->add(in.seq.data(), nullptr, (int64_t)in.seq.size());
            if (arena->padded_bases() >= kBatchBases) flush();
            progress(false);
        }
        flush();
        if (!hold_all) return;
        uint64_t bases = 0;
        for (const auto &a : held) bases += a->bases();
        configure(bases);
        for (auto &a : held) {
            add(*a);
            a.reset();
        }
    };
    MappedFile f;
    std::vector<Chunk> plan;
    const bool timing = getenv("FL_CLI_TIMING") != nullptr;
    bool inflated = false;
    bool text_path = !getenv("FL_HOST_PARSER") && f.open_any(filename, &inflated, nullptr, device_inflater()) &&
                     (f.format() == FL_TEXT_FASTQ || f.format() == FL_TEXT_FASTA);
    if (timing && inflated) std::cerr << "[timing] reference " << filename << ": gzip input inflated into memory, " << f.inflater << "\n";
    if (text_path) {
        // a chunk holds whole records: FASTA chunks are large enough for a chromosome on one line or wrapped
        const uint64_t target = chunk_target(f.format() == FL_TEXT_FASTA ? 512ull << 20 : 128ull << 20);
        text_path = plan_chunks(f.base, f.size, f.format(), target, target, plan) && !plan.empty();
    }
    if (text_path) {
        fl_ctx *c = context();
        if (sized) configure(f.size);
        for (size_t i = 0; i < plan.size(); ++i) {
            const Chunk &ch = plan[i];
            uint64_t n_rec = 0, n_bases = 0, used = 0;
            int status = FL_TEXT_OK;
            const int last = i + 1 == plan.size() ? 1 : 0;
            if (contam)
                check(c, fl_contam_add_text(c, f.base + ch.begin, ch.end - ch.begin, f.format(), last, &n_rec, &n_bases, &used, &status),
                      "fl_contam_add_text");
            else
                check(c, fl_kmers_add_text(c, f.base + ch.begin, ch.end - ch.begin, f.format(), last, multi ? 1 : 0, &n_rec, &n_bases, &used,
                                           &status), "fl_kmers_add_text");
            if (status == FL_TEXT_OK) {                                 // the chunk's whole records (all of it, normally) are in
                sequence_count += (int)n_rec;
                base_count += (long long)n_bases;
                progress(false);
            } else {
                used = 0;                                               // not the layout: nothing of this chunk was added
            }
            if (used != ch.end - ch.begin) {                            // the host reader takes over at the first byte not consumed
                if (timing) std::cerr << (last_progress ? "\n" : "") << "[timing] reference " << filename << ": host reader from byte " << ch.begin + used << "\n";
                FastxReader in(f.base + ch.begin + used, f.size - ch.begin - used);
                host_parse(in, false);
                break;
            }
            if (timing && i + 1 == plan.size())
                std::cerr << (last_progress ? "\n" : "") << "[timing] reference " << filename << ": device text, " << plan.size() << " chunks\n";
        }
    } else {
        if (timing) std::cerr << "[timing] reference " << filename << ": host reader\n";
        FastxReader in(filename);
        host_parse(in, sized);
    }
    progress(true);
    std::cerr << "\n";
    return sequence_count;
}

bool Kmers::is_kmer_present(uint32_t kmer) {
    uint8_t out = 0;
    if (!ctx_) return false;
    check(ctx_, fl_kmers_contains(ctx_, &kmer, 1, &out), "fl_kmers_contains");
    return out != 0;
}

uint32_t Kmers::base_to_bits_forward(char base) {          // kmers.cpp:176-196
    switch (base) {
        case 'C': case 'c': return 1u;
        case 'G': case 'g': return 2u;
        case 'T': case 't': return 3u;
        default: return 0u;
    }
}

uint32_t Kmers::base_to_bits_reverse(char base) {          // kmers.cpp:199-219
    switch (base) {
        case 'G': case 'g': return 1u << 30;
        case 'C': case 'c': return 2u << 30;
        case 'A': case 'a': return 3u << 30;
        default: return 0u;
    }
}

uint32_t Kmers::starting_kmer_to_bits_forward(char *sequence) {
    uint32_t kmer = 0;
    for (int i = 0; i < 16; ++i) kmer = (kmer << 2) | base_to_bits_forward(sequence[i]);
    return kmer;
}

uint32_t Kmers::starting_kmer_to_bits_reverse(char *sequence) {
    uint32_t kmer = 0;
    for (int i = 0; i < 16; ++i) kmer = (kmer >> 2) | base_to_bits_reverse(sequence[i]);
    return kmer;
}

// filtlong_b200/csrc/host/main.cpp -- the `filtlong` command line on an H100.
//
// Same flow, same stderr log and same stdout as the reference's main (reference
// src/main.cpp:37-321), restructured around batches: records are parsed and packed on the host,
// scored on the GPU batch by batch (instead of one `new Read` per record, main.cpp:108), and the
// normalise / sort / threshold block (main.cpp:169-261) is one fl_finalize call. Pass 2 re-reads
// the input and prints the survivors exactly like main.cpp:263-313.
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "arguments.h"
#include "bgzf_out.h"
#include "fastx.h"
#include "feeder.h"
#include "kmers.h"
#include "misc.h"
#include "read.h"

#define PROGRAM_VERSION "0.3.1"

// FL_CLI_TIMING=1: wall-clock seconds per phase on stderr after the run (never on by default: the
// stderr log is part of the drop-in surface)
namespace {
struct PhaseTimer {
    bool on = getenv("FL_CLI_TIMING") != nullptr;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now(), last = t0;
    std::string report;
    void mark(const char *what) {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        char buf[128];
        snprintf(buf, sizeof buf, "[timing] %-28s %8.3f s\n", what, std::chrono::duration<double>(now - last).count());
        report += buf;
        last = now;
    }
    ~PhaseTimer() {
        if (!on) return;
        char buf[128];
        snprintf(buf, sizeof buf, "[timing] %-28s %8.3f s\n", "total", std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
        fputs((report + buf).c_str(), stderr);
    }
};
}  // namespace

int main(int argc, char **argv) {
    Arguments args(argc, argv);
    if (args.parsing_result == BAD) return 1;
    else if (args.parsing_result == HELP) return 0;
    else if (args.parsing_result == VERSION) {
        std::cout << "Filtlong v" << PROGRAM_VERSION << "\n";
        return 0;
    }
    std::ios::sync_with_stdio(false);
    std::cerr << "\n";
    PhaseTimer timer;
    // The CUDA driver and context take about a second to come up: start that now, on
    // its own thread, and parse / pack the first records meanwhile (Kmers creates its context on
    // first use). Joined on every way out of main.
    struct Warmup {
        std::thread t{[] { (void)fl_device_warmup(0); }};
        ~Warmup() { if (t.joinable()) t.join(); }
    } warmup;
    try {
        Kmers kmers;                                                      // main.cpp:53-59
        if (args.assembly_set) kmers.add_assembly_fasta(args.assembly);
        if (!args.short_reads.empty()) kmers.add_read_fastqs(args.short_reads);
        const bool kmers_empty = kmers.empty();
        timer.mark("reference k-mers (+ CUDA init)");

        // ---- the device-first input path: the file as text to the device, survivors by writev from the mapping ----
        {
            const FeederOutcome fo = run_text_feeder(args, kmers, [&](const char *what) { timer.mark(what); });
            if (fo.handled) return fo.exit_code;
        }

        // ---- pass 1: parse, pack and score (main.cpp:61-130) ----
        long long total_bases = 0, last_progress = 0;
        if (!args.verbose) std::cerr << "Scoring long reads\n";
        ReadSet reads(&kmers, &args);
        std::unordered_set<std::string> seen_names;
        bool any_fasta = false, any_fastq = false;
        const unsigned long long kBatchBases = 512ull << 20;
        reads.reserve(kBatchBases + (4ull << 20), 1u << 18);
        unsigned long long queued = 0;
        size_t verbose_done = 0;
        // where each record's comment / sequence / quality sit in the input, when the reader can vouch
        // for it (uncompressed file, single-line records): pass 2 then copies slices of the mapped file
        // instead of parsing it a second time
        bool slices_ok = true;
        std::vector<uint64_t> rec_comment_off, rec_seq_off, rec_qual_off;
        std::vector<uint32_t> rec_comment_len;
        auto verbose_flush = [&]() {
            if (!args.verbose) return;
            reads.download();
            for (; verbose_done < reads.n_reads(); ++verbose_done) {
                Read *r = reads.make_read(verbose_done);
                r->print_verbose_read_info();                             // main.cpp:110-111
                delete r;
            }
        };
        {
            FastxReader in(args.input_reads);
            while (true) {
                int64_t l64 = in.ok() ? in.next() : -1;
                int l = (int)l64;                                         // main.cpp:69,77 (int truncation)
                if (l == -1) break;
                if (l == -2) {
                    verbose_flush();
                    std::cerr << "Error: incorrect FASTQ format for read " << in.name << "\n";
                    return 1;
                }
                if (l == -3) {
                    std::cerr << "Error reading " << args.input_reads << "\n";
                    return 1;
                }
                total_bases += (long long)in.seq.size();
                const bool fasta_format = in.qual.empty() && !in.seq.empty();
                const bool fastq_format = !in.qual.empty() && !in.seq.empty() && in.qual.size() == in.seq.size();
                any_fasta = any_fasta || fasta_format;
                any_fastq = any_fastq || fastq_format;
                if (any_fasta && any_fastq) {
                    std::cerr << "\n\n" << "Error: could not parse input reads" << "\n";
                    std::cerr << "  problem occurred at read " << in.name << "\n";
                    return 1;
                }
                if (fasta_format && kmers_empty) {
                    std::cerr << "\n\n" << "Error: FASTA input not supported without an external reference" << "\n";
                    return 1;
                }
                if (slices_ok) {
                    if (in.simple && in.plain() && in.comment.size() < (1u << 31)) {
                        rec_comment_off.push_back(in.comment_off);
                        rec_comment_len.push_back((uint32_t)in.comment.size());
                        rec_seq_off.push_back(in.seq_off);
                        rec_qual_off.push_back(in.qual_off);
                    } else {
                        slices_ok = false;
                        rec_comment_off.clear(); rec_comment_len.clear(); rec_seq_off.clear(); rec_qual_off.clear();
                    }
                }
                // Phred mode needs a quality byte per base; an empty record has neither
                reads.add(in.name, in.seq.data(), in.qual.empty() ? (kmers_empty ? "" : nullptr) : in.qual.data(), (int)in.seq.size());
                if (!seen_names.insert(in.name).second) {
                    verbose_flush();
                    std::cerr << "Error: duplicate read name: " << in.name << "\n";
                    return 1;
                }
                queued += in.seq.size();
                if (queued >= kBatchBases) {
                    reads.flush();
                    queued = 0;
                    verbose_flush();
                }
                if (total_bases - last_progress >= 483611) {
                    last_progress = total_bases;
                    if (!args.verbose) print_read_score_progress((long long)reads.n_reads(), total_bases);
                }
            }
        }
        reads.flush();
        timer.mark("pass 1 (parse, pack, push)");
        verbose_flush();
        if (!args.verbose) print_read_score_progress((long long)reads.n_reads(), total_bases);
        std::cerr << "\n";
        const bool fasta_output = any_fasta, fastq_output = any_fastq;

        // ---- normalise, final score, target (main.cpp:136-261), on the GPU ----
        fl_summary summary = reads.finalize(total_bases);
        timer.mark("finalize + download");
        size_t longest_read_name = 0;
        if (args.verbose)
            for (size_t row = 0; row < reads.n_rows(); ++row) longest_read_name = std::max(longest_read_name, reads.row_name(row).size());
        if (args.trim || args.split_set) {
            if (args.trim && args.split_set) std::cerr << "  after trimming and splitting: ";
            else if (args.trim) std::cerr << "  after trimming: ";
            else std::cerr << "  after splitting: ";
            std::cerr << int_to_string((long long)reads.n_rows()) << " reads (" << int_to_string(summary.rows_bases) << " bp)\n";
        }
        std::cerr << "\n";
        if (args.verbose) {
            std::cerr << "\n\n" << "Read name" << "\t" << "Length score" << "\t" << "Mean quality score" << "\t"
                      << "Window quality score" << "\t" << "Final score" << "\n";
            for (size_t row = 0; row < reads.n_rows(); ++row) {
                std::string nm = reads.row_name(row);
                if (longest_read_name > nm.size()) nm += std::string(longest_read_name - nm.size(), ' ');
                std::cerr << nm << "\t" << double_to_string(reads.row_lscore[row]) << "\t" << double_to_string(reads.row_nmean[row])
                          << "\t" << double_to_string(reads.row_nwindow[row]) << "\t" << double_to_string(reads.row_final[row]) << "\n";
            }
            std::cerr << "\n";
        }
        if (args.target_bases_set || args.keep_percent_set) {
            std::cerr << "Filtering long reads\n";
            std::cerr << "  target: " << int_to_string(summary.target) << " bp\n";
            if (summary.status == 1) std::cerr << "  not enough reads to reach target\n";
            else if (summary.status == 2) std::cerr << "  reads already fall below target after filtering\n";
            else std::cerr << "  keeping " << int_to_string(summary.keeping) << " bp\n";
            std::cerr << "\n";
        }

        // ---- pass 2: output the keepers in input order (main.cpp:263-313) ----
        std::cerr << "Outputting passed long reads\n";
        std::unique_ptr<BgzfOut> zout;                                    // --bgzip: compressed on the scoring context's GPU
        if (args.bgzip) zout.reset(new BgzfOut(kmers.context(), 1));
        auto write_out = [&](const std::string &o) {
            if (zout) zout->put(o.data(), o.size());
            else fwrite(o.data(), 1, o.size(), stdout);
        };
        bool printed = false;
        if (slices_ok && rec_seq_off.size() == reads.n_reads() && reads.n_reads() > 0) {
            // same bytes as the loop below, taken from the mapped input at the offsets pass 1 recorded
            const int fd = open(args.input_reads.c_str(), O_RDONLY);
            struct stat st;
            if (fd >= 0 && fstat(fd, &st) == 0 && st.st_size > 0) {
                void *mp = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
                if (mp != MAP_FAILED) {
                    const char *base = (const char *)mp;
                    const uint64_t fsize = (uint64_t)st.st_size;
                    bool in_bounds = true;
                    for (size_t i = 0; i < reads.n_reads() && in_bounds; ++i) {
                        const uint64_t L = (uint64_t)reads.length[i];
                        in_bounds = rec_seq_off[i] + L <= fsize && (!fastq_output || rec_qual_off[i] + L <= fsize) &&
                                    rec_comment_off[i] + rec_comment_len[i] <= fsize;
                    }
                    if (in_bounds) {
                        std::string out;
                        out.reserve(1 << 20);
                        auto emit = [&](size_t i, const std::string &nm, int start, int length) {
                            out += fasta_output ? '>' : '@';
                            out += nm;
                            if (rec_comment_len[i]) { out += ' '; out.append(base + rec_comment_off[i], rec_comment_len[i]); }
                            out += '\n';
                            out.append(base + rec_seq_off[i] + start, (size_t)length);
                            out += '\n';
                            if (fastq_output) { out += "+\n"; out.append(base + rec_qual_off[i] + start, (size_t)length); out += '\n'; }
                        };
                        for (size_t i = 0; i < reads.n_reads(); ++i) {
                            const size_t rs = (size_t)reads.row_start[i];
                            if (reads.n_child[i] == 0) {
                                if (reads.row_pfinal[rs]) emit(i, reads.names[i], 0, reads.length[i]);
                            } else {
                                for (int c = 0; c < reads.n_child[i]; ++c) {
                                    const size_t row = rs + (size_t)c;
                                    if (!reads.row_pfinal[row]) continue;
                                    const int start = reads.row_s[row], length = reads.row_e[row] - reads.row_s[row];
                                    if (length <= 0) continue;
                                    emit(i, reads.row_name(row), start, length);
                                }
                            }
                            if (out.size() >= (1 << 20)) { write_out(out); out.clear(); }
                        }
                        write_out(out);
                        fflush(stdout);
                        printed = true;
                    }
                    munmap(mp, (size_t)st.st_size);
                }
            }
            if (fd >= 0) close(fd);
        }
        if (!printed) {
            FastxReader in(args.input_reads);
            size_t i = 0;
            std::string out;
            out.reserve(1 << 20);
            while (in.ok() && in.next() >= 0 && i < reads.n_reads()) {
                const size_t rs = (size_t)reads.row_start[i];
                if (reads.n_child[i] == 0) {
                    if (reads.row_pfinal[rs]) {
                        out += fasta_output ? '>' : '@';
                        out += in.name;
                        if (!in.comment.empty()) { out += ' '; out += in.comment; }
                        out += '\n';
                        out += in.seq;
                        out += '\n';
                        if (fastq_output) { out += "+\n"; out += in.qual; out += '\n'; }
                    }
                } else {
                    for (int c = 0; c < reads.n_child[i]; ++c) {
                        const size_t row = rs + (size_t)c;
                        if (!reads.row_pfinal[row]) continue;
                        const int start = reads.row_s[row], length = reads.row_e[row] - reads.row_s[row];
                        if (length <= 0) continue;
                        out += fasta_output ? '>' : '@';
                        out += reads.row_name(row);
                        if (!in.comment.empty()) { out += ' '; out += in.comment; }
                        out += '\n';
                        out.append(in.seq, (size_t)start, (size_t)length);
                        out += '\n';
                        if (fastq_output) { out += "+\n"; out.append(in.qual, (size_t)start, (size_t)length); out += '\n'; }
                    }
                }
                if (out.size() >= (1 << 20)) { write_out(out); out.clear(); }
                ++i;
            }
            write_out(out);
            fflush(stdout);
        }
        if (zout && !zout->finish()) {
            if (!zout->error().empty()) std::cerr << "Error: " << zout->error() << "\n";
            return 1;
        }
        timer.mark("pass 2 (parse, print)");
        std::cerr << "\n";
    } catch (const std::exception &e) {
        std::cerr << "\nError: " << e.what() << "\n";
        return 1;
    }
    return 0;
}

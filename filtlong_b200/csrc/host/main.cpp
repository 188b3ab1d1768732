// filtlong_b200/csrc/host/main.cpp -- the `filtlong` command line on an H100.
//
// Same flow, same stderr log and same stdout as the reference's main (reference src/main.cpp:37-321). The device feeder
// (feeder.h) takes the input reads when the GPU can parse them; whatever it declines, the host path below parses with
// FastxReader and scores on the GPU batch by batch (instead of one `new Read` per record, main.cpp:108). On both, the
// normalise / sort / threshold block (main.cpp:169-261) is one fl_finalize call, and pass 2 prints the survivors exactly
// like main.cpp:263-313, from slices of the input when every record's place is known, else from a second parse.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "arguments.h"
#include "fastx.h"
#include "feeder.h"
#include "kmers.h"
#include "misc.h"
#include "read.h"
#include "streamsrc.h"
#include "survivors.h"
#include "textsrc.h"

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
    void note(const char *what) {
        if (on) report += std::string("[timing] ") + what + "\n";
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
    // Input that can be read only once (a pipe, standard input) is held in memory; reading it starts now, so that its
    // producer is not blocked on a full pipe while the reference k-mers are built
    StreamInput stream;
    const bool streamed = stream_input(&args.input_reads);
    // The CUDA driver and context take about a second to come up: start that now, on
    // its own thread, and parse / pack the first records meanwhile (Kmers creates its context on
    // first use). Joined on every way out of main.
    struct Warmup {
        std::thread t{[] { (void)fl_device_warmup(0); }};
        ~Warmup() { if (t.joinable()) t.join(); }
    } warmup;
    try {
        if (streamed) stream.start(args.input_reads);
        Kmers kmers;                                                      // main.cpp:53-59
        if (args.assembly_set) kmers.add_assembly_fasta(args.assembly);
        if (!args.short_reads.empty()) kmers.add_read_fastqs(args.short_reads);
        const bool kmers_empty = kmers.empty();
        if (args.contam_set) kmers.add_contaminant_fasta(args.contam, args.contam_k);   // after -1/-2, whose build state is released by now
        timer.mark("reference k-mers (+ CUDA init)");

        // ---- the device feeder ----
        {
            const FeederOutcome fo = run_device_feeder(args, kmers, streamed ? &stream : nullptr, [&](const char *what) { timer.mark(what); });
            if (streamed) {
                char buf[160];
                snprintf(buf, sizeof buf, "stream: %llu bytes, %zu of %zu chunks scored before its end",
                         (unsigned long long)stream.stream_bytes(), stream.chunks_before_end.load(), stream.chunks.load());
                timer.note(buf);
            }
            if (fo.handled) return fo.exit_code;
        }
        // ---- the host path: a stream is parsed from its bytes in memory, a file by its path ----
        std::string why;
        if (streamed && !stream.finish(&why, kmers.device_inflater())) throw std::runtime_error(why);
        const MappedFile &mem = stream.file();
        const FastxInput reads_in = streamed ? FastxInput(mem.base, mem.size) : FastxInput(args.input_reads);

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
        // where each record sits in the input, when the reader can vouch for it (uncompressed file,
        // single-line records): pass 2 then copies slices of the mapped file instead of parsing it a
        // second time
        bool table_ok = true;
        Records table;
        auto verbose_flush = [&]() {
            if (!args.verbose) return;
            reads.download();
            for (; verbose_done < reads.n_reads(); ++verbose_done) {
                if (reads.removed[verbose_done]) continue;                // --contam: as if the read were not in the input
                Read *r = reads.make_read(verbose_done);
                r->print_verbose_read_info();                             // main.cpp:110-111
                delete r;
            }
        };
        {
            const std::unique_ptr<FastxReader> reader = reads_in.open();
            FastxReader &in = *reader;
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
                if (table_ok) {
                    if (in.simple && in.plain() && in.comment.size() < (1u << 31) && in.name.size() < (1u << 31)) {
                        table.add(in.name_off, (uint32_t)in.name.size(), (uint32_t)in.comment.size(), in.seq_off, in.qual_off,
                                  (int32_t)in.seq.size());
                    } else {
                        table_ok = false;
                        table = Records();
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

        // ---- normalise, final score, target (main.cpp:136-261), on the GPU ----
        fl_summary summary = reads.finalize(total_bases);
        timer.mark("finalize + download");
        size_t longest_read_name = 0;
        if (args.verbose)
            for (size_t row = 0; row < reads.n_rows(); ++row)
                if (reads.ranked(row)) longest_read_name = std::max(longest_read_name, reads.row_name(row).size());
        log_after_trim_split(args, reads.n_rows() - reads.contam.rows, summary);
        if (args.contam_set) print_contam_removal(args.max_contam, (long long)reads.contam.reads, (long long)reads.contam.bases, args.contam_k);
        if (args.verbose) {
            std::cerr << "\n\n" << "Read name" << "\t" << "Length score" << "\t" << "Mean quality score" << "\t"
                      << "Window quality score" << "\t" << "Final score" << "\n";
            for (size_t row = 0; row < reads.n_rows(); ++row) {
                if (!reads.ranked(row)) continue;                        // a removed read's rows are not ranked
                std::string nm = reads.row_name(row);
                if (longest_read_name > nm.size()) nm += std::string(longest_read_name - nm.size(), ' ');
                std::cerr << nm << "\t" << double_to_string(reads.row_lscore[row]) << "\t" << double_to_string(reads.row_nmean[row])
                          << "\t" << double_to_string(reads.row_nwindow[row]) << "\t" << double_to_string(reads.row_final[row]) << "\n";
            }
            std::cerr << "\n";
        }
        log_filtering(args, summary);

        // ---- pass 2: output the keepers in input order (main.cpp:263-313) ----
        std::cerr << "Outputting passed long reads\n";
        const Format fmt{any_fasta ? '>' : '@', any_fastq};
        fl_ctx *bgzf = args.bgzip ? kmers.context() : nullptr;           // --bgzip: compressed on the scoring context's GPU
        MappedFile f;
        const MappedFile &src = streamed ? mem : f;
        bool ok;
        if (table_ok && (streamed || f.open_plain(args.input_reads)) && table.within(src.size, fmt.quality)) {
            ok = write_outputs(args, 1, src.base, {Part{&table, Results::of(reads)}}, fmt, bgzf);
        } else {                                                         // --failed: the other rows, from the same parse
            bool failed_ok = true;
            ok = reparse_survivors(1, reads_in, Results::of(reads), reads.n_reads(), fmt, bgzf, args.failed_fd, &failed_ok);
            if (!report_failed_write(args, failed_ok)) ok = false;
        }
        timer.mark("pass 2 (parse, print)");
        std::cerr << "\n";
        if (!ok) return 1;
    } catch (const std::exception &e) {
        std::cerr << "\nError: " << e.what() << "\n";
        return 1;
    }
    return 0;
}

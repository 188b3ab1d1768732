// filtlong_b200/csrc/host/read.h -- drop-in for the reference's Read (reference src/read.h:29-65):
// same constructor signature, same public data members and methods. All scoring happens on the GPU
// behind the C ABI; a Read object is a host-side record of the result rows.
//
//   Deviations from the reference's object, both invisible to main(): (1) a child's m_first_base_in_kmer /
//   m_last_base_in_kmer are -1 (the reference's child re-runs the constructor and computes its own; nothing
//   reads them); (2) constructing a Read scores on the Kmers' context and forgets whatever a ReadSet had
//   pushed there: use one or the other on a given Kmers, not both.
//   Read(name, seq, qscores, length, kmers, args)   scores ONE read synchronously (one small batch
//       through fl_reads_push): signature-compatible, meant for callers and tests written against
//       the reference. Throughput code uses ReadSet below, which scores a whole batch per call and
//       materialises Read objects from the result rows.
#pragma once
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "arguments.h"
#include "kmers.h"

class ReadSet;

class Read {
public:
    Read(std::string name, char *seq, char *qscores, int length, Kmers *kmers, Arguments *args);   // read.h:32
    ~Read();
    Read(const Read &) = delete;
    Read &operator=(const Read &) = delete;

    void print_verbose_read_info();                                            // read.h:35
    void print_scores(size_t name_length);                                     // read.h:36
    void set_final_score(double length_weight, double mean_q_weight, double window_q_weight);   // read.h:38

    std::string m_name;                                                        // read.h:40-56
    int m_length;
    double m_length_score;
    double m_mean_quality;
    double m_window_quality;
    double m_final_score;
    bool m_passed;
    int m_first_base_in_kmer;
    int m_last_base_in_kmer;
    std::vector<std::pair<int, int> > m_bad_ranges;
    std::vector<Read *> m_child_reads;
    std::vector<std::pair<int, int> > m_child_read_ranges;

private:
    friend class ReadSet;
    Read() {}
};

// fl_params from the parsed command line
fl_params params_from_arguments(const Arguments &args);

// Batch-granular scoring: push records, then finalize(), then read the result rows.
class ReadSet {
public:
    ReadSet(Kmers *kmers, Arguments *args);
    ~ReadSet();
    ReadSet(const ReadSet &) = delete;
    ReadSet &operator=(const ReadSet &) = delete;
    // queues one record (buffers are copied / packed inside the call, like read.cpp does with kseq's)
    void add(const std::string &name, const char *seq, const char *qscores, int length);
    void reserve(uint64_t bases, uint32_t reads);  // capacity hint for one batch
    void flush();                                  // scores what is queued (fl_reads_push)
    void download();                               // per-read and per-row result arrays -> host
    fl_summary finalize(long long total_bases);    // main.cpp:169-261 on the GPU, then download()

    size_t n_reads() const { return names.size(); }
    size_t n_rows() const { return row_parent.size(); }
    // materialise read i (and its children) as a reference-style object; caller owns it
    Read *make_read(size_t i) const;
    std::string row_name(size_t row) const;       // parent name, or name_<start+1>-<end> for a child (read.cpp:135-136)

    std::vector<std::string> names;
    // per read
    std::vector<int32_t> length, first, last, n_bad, n_child;
    std::vector<double> mean_q, window_q, length_score;
    std::vector<uint8_t> passed;
    std::vector<uint64_t> row_start;
    // per reads2 row
    std::vector<uint32_t> row_parent;
    std::vector<int32_t> row_s, row_e;
    std::vector<double> row_mean, row_window, row_lscore, row_nmean, row_nwindow, row_final;
    std::vector<uint8_t> row_passed, row_pfinal;
    // --contam: per read, removed by the contaminant set (all 0 without one), and the removed reads / bases / rows
    std::vector<uint8_t> removed;
    fl_contam_counts contam{};
    bool ranked(size_t row) const { return !removed[row_parent[row]]; }   // the row takes part in the ranking

private:
    fl_ctx *ready_context();                       // the context, with this run's parameters set
    Kmers *kmers_;
    Arguments *args_;
    class HostArena *arena_;
    bool kmer_mode_;
    bool params_set_ = false;
    friend class Read;
};

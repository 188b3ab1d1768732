// filtlong_b200/csrc/host/read.cpp -- see read.h. Printing follows reference src/read.cpp:153-205.
#include "read.h"

#include <cmath>
#include <iostream>
#include <stdexcept>

#include "arena.h"
#include "misc.h"
#include "survivors.h"

fl_params params_from_arguments(const Arguments &a) {
    fl_params p{};
    p.window_size = a.window_size;
    p.trim = a.trim; p.split_set = a.split_set; p.split = a.split;
    p.min_length_set = a.min_length_set; p.min_length = a.min_length;
    p.max_length_set = a.max_length_set; p.max_length = a.max_length;
    p.min_mean_q_set = a.min_mean_q_set; p.min_window_q_set = a.min_window_q_set;
    p.min_mean_q = a.min_mean_q; p.min_window_q = a.min_window_q;
    p.length_weight = a.length_weight; p.mean_q_weight = a.mean_q_weight; p.window_q_weight = a.window_q_weight;
    p.target_bases_set = a.target_bases_set; p.keep_percent_set = a.keep_percent_set;
    p.target_bases = a.target_bases; p.keep_percent = a.keep_percent;
    p.trim_q = a.trim_q;
    p.max_contam = a.max_contam;
    return p;
}

// ---------------------------------------------------------------------------------------------
// ReadSet
// ---------------------------------------------------------------------------------------------
ReadSet::ReadSet(Kmers *kmers, Arguments *args) : kmers_(kmers), args_(args) {
    // nothing here waits for the GPU: records can be parsed and packed while the CUDA context is still coming up
    // (Kmers creates it on first use; both sets are finalised by the time they are asked for their size here); the
    // parameters are set with the first batch
    kmer_mode_ = !kmers->empty();                          // read.cpp:35
    // the bases are packed in k-mer mode, and for the contaminant set's probe
    arena_ = new HostArena(kmer_mode_ || kmers->contam_size() > 0, !kmer_mode_, false);
}

fl_ctx *ReadSet::ready_context() {
    fl_ctx *c = kmers_->context();
    if (!params_set_) {
        fl_params p = params_from_arguments(*args_);
        Kmers::check(c, fl_ctx_set_params(c, &p), "fl_ctx_set_params");
        params_set_ = true;
    }
    return c;
}

ReadSet::~ReadSet() { delete arena_; }

void ReadSet::add(const std::string &name, const char *seq, const char *qscores, int length) {
    if (!kmer_mode_ && !qscores)
        throw std::runtime_error("FASTA input not supported without an external reference");   // main.cpp:103-106
    names.push_back(name);
    arena_->add(seq, qscores, length);
}

void ReadSet::reserve(uint64_t bases, uint32_t reads) { arena_->reserve(bases + 64ull * reads, reads); }

void ReadSet::flush() {
    if (arena_->empty()) return;
    fl_batch b = arena_->batch();
    fl_ctx *c = ready_context();
    Kmers::check(c, fl_reads_push(c, &b), "fl_reads_push");
    arena_->clear();
}

void ReadSet::download() {
    flush();
    fl_ctx *c = ready_context();
    uint64_t nr = 0, nw = 0;
    Kmers::check(c, fl_reads_count(c, &nr, &nw, nullptr), "fl_reads_count");
    length.resize(nr); first.resize(nr); last.resize(nr); n_bad.resize(nr); n_child.resize(nr);
    mean_q.resize(nr); window_q.resize(nr); length_score.resize(nr); passed.resize(nr); row_start.resize(nr);
    fl_read_results rr{};
    rr.length = length.data(); rr.mean_q = mean_q.data(); rr.window_q = window_q.data();
    rr.length_score = length_score.data(); rr.passed = passed.data();
    rr.first_base_in_kmer = first.data(); rr.last_base_in_kmer = last.data();
    rr.n_bad = n_bad.data(); rr.n_child = n_child.data(); rr.row_start = row_start.data();
    Kmers::check(c, fl_results_reads(c, &rr), "fl_results_reads");
    row_parent.resize(nw); row_s.resize(nw); row_e.resize(nw);
    row_mean.resize(nw); row_window.resize(nw); row_lscore.resize(nw);
    row_nmean.resize(nw); row_nwindow.resize(nw); row_final.resize(nw);
    row_passed.resize(nw); row_pfinal.resize(nw);
    fl_row_results wr{};
    wr.parent = row_parent.data(); wr.start = row_s.data(); wr.end = row_e.data();
    wr.mean_q = row_mean.data(); wr.window_q = row_window.data(); wr.length_score = row_lscore.data();
    wr.norm_mean = row_nmean.data(); wr.norm_window = row_nwindow.data(); wr.final_score = row_final.data();
    wr.passed = row_passed.data(); wr.passed_final = row_pfinal.data();
    Kmers::check(c, fl_results_rows(c, &wr), "fl_results_rows");
    removed.resize(nr);
    Kmers::check(c, fl_results_contam(c, nullptr, removed.data(), &contam), "fl_results_contam");
}

fl_summary ReadSet::finalize(long long total_bases) {
    flush();
    fl_summary s{};
    fl_ctx *c = ready_context();
    Kmers::check(c, fl_finalize(c, total_bases, &s), "fl_finalize");
    download();
    return s;
}

std::string ReadSet::row_name(size_t row) const {
    const uint32_t p = row_parent[row];
    if (n_child[p] == 0) return names[p];
    std::string s;
    append_child_name(s, names[p].data(), names[p].size(), row_s[row], row_e[row]);
    return s;
}

Read *ReadSet::make_read(size_t i) const {
    Read *r = new Read();
    r->m_name = names[i];
    r->m_length = length[i];
    r->m_length_score = length_score[i];
    r->m_mean_quality = mean_q[i];
    r->m_window_quality = window_q[i];
    r->m_final_score = 0.0;
    r->m_passed = passed[i] != 0;
    r->m_first_base_in_kmer = first[i];
    r->m_last_base_in_kmer = last[i];
    const size_t rs = (size_t)row_start[i];
    for (int c = 0; c < n_child[i]; ++c) {
        const size_t row = rs + (size_t)c;
        r->m_child_read_ranges.push_back(std::make_pair(row_s[row], row_e[row]));
        Read *ch = new Read();
        ch->m_name = row_name(row);
        ch->m_length = row_e[row] - row_s[row];
        ch->m_length_score = row_lscore[row];
        ch->m_mean_quality = row_mean[row];
        ch->m_window_quality = row_window[row];
        ch->m_final_score = row_final[row];
        ch->m_passed = row_passed[row] != 0;
        // a child is a full Read of its own in the reference; its first/last follow from the parent's
        // mask restricted to the range, and it never has bad ranges or children (SURVEY 8a-R7)
        ch->m_first_base_in_kmer = -1;
        ch->m_last_base_in_kmer = -1;
        r->m_child_reads.push_back(ch);
    }
    // m_bad_ranges are exactly the gaps between the child ranges (read.cpp:119-130 inverted); a read
    // with bad ranges but no children is bad from end to end
    if (n_bad[i] > 0) {
        if (n_child[i] == 0) r->m_bad_ranges.push_back(std::make_pair(0, length[i]));
        else {
            int pos = 0;
            for (auto &cr : r->m_child_read_ranges) {
                if (cr.first > pos) r->m_bad_ranges.push_back(std::make_pair(pos, cr.first));
                pos = cr.second;
            }
            if (pos < length[i]) r->m_bad_ranges.push_back(std::make_pair(pos, length[i]));
        }
    }
    return r;
}

// ---------------------------------------------------------------------------------------------
// Read
// ---------------------------------------------------------------------------------------------
Read::Read(std::string name, char *seq, char *qscores, int length, Kmers *kmers, Arguments *args) {
    fl_ctx *c = kmers->context();
    Kmers::check(c, fl_reads_reset(c), "fl_reads_reset");
    ReadSet set(kmers, args);
    set.add(name, seq, qscores, length);
    set.download();
    Read *r = set.make_read(0);
    m_name = r->m_name;
    m_length = r->m_length;
    m_length_score = r->m_length_score;
    m_mean_quality = r->m_mean_quality;
    m_window_quality = r->m_window_quality;
    m_final_score = 0.0;
    m_passed = r->m_passed;
    m_first_base_in_kmer = r->m_first_base_in_kmer;
    m_last_base_in_kmer = r->m_last_base_in_kmer;
    m_bad_ranges = r->m_bad_ranges;
    m_child_read_ranges = r->m_child_read_ranges;
    m_child_reads.swap(r->m_child_reads);
    delete r;
    Kmers::check(c, fl_reads_reset(c), "fl_reads_reset");
}

Read::~Read() {
    for (auto child : m_child_reads) delete child;
}

static std::string pad(const std::string &s, size_t width) {
    return width > s.size() ? s + std::string(width - s.size(), ' ') : s;
}

void Read::print_verbose_read_info() {                                   // read.cpp:169-195
    std::cerr << "\n" << m_name << "\n";
    std::cerr << "            length = " << pad(std::to_string(m_length), 11);
    std::cerr << "mean quality = " << double_to_string(m_mean_quality);
    std::cerr << "      window quality = " << double_to_string(m_window_quality) << "\n";
    if (!m_bad_ranges.empty()) {
        std::cerr << "        bad ranges = ";
        for (size_t i = 0; i < m_bad_ranges.size(); ++i)
            std::cerr << m_bad_ranges[i].first << "-" << m_bad_ranges[i].second << (i + 1 < m_bad_ranges.size() ? ", " : "");
        std::cerr << "\n";
    }
    if (!m_child_read_ranges.empty()) {
        std::cerr << "      child ranges = ";
        for (size_t i = 0; i < m_child_read_ranges.size(); ++i)
            std::cerr << m_child_read_ranges[i].first << "-" << m_child_read_ranges[i].second
                      << (i + 1 < m_child_read_ranges.size() ? ", " : "");
        std::cerr << "\n";
    }
    for (auto child : m_child_reads) child->print_verbose_read_info();
}

void Read::print_scores(size_t name_length) {                            // read.cpp:198-204
    std::cerr << pad(m_name, name_length) << "\t" << double_to_string(m_length_score) << "\t"
              << double_to_string(m_mean_quality) << "\t" << double_to_string(m_window_quality) << "\t"
              << double_to_string(m_final_score) << "\n";
}

// Host-side final score for callers that drive Read objects one at a time (read.cpp:249-267, same
// operation order, host libm). The batch path computes this on the GPU (fl_finalize).
void Read::set_final_score(double length_weight, double mean_q_weight, double window_q_weight) {
    double product = pow(m_length_score, length_weight) * pow(m_mean_quality, mean_q_weight);
    double total_weight = length_weight + mean_q_weight;
    double final_score = pow(product, 1.0 / total_weight);
    double scaling_factor;
    if (m_mean_quality > 0.0) {
        double r = m_window_quality / m_mean_quality;
        scaling_factor = (1.0 < r) ? 1.0 : r;
    } else scaling_factor = 1.0;
    total_weight = length_weight + mean_q_weight + window_q_weight;
    double window_weight_fraction = window_q_weight / total_weight;
    double non_window_weight_fraction = 1.0 - window_weight_fraction;
    scaling_factor = non_window_weight_fraction + (scaling_factor * window_weight_fraction);
    m_final_score = final_score * scaling_factor;
}

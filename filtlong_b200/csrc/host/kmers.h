// filtlong_b200/csrc/host/kmers.h -- drop-in for the reference's Kmers (reference
// src/kmers.h:28-55): same public methods, but the 16-mer set lives in GPU memory behind the C
// ABI (fl_kmers_*). The object owns the fl_ctx that Read / the CLI score against.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../../include/filtlong_b200.h"

class Kmers {
public:
    // The CUDA context is created on first use (the first reference file, the first batch of
    // reads, ...): that call throws std::runtime_error if no CUDA device is usable (no CPU fallback).
    Kmers();
    explicit Kmers(int device);
    ~Kmers();
    Kmers(const Kmers &) = delete;
    Kmers &operator=(const Kmers &) = delete;

    bool empty() { return !ctx_ || size() == 0; }                      // kmers.h:34
    void add_read_fastqs(std::vector<std::string> filenames);          // kmers.h:36
    void add_assembly_fasta(std::string filename);                     // kmers.h:37
    bool is_kmer_present(uint32_t kmer);                               // kmers.h:38

    uint32_t starting_kmer_to_bits_forward(char *sequence);            // kmers.h:40-44
    uint32_t starting_kmer_to_bits_reverse(char *sequence);
    uint32_t base_to_bits_forward(char base);
    uint32_t base_to_bits_reverse(char base);

    // additions of the CUDA build
    uint64_t size();               // m_kmers.size()
    fl_ctx *context();
    static void check(fl_ctx *ctx, int rc, const char *what);          // throws on a non-zero status

private:
    int add_reference(const std::string &filename, bool require_multiple_copies);   // kmers.cpp:75-134
    fl_ctx *ctx_ = nullptr;
    int device_ = 0;
};

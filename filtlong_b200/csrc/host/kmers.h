// filtlong_b200/csrc/host/kmers.h -- drop-in for the reference's Kmers (reference
// src/kmers.h:28-55): same public methods, but the 16-mer set lives in GPU memory behind the C
// ABI (fl_kmers_*). The object owns the fl_ctx that Read / the CLI score against.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../../include/filtlong_b200.h"
#include "gzmem.h"

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
    // --contam: the contaminant set on the same context, built like add_assembly_fasta's set, with its log block
    // k: the contaminant k-mers' length (--contam_k); the set's table is sized by the file's bases (fl_contam_configure)
    void add_contaminant_fasta(const std::string &filename, int k = 16);
    uint64_t contam_size();        // 0 when none was added
    int contam_k() const { return contam_k_; }
    uint64_t contam_max_kmers() const { return contam_max_kmers_; }   // what fl_contam_configure was given

    // fl_gzip_inflate on context(), for inflate_gzip_memory (gzmem.h): tried on gzip input that is not BGZF and has at
    // least kDeviceGunzipMinBytes compressed bytes; a decline or a CUDA failure leaves the file to the host z_stream.
    GzipDeviceInflate device_inflater();
    static constexpr uint64_t kDeviceGunzipMinBytes = 64ull << 20;
    static void check(fl_ctx *ctx, int rc, const char *what);          // throws on a non-zero status

private:
    // kmers.cpp:75-134 into the reference set, or (contam) into the contaminant set
    int add_reference(const std::string &filename, bool require_multiple_copies, bool contam = false);
    fl_ctx *ctx_ = nullptr;
    int device_ = 0;
    int contam_k_ = 16;
    uint64_t contam_max_kmers_ = 0;
};

// filtlong_b200/csrc/host/feeder.h -- the device-first input path of the CLI (SURVEY 8f-1..3).
//
// The reference parses its input one record at a time on one thread, twice (reference src/main.cpp:70-125 and
// 263-313, klib kseq over zlib). Here, for an uncompressed file in the common layout (4-line FASTQ / 2-line
// FASTA, LF line ends), the host never looks at a record:
//   * the file is mapped; record-aligned chunks of ~256 MB are copied into a ring of pinned buffers by a few
//     copy threads and handed to the device as TEXT (fl_reads_push_text): boundaries, validation, 2-bit
//     packing / quality gather, per-record extents and a 64-bit hash of every name all happen there;
//   * duplicate names (main.cpp:113-117) are found in a flat open-addressing table over those hashes -- names
//     are compared byte for byte, in the mapping, only when two hashes agree; no string is ever built;
//   * with --gpus N the chunks are dealt to N contexts as contiguous ranges (one thread + one NCCL rank per
//     GPU, the 16-mer set broadcast from GPU 0, fl_finalize collective): the output is what one GPU prints;
//   * pass 2 writes the survivors with writev() straight from the mapping (no second parse, no copies).
//   * a gzip file is inflated ONCE into memory (gzmem.h: BGZF blocks by several host threads, anything else by one)
//     and then goes down the same path; the reference inflates it once per pass.
// Anything else -- CR LF, multi-line records, broken records, a gzip file that is damaged or would not fit in memory,
// --verbose -- makes run_text_feeder return handled == false before anything was printed to stdout, and main() runs
// the kseq-compatible host parser.
#pragma once
#include <functional>

#include "arguments.h"
#include "kmers.h"

struct FeederOutcome {
    bool handled = false;      // false: nothing was done; use the host parser
    int exit_code = 0;
};

FeederOutcome run_text_feeder(Arguments &args, Kmers &kmers, const std::function<void(const char *)> &mark);

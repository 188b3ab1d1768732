// filtlong_b200/csrc/host/feeder.h -- the device-first input path of the CLI (SURVEY 8f-1..3).
//
// The reference parses its input one record at a time on one thread, twice (reference src/main.cpp:70-125 and
// 263-313, klib kseq over zlib). Here, for input in the common layout (4-line FASTQ / 2-line FASTA, LF line ends, or
// unaligned BAM), the host never parses a record:
//   * the input is one byte range: a mapped file, a gzip file inflated ONCE into memory (gzmem.h: BGZF blocks by several
//     host threads, other gzip by the GPU inflater or one host thread; the reference inflates it once per pass), or a
//     stream held in memory (streamsrc.h);
//   * record-aligned chunks of 128 MiB (FL_CHUNK_MB) are copied into a ring of pinned buffers by a few copy threads and
//     handed to the device as TEXT (fl_reads_push_text): boundaries, validation, 2-bit packing / quality gather,
//     per-record extents and a 64-bit hash of every name all happen there;
//   * a BAM file's chunks are cut at record boundaries (bam.h); the reader threads check and index its records, the
//     device gathers and scores them (fl_reads_push_bam) and pass 2 writes BAM. It always takes this path: its errors are
//     thrown from here (nothing reaches stdout), and --verbose with it is one of them;
//   * duplicate names (main.cpp:113-117) are found in a flat open-addressing table over those hashes -- names are
//     compared byte for byte, in memory, only when two hashes agree; no string is ever built;
//   * with --gpus N the chunks are dealt to N contexts as contiguous ranges (one thread + one NCCL rank per GPU, the
//     16-mer set broadcast from GPU 0, fl_finalize collective): the output is what one GPU prints;
//   * a stream's plain text is cut into chunks as it arrives, and with one GPU each chunk is scored while the next is
//     still arriving; any other stream is read to its end first and then goes as a file does;
//   * pass 2 writes the survivors straight from memory (survivors.h: writev, or pwrite groups into a regular file).
// Anything else -- CR LF, multi-line records, broken records, a gzip file that is damaged or would not fit in memory,
// --verbose -- makes run_device_feeder return handled == false before anything was printed to stdout, and main() runs
// the kseq-compatible host parser.
#pragma once
#include <functional>

#include "arguments.h"
#include "kmers.h"

class StreamInput;

struct FeederOutcome {
    bool handled = false;      // false: nothing was done; use the host parser
    int exit_code = 0;
};

// stream: the input reads when they are a stream (read already started), else nullptr. mark: FL_CLI_TIMING's phase marks.
FeederOutcome run_device_feeder(Arguments &args, Kmers &kmers, StreamInput *stream, const std::function<void(const char *)> &mark);

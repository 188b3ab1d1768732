/* include/filtlong_b200.h -- C ABI of libfiltlong_b200.so (sm_90a CUDA inside).
 *
 * Drop-in boundary for Filtlong's per-read scoring / filtering hot path. Every entry point names
 * the reference interface it replaces (file:line relative to rrwick/Filtlong v0.3.1):
 *
 *   Kmers   (src/kmers.h:28-55, src/kmers.cpp:28-239)      -> fl_kmers_*
 *   Read    (src/read.h:29-65,  src/read.cpp:25-273)       -> fl_reads_*, fl_results_*
 *   the inline normalise / sort / threshold block of main   -> fl_finalize (+ split-phase fl_norm_*,
 *           (src/main.cpp:136-261)                             fl_select_* for sharded read sets)
 *
 * Conventions: plain C, POD in / POD out, no exceptions cross the ABI. Every function returns
 * 0 on success or a negative FL_E* code; fl_last_error(ctx) gives the message. One host thread
 * per context. "host" pointers are ordinary (ideally pinned) host memory; "dev" pointers are CUDA
 * device pointers on the context's device (e.g. torch tensors' data_ptr()). The library never
 * falls back to the CPU: without a usable CUDA device fl_ctx_create fails.
 *
 * Sequence arena layout (both host and device flavours):
 *   - coordinates are PADDED BASE coordinates; sequence i starts at off[i], a multiple of
 *     FL_ALIGN_BASES (64), and has len[i] bases;
 *   - seq2b: 2-bit codes, 16 bases per little-endian uint32 word, the FIRST base of a word in bits
 *     31:30 (so a word read as an integer is directly a forward 16-mer in the reference's
 *     encoding, kmers.cpp:222-229). Code = A0 C1 G2 T3, any other character 0 (kmers.cpp:176-196).
 *     Word index of padded base b is b/16;
 *   - qual: one byte per padded base, the raw FASTQ quality character (Phred+33); may be NULL
 *     when a k-mer reference is loaded (read.cpp:35-58 never touches it then);
 *   - ascii: alternative to seq2b (+ nmask) for callers that hold text: one character per padded base;
 *     the 2-bit packing of kmers.cpp:176-219 then happens on the device (k_pack_ascii);
 *   - nmask: 1 bit per padded base, bit (b & 31) of word b/32, set where the character was not
 *     one of ACGTacgt. Only reference sequences need it (kmers.cpp:199-219: the reverse encoder
 *     maps such characters to 0, i.e. NOT to the complement of the forward code); may be NULL.
 */
#ifndef FILTLONG_B200_H
#define FILTLONG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FL_ALIGN_BASES 64u
#define FL_K 16

enum {
    FL_OK = 0,
    FL_EINVAL = -1,   /* bad argument / call order */
    FL_ECUDA = -2,    /* CUDA runtime failure (message has the cudaError string) */
    FL_ENOMEM = -3,   /* host or device allocation failed */
    FL_ENODEV = -4,   /* no usable CUDA device: there is no CPU fallback */
    FL_ERANGE = -5    /* a capacity was exceeded (e.g. output buffer too small) */
};

/* Filtering options: the subset of `Arguments` (src/arguments.h:50-96) the hot path reads. */
typedef struct fl_params {
    int32_t window_size;                         /* arguments.h:90, default 250 */
    int32_t trim, split_set, split;              /* arguments.h:84-88 */
    int32_t min_length_set, min_length;          /* arguments.h:63-64 */
    int32_t max_length_set, max_length;          /* arguments.h:66-67 */
    int32_t min_mean_q_set, min_window_q_set;    /* arguments.h:69,72 */
    double min_mean_q, min_window_q;             /* arguments.h:70,73 */
    double length_weight, mean_q_weight, window_q_weight;   /* arguments.h:79-81 */
    int32_t target_bases_set, keep_percent_set;  /* arguments.h:57,60 */
    int64_t target_bases;                        /* arguments.h:58 */
    double keep_percent;                         /* arguments.h:61 */
    /* Not a reference option: 1..93 makes --trim / --split work without a k-mer set. A base is "good" (the
     * role of "in a reference 16-mer") when it lies in a run of FL_K consecutive bases whose quality bytes are
     * all >= 33 + trim_q; children are scored on their own quality bytes. 0 = off. A push with trim_q > 0 onto a
     * context whose k-mer set is not empty is FL_EINVAL. */
    int32_t trim_q;
    /* Not a reference option (--max_contam): a read is removed when more than this percentage of its bases lie in a
     * 16-mer of the contaminant set (fl_contam_*), compared in double, so a NaN (empty read) never is. Only read when that
     * set is not empty; a push onto such a context with a value outside [0, 100) is FL_EINVAL. */
    double max_contam;
} fl_params;

/* A batch of sequences in the arena layout above. */
typedef struct fl_batch {
    uint32_t n;              /* number of sequences */
    uint32_t reserved;
    uint64_t padded_bases;   /* arena size in padded bases (multiple of FL_ALIGN_BASES) */
    const uint64_t *off;     /* [n]  */
    const int32_t *len;      /* [n]  */
    const uint32_t *seq2b;   /* [padded_bases/16] or NULL (Phred-only scoring never reads it) */
    const uint8_t *qual;     /* [padded_bases]    or NULL */
    const uint32_t *nmask;   /* [padded_bases/32] or NULL */
    const char *ascii;       /* [padded_bases] or NULL: the bases as TEXT (what read.h:32 / kseq hand over),
                                one byte per padded base (padding bytes are ignored). Used when seq2b is
                                NULL: the library packs 2-bit codes (and the non-ACGT mask of reference
                                sequences) on the DEVICE, so a host caller only copies bytes */
} fl_batch;

typedef struct fl_ctx fl_ctx;

/* ---- context ------------------------------------------------------------------------------ */
int fl_ctx_create(const fl_params *params, int device, fl_ctx **out);
/* Optional: initialise the CUDA driver and the device's primary context (typically 0.5-1.5 s) from
 * any thread, e.g. while the caller is still parsing its input (the reference has no counterpart:
 * its Kmers / Read constructors are ready instantly, src/main.cpp:53,108). fl_ctx_create works
 * without it. Returns FL_OK or FL_ENODEV. */
int fl_device_warmup(int device);
void fl_ctx_destroy(fl_ctx *ctx);
const char *fl_last_error(const fl_ctx *ctx);      /* ctx may be NULL: last create error */
/* Run all work on a caller-owned CUDA stream (a cudaStream_t passed as void*), e.g. torch's
 * current stream, so the caller can bracket calls with its own events. NULL restores the
 * context's own stream. */
int fl_ctx_set_stream(fl_ctx *ctx, void *cuda_stream);
int fl_ctx_sync(fl_ctx *ctx);
int fl_ctx_set_params(fl_ctx *ctx, const fl_params *params);
/* Kernel launches issued by this context so far (for the bench's gpu_launches claim). */
uint64_t fl_ctx_launch_count(const fl_ctx *ctx);
/* Optional per-kernel device timing: when enabled, the dominant kernels are bracketed with CUDA
 * events on the launching stream. fl_ctx_kernel_time synchronises and returns the accumulated
 * milliseconds and launch count of one kernel since the last fl_ctx_reset_timing. */
enum { FL_KERNEL_SCORE_PHRED = 0, FL_KERNEL_PROBE_PAINT = 1, FL_KERNEL_KMER_STATS = 2, FL_KERNEL_KMERS_ADD = 3,
       /* --trim_q: the quality mask, the two row passes of the mask (with their scan), the gather of the children's
        * quality bytes, and the Phred pass over the children (its kernels also count in FL_KERNEL_SCORE_PHRED) */
       FL_KERNEL_QUAL_MASK = 4, FL_KERNEL_ROW_SCAN = 5, FL_KERNEL_QUAL_GATHER = 6, FL_KERNEL_QUAL_CHILDREN = 7,
       /* --contam: the probe of the contaminant set, the per-read count and the per-row exclusion */
       FL_KERNEL_CONTAM = 8,
       /* BAM output: the two passes of the child-record builder (fl_bam_build), and the BGZF compressor's kernels */
       FL_KERNEL_BAM_BUILD = 9, FL_KERNEL_BGZF = 10,
       FL_KERNEL_COUNT = 11 };
int fl_ctx_enable_timing(fl_ctx *ctx, int on);
int fl_ctx_reset_timing(fl_ctx *ctx);
int fl_ctx_kernel_time(fl_ctx *ctx, int which, double *total_ms, uint64_t *launches);
/* Diagnostics: how the default Phred window kernel decided the minimum of the reads longer than the window,
 * accumulated since the context was created. out[2p] counts reads and out[2p+1] their bases for path
 * p = 0 (the candidate steps of the filter pass walked exactly), 1 (the whole chain walked exactly),
 * 2 (sent to the sequential fallback by the filter pass: a quality byte the exact path cannot take, or a
 * first window outside its range), 3 (sent there by the exact minimum: the window came near or below 0.5);
 * out[8] is the number of exact steps walked.
 * Synchronises the context's stream. */
int fl_ctx_phred_paths(fl_ctx *ctx, uint64_t out[9]);

/* Test hook (host): where the probe kernel looks for `kmer` when the 16-mer starts at a read position
 * whose low two bits are pos_lo2 -- 32-bit word index into the 2 GiB position-anchored table and the
 * bit inside it (DESIGN.md section 3). Four consecutive 16-mers of a read share one 32-byte sector. */
void fl_anchor_slot_host(uint32_t kmer, uint32_t pos_lo2, uint32_t *word, uint32_t *bit);

/* ---- host-side packer (replaces the char* hand-off of read.h:32 / kmers.cpp:96-121) ------- */
/* Padded size of a sequence of `len` bases. */
uint64_t fl_padded_len(int64_t len);
/* Packs one sequence of ASCII bases (and optional quality string) into caller-provided arena
 * buffers at padded offset `off`. seq2b/nmask words touched by this sequence must be zeroed by
 * the caller beforehand (fresh arenas are). Any of seq2b / qual_out / nmask may be NULL. */
void fl_pack_sequence(const char *seq, const char *qual, int64_t len, uint64_t off,
                      uint32_t *seq2b, uint8_t *qual_out, uint32_t *nmask);

/* ---- Kmers: reference 16-mer set (src/kmers.h:28-55) --------------------------------------- */
/* Kmers::add_assembly_fasta (kmers.cpp:61-72) when require_multiple_copies == 0 (every 16-mer,
 * forward and reverse strand, enters the set: kmers.cpp:137-139); Kmers::add_read_fastqs
 * (kmers.cpp:50-58) when != 0 (a 16-mer enters at its 4th sighting, or its 3rd if the Bloom
 * filter false-positived on the 1st: kmers.cpp:142-166). Batches must be passed in file order;
 * sequences shorter than 16 contribute nothing (kmers.cpp:99-100). Host buffers. */
int fl_kmers_add_batch(fl_ctx *ctx, const fl_batch *host_batch, int require_multiple_copies);
/* Same with the arena already resident in device memory. */
int fl_kmers_add_batch_device(fl_ctx *ctx, const fl_batch *dev_batch, int require_multiple_copies);
/* Resolves pending multiple-copy state into the set and returns m_kmers.size() (kmers.h:34;
 * the "N 16-mers" log line of kmers.cpp:56-57,69-70). Idempotent; more batches may follow. */
int fl_kmers_finalize(fl_ctx *ctx, uint64_t *n_kmers_out);
/* Kmers::is_kmer_present (kmers.cpp:170-172) for n host k-mers -> out[i] in {0,1}. */
int fl_kmers_contains(fl_ctx *ctx, const uint32_t *kmers, uint32_t n, uint8_t *out);
/* Copies the set out in ascending order (at most cap entries); *n_out = set size. */
int fl_kmers_export(fl_ctx *ctx, uint32_t *out, uint64_t cap, uint64_t *n_out);
/* Device pointer to the direct-address membership bitmap (2^32 bits = 512 MiB; bit (k & 31) of
 * word k >> 5) so a sharded run can broadcast / OR-reduce it between GPUs. */
int fl_kmers_bitmap_dev(fl_ctx *ctx, void **dev_ptr, uint64_t *n_bytes);
/* Must be called after the bitmap was modified externally (recounts the set). */
int fl_kmers_bitmap_changed(fl_ctx *ctx);
/* Releases the transient multiple-copy build state (counters, first-seen times, Bloom times), after resolving it into the
 * set. Once multiple-copy 16-mers were added, the counts of those adds are gone with it: a later add with
 * require_multiple_copies != 0 (fl_kmers_add_batch, fl_kmers_add_batch_device, fl_kmers_add_text) returns FL_EINVAL.
 * Assembly adds (require_multiple_copies == 0) stay allowed. */
int fl_kmers_release_build_state(fl_ctx *ctx);
/* How the finalised set is laid out for the probe kernel (diagnostics / measurement): info[0] = a pre-filter is in use,
 * info[1] = its flavour (bit 2: one word per table group of four 16-mers, bit 3: one word per pair, bit 4: four bits per
 * member), info[2] = log2 of its 64-bit words, info[3] = the position-anchored table is in use. */
int fl_kmers_probe_info(fl_ctx *ctx, int32_t info[4]);

/* ---- contaminant set (no reference counterpart: --contam) ----------------------------------- */
/* A second 16-mer set on the same context, built exactly as fl_kmers_add_text / fl_kmers_add_batch build the reference set
 * with require_multiple_copies == 0 (an assembly: every forward and reverse 16-mer, non-ACGT handling of kmers.cpp:199-219).
 * It does not decide the scoring mode (that is the reference set's alone). When it is not empty, every push also finds,
 * per input read, c = 100 * (bases covered by a 16-mer of the set) / length -- the raw mean quality k-mer mode would give
 * the read against this set -- and removes the read when c > params.max_contam: its rows are not passed, and they take
 * no part in the statistics, the passed bases or the selection of fl_finalize. The reads' bases are then needed in Phred
 * mode too (seq2b or ascii; a push without them is FL_EINVAL). Build the set before any read is pushed: an add after
 * that is FL_EINVAL. About 2.5 GiB of device memory are allocated with the first add. */
int fl_contam_add_text(fl_ctx *ctx, const char *host_text, uint64_t n_bytes, int format, int is_last_chunk,
                       uint64_t *n_records, uint64_t *n_bases, uint64_t *bytes_consumed, int *status);
int fl_contam_add_batch(fl_ctx *ctx, const fl_batch *host_batch);
int fl_contam_finalize(fl_ctx *ctx, uint64_t *n_kmers_out);
int fl_contam_export(fl_ctx *ctx, uint32_t *out, uint64_t cap, uint64_t *n_out);
/* collective, like fl_kmers_broadcast. A set of k > 16 goes as its table's bytes: every rank must have called
 * fl_contam_configure with the same k and max_kmers. The ranks first compare k and the table size; when any differs,
 * every rank returns FL_EINVAL and nothing is sent. */
int fl_contam_broadcast(fl_ctx *ctx, int root);
/* Not a reference option (--contam_k): the contaminant set's k-mer length, 16 to 32 (16 = the set above, the default).
 * Call before the first contaminant add and before any read is pushed (FL_EINVAL after either, or for k outside 16..32).
 * For k > 16 the set is a device hash set of canonical k-mers, sized here for at most max_kmers of them (a bound on the
 * contaminant's bases will do): 32 bytes per 3.2 k-mers, rounded up to a power of two; FL_ENOMEM, with the GiB it needed
 * in the message, when the device lacks the memory. Every window of k bases of a contaminant record that holds only ACGTacgt
 * adds min(forward, reverse complement); a window with any other character adds nothing. An add that could take the set
 * past its reservation is FL_EINVAL and adds nothing. A read's k-mers come from its 2-bit codes (a non-ACGT base is A), and a
 * base is covered when a k-mer containing it is in the set on either strand. fl_contam_finalize then counts the forward and
 * reverse k-mers: 2 * canonical - palindromes. */
int fl_contam_configure(fl_ctx *ctx, int k, uint64_t max_kmers);
/* k > 16: the canonical members in any order (at most cap; *n_out = how many there are). fl_contam_export is FL_EINVAL then. */
int fl_contam_export64(fl_ctx *ctx, uint64_t *out, uint64_t cap, uint64_t *n_out);
/* k > 16: out[i] = the forward k-mer fwd_kmers[i] (2-bit codes, first base in the high bits) is in the set on either strand */
int fl_contam_contains64(fl_ctx *ctx, const uint64_t *fwd_kmers, uint32_t n, uint8_t *out);
/* k > 16, for measurement: hist[0, n_bins) counts members by the buckets (32-byte sectors) a look-up of them reads,
 * hist[n_bins, 2 * n_bins) counts buckets by the sectors a look-up of an absent k-mer hashed there reads; the last bin of
 * each holds that many or more. */
int fl_contam_probe_lengths(fl_ctx *ctx, uint64_t *hist, int n_bins);
typedef struct fl_contam_counts {
    uint64_t reads;    /* input reads removed */
    int64_t bases;     /* their bases */
    uint64_t rows;     /* their rows (the reads themselves, or their children) */
} fl_contam_counts;
/* Per INPUT READ (length n_reads): percent = c, removed = c > max_contam (0 and 0 when the set is empty); counts of this
 * context's removed reads. Any pointer may be NULL. */
int fl_results_contam(fl_ctx *ctx, double *percent, uint8_t *removed, fl_contam_counts *counts);

/* ---- Read: per-read scoring (src/read.cpp:25-144) ------------------------------------------ */
/* Scores a batch the way one `new Read(...)` per record does (main.cpp:108) and appends the
 * result rows to the context. Mode = Phred if the k-mer set is empty, k-mer otherwise
 * (read.cpp:35). Host buffers: copies are issued inside the call and the buffers may be reused when it
 * returns. In k-mer mode with --trim / --split the batch's rows are completed at the start of the next
 * call on the context, whichever it is (the row count costs a host round trip, which is paid once the next
 * batch's copy is under way); fl_reads_count, fl_finalize, fl_results_* ... all see the batch. */
int fl_reads_push(fl_ctx *ctx, const fl_batch *host_batch);
/* Same with the arena already resident in device memory (no copies). */
int fl_reads_push_device(fl_ctx *ctx, const fl_batch *dev_batch);
/* The feeder (replaces the kseq_read loop of main.cpp:70-125 for the common file layout): hands a chunk of
 * the input FILE -- bytes, as mapped -- to the device, which finds the record boundaries, validates them,
 * extracts per-record extents and a 64-bit hash of every name (for the duplicate check of main.cpp:113-117),
 * packs the sequences (k-mer mode) or gathers the qualities (Phred mode) into the arena and scores the
 * records like fl_reads_push. The chunk must START at a record boundary; records are 4-line FASTQ
 * (FL_TEXT_FASTQ) or 2-line FASTA (FL_TEXT_FASTA) with LF line ends. *bytes_consumed = end of the last whole
 * record (the caller starts its next chunk there); with is_last_chunk the final line may lack its newline.
 * FL_ERANGE: out->cap is too small; nothing was scored and *n_records holds the number needed.
 * If the text is not in that layout (CR LF, multi-line records, blank lines, quality / sequence length
 * mismatch ...) nothing is scored and *status = FL_TEXT_FALLBACK: the caller parses on the host instead
 * (kseq semantics, and the reference's error messages for broken input). Offsets in `out` are relative to the
 * chunk's first byte; comment_len == 0 means no comment, otherwise it starts at name_off + name_len + 1. */
enum { FL_TEXT_FASTQ = 1, FL_TEXT_FASTA = 2 };
enum { FL_TEXT_OK = 0, FL_TEXT_FALLBACK = 1 };
typedef struct fl_text_records {
    uint64_t cap;                      /* capacity of each array, in records */
    uint64_t *name_off;                /* any array may be NULL */
    uint32_t *name_len, *comment_len;
    uint64_t *seq_off, *qual_off;
    int32_t *len;
    uint64_t *name_hash;
} fl_text_records;
int fl_reads_push_text(fl_ctx *ctx, const char *host_text, uint64_t n_bytes, int format, int is_last_chunk,
                       const fl_text_records *out, uint64_t *n_records, uint64_t *bytes_consumed, int *status);
/* Unaligned BAM input: a chunk of inflated BAM bytes holding n_rec whole records, and per record where its SEQ
 * (seq_off, 4-bit codes) and QUAL (qual_off) start, relative to the chunk, and its length (l_seq >= 1). The caller has
 * walked and checked the records (host/bam.cpp). Each record is scored as the record of its FASTQ equivalent: in Phred
 * mode the quality is QUAL + 33, in k-mer mode the sequence is SEQ decoded with "=ACMGRSVTWYHKDBN". Same buffer-reuse
 * rules as fl_reads_push_text: the chunk and the arrays may be reused when the call returns. FL_EINVAL if a record does
 * not lie inside the chunk. */
int fl_reads_push_bam(fl_ctx *ctx, const char *chunk, uint64_t n_bytes, uint64_t n_rec, const uint32_t *seq_off,
                      const uint32_t *qual_off, const int32_t *len);
/* Aligned BAM input: the same, with reverse[i] != 0 for a record that stores its read reverse-complemented (flag 0x10).
 * Such a record is scored as the read in its original orientation, as `samtools fastq` writes it: QUAL reversed, SEQ
 * reversed and complemented (A <-> T, C <-> G, every other code counts as a base outside ACGT). reverse == NULL: every
 * record is forward, as with fl_reads_push_bam. */
int fl_reads_push_bam_strand(fl_ctx *ctx, const char *chunk, uint64_t n_bytes, uint64_t n_rec, const uint32_t *seq_off,
                             const uint32_t *qual_off, const int32_t *len, const uint8_t *reverse);
/* BAM output built on the device. A batch holds BAM bytes: whole records and pieces of raw stream. Each item is one
 * piece of the output, in order: s < 0 copies bytes [off, off + e) of the batch; s >= 0 builds the child [s, e) (0 <= s
 * < e <= l_seq) of the record that starts at byte `off` of the batch, as bam_child_record (host/bam.h) builds it --
 * the parent's fixed fields, read_name name_<s+1>-<e>, the slice of SEQ and QUAL, the parent's RG fields and, with
 * keep_mods and valid modification tags, the re-based MM / ML and MN:I (fl_bam_mods.h). A record's children are
 * consecutive items that name the same record; they are cheapest in the order of their starts. The uncompressed
 * records are written to out[0, *n_out). counts[0]: children that kept modification tags, counts[1]: children whose
 * parent has an MM tag and invalid tags (keep_mods only; both added to, not set). FL_ERANGE: cap is too small, *n_out
 * holds the size needed; FL_EINVAL: an item outside the batch, a child's record whose fixed fields, read_name, CIGAR,
 * SEQ and QUAL do not fit its block_size (or l_read_name 0), a child outside [0, l_seq), or a child name longer than a
 * BAM record allows. Aux fields are read up to the first that does not parse. */
typedef struct fl_bam_item {
    uint64_t off;
    int32_t s, e;
} fl_bam_item;
#define FL_BAM_MODS_KEPT 1
#define FL_BAM_MODS_INVALID 2
/* Host buffers. */
int fl_bam_build(fl_ctx *ctx, const void *host_batch, uint64_t n_bytes, const fl_bam_item *items, uint64_t n_items, int keep_mods,
                 void *host_out, uint64_t cap, uint64_t *n_out, uint64_t counts[2]);
/* Device buffers on the context's device (the batch readable 16 bytes past n_bytes). */
int fl_bam_build_device(fl_ctx *ctx, const void *dev_batch, uint64_t n_bytes, const fl_bam_item *dev_items, uint64_t n_items,
                        int keep_mods, void *dev_out, uint64_t cap, uint64_t *n_out, uint64_t counts[2]);
/* One BGZF-compressed BAM output stream built batch by batch: each push builds the batch's records on the device
 * (fl_bam_build_device), appends them to what the stream holds back, compresses the whole FL_BGZF_BLOCK-byte blocks
 * (fl_bgzf_compress_device) into host_out[0, *n_out) and holds back the rest on the device, so that the members are cut
 * every FL_BGZF_BLOCK bytes of the stream whatever the batches are. The push with last != 0 compresses everything
 * left (no EOF member). A writer uses its context on the calling thread and keeps its own device buffers; several
 * writers may share a context, one call at a time. cap >= fl_bgzf_bound(FL_BGZF_BLOCK + the batch's built bytes); a push
 * that returns FL_ERANGE (with the size needed in *n_out) leaves the stream as it was, and may be made again. */
typedef struct fl_bam_writer fl_bam_writer;
int fl_bam_writer_create(fl_ctx *ctx, fl_bam_writer **out);
int fl_bam_writer_push(fl_bam_writer *w, const void *host_batch, uint64_t n_bytes, const fl_bam_item *items, uint64_t n_items,
                       int keep_mods, int last, void *host_out, uint64_t cap, uint64_t *n_out, uint64_t counts[2]);
void fl_bam_writer_destroy(fl_bam_writer *w);
/* The reference set from a chunk of the reference FILE (replaces the kseq_read loop of Kmers::add_reference,
 * kmers.cpp:75-134, for the common layouts): same contract as fl_reads_push_text -- the chunk starts at a record boundary,
 * LF line ends, FL_TEXT_FALLBACK and nothing added otherwise -- but the records' sequences go to the 16-mer set like
 * fl_kmers_add_batch(require_multiple_copies). FASTQ: 4-line records. FASTA: a record's sequence may be WRAPPED (kseq joins
 * the lines, kseq.h:199-203) as long as all of its lines but the last have one width and the last is not longer (what
 * assemblers write); a FASTA chunk that is not the file's last must end with a newline and is consumed whole or not at
 * all. *n_records counts every record of the chunk (kmers.cpp:96), *n_bases the bases of those of at least 16
 * (kmers.cpp:99-101). Chunks in file order. */
int fl_kmers_add_text(fl_ctx *ctx, const char *host_text, uint64_t n_bytes, int format, int is_last_chunk,
                      int require_multiple_copies, uint64_t *n_records, uint64_t *n_bases, uint64_t *bytes_consumed, int *status);
/* Page-locked host memory for the caller's chunk ring (portable across devices); the host side of the
 * boundary links no CUDA runtime of its own. */
int fl_host_alloc(uint64_t n_bytes, void **out);
void fl_host_free(void *p);
/* Page-locks memory the caller owns (it may already be filling it from another thread: a reader can start on
 * the input while the CUDA context is still coming up). FL_ENOMEM if the driver refuses: the buffers still work,
 * copies are just staged by the driver. */
int fl_host_register(void *p, uint64_t n_bytes);
void fl_host_unregister(void *p);
/* Forget all scored reads (keeps the k-mer set and parameters). */
int fl_reads_reset(fl_ctx *ctx);
/* Number of input reads / of "reads2" rows (children replace their parent, main.cpp:138-147). */
int fl_reads_count(fl_ctx *ctx, uint64_t *n_reads, uint64_t *n_rows, int64_t *total_bases);

/* ---- normalise + select (src/main.cpp:169-261) --------------------------------------------- */
typedef struct fl_summary {
    double min_q, max_q, mean_q, stdev_q, min_z, max_z;   /* main.cpp:170-196 */
    int32_t status;          /* 0 no target option; 1 "not enough reads to reach target";
                                2 "reads already fall below target after filtering";
                                3 sorted and thresholded (main.cpp:239-259) */
    int32_t reserved;
    int64_t target, passed_bases, keeping, total_bases, rows_bases;
} fl_summary;

/* Whole block main.cpp:169-261. total_bases = sum of the input read lengths THIS context was given
 * (main.cpp:89; --keep_percent uses the sum over all shards); pass -1 to use the context's own count.
 * On a context with a communicator (fl_comm_init) the call is collective: every rank calls it, the
 * statistics, the base-weighted score histogram (13-bit digits, 5 levels) and the tie class at the cut-off
 * are exchanged with NCCL on the context's stream (no host round trip in between), and every rank gets the
 * same summary while its rows keep their own pass flags. Without a communicator the same code runs with
 * the collectives degenerated to local copies. */
int fl_finalize(fl_ctx *ctx, int64_t total_bases, fl_summary *out);

/* ---- read set sharded across GPUs: one context + one rank per GPU (SURVEY 8e) ----------------- */
/* The reference is a single thread (main.cpp:37-321); a sharded run couples its shards only through the
 * block main.cpp:169-261 and through the shared Kmers object. One process per GPU or one thread per GPU.
 * fl_comm_unique_id: rank 0 creates the 128-byte id (ncclGetUniqueId) and hands it to the other ranks by
 * any means; fl_comm_init: ncclCommInitRank on the context's device (collective). */
#define FL_COMM_ID_BYTES 128
int fl_comm_unique_id(void *out128);
int fl_comm_init(fl_ctx *ctx, const void *id128, int rank, int nranks);
int fl_comm_destroy(fl_ctx *ctx);
int fl_comm_info(const fl_ctx *ctx, int *rank, int *nranks);
/* Kmers built on one rank, used by all (main.cpp:53-59 once per run): broadcasts the finished
 * direct-address bitmap (512 MiB) from `root` over NVLink; collective. */
int fl_kmers_broadcast(fl_ctx *ctx, int root);
/* Sum of up to 24 host int64 over the ranks (e.g. the shards' read and base counts for the log lines of
 * misc.cpp:47-49); collective, synchronises the context's stream. */
int fl_comm_allreduce_i64_host(fl_ctx *ctx, int64_t *inout, int n);
/* NCCL calls issued by this context so far. */
uint64_t fl_comm_collective_count(const fl_ctx *ctx);

/* Split-phase form of the same block for callers that bring their OWN transport (the CPU test double
 * over gloo in tests/test_sharded_select.py; 8 levels of 256 bins): the caller all-reduces the small
 * DEVICE buffers between phases. Buffers are caller-allocated device memory.
 *   1. fl_norm_partial1(ctx, sums, mins, maxs)         sums = f64[4]: n, sum(mean_q), passed_bases,
 *                                                       rows_bases; mins/maxs = f64[1]
 *                                                       -> all-reduce SUM / MIN / MAX
 *   2. fl_norm_partial2(ctx, sums, mins, maxs, sq)     sq = f64[1]: sum((x-mean)^2) -> all-reduce SUM
 *   3. fl_norm_apply(ctx, sums, mins, maxs, sq)        rescale + final score for every local row
 *   4. fl_select_begin(ctx, total_bases_global, sums)
 *      for level in 0..7:  fl_select_hist(ctx, level, hist)   hist = u64[256] -> all-reduce SUM
 *                          fl_select_pick(ctx, level, hist)
 *      fl_select_tie_local(ctx, tie, rank, nranks)     tie = u64[nranks], own slot written
 *                                                       -> all-reduce SUM
 *      fl_select_apply(ctx, tie, rank, keeping)        keeping = u64[1], local kept bases
 *                                                       -> all-reduce SUM
 *   5. fl_select_summary(ctx, sums, mins, maxs, sq, keeping, total, &summary)
 */
int fl_norm_partial1(fl_ctx *ctx, double *dev_sums4, double *dev_min1, double *dev_max1);
int fl_norm_partial2(fl_ctx *ctx, const double *dev_sums4, const double *dev_min1,
                     const double *dev_max1, double *dev_sq1);
int fl_norm_apply(fl_ctx *ctx, const double *dev_sums4, const double *dev_min1,
                  const double *dev_max1, const double *dev_sq1);
int fl_select_begin(fl_ctx *ctx, int64_t total_bases_global, const double *dev_sums4);
int fl_select_hist(fl_ctx *ctx, int level, uint64_t *dev_hist256);
int fl_select_pick(fl_ctx *ctx, int level, const uint64_t *dev_hist256);
int fl_select_tie_local(fl_ctx *ctx, uint64_t *dev_tie_per_rank, int rank, int nranks);
int fl_select_apply(fl_ctx *ctx, const uint64_t *dev_tie_per_rank, int rank, uint64_t *dev_keeping1);
int fl_select_summary(fl_ctx *ctx, const double *dev_sums4, const double *dev_min1,
                      const double *dev_max1, const double *dev_sq1, const uint64_t *dev_keeping1,
                      int64_t total_bases_global, fl_summary *out);

/* ---- results (the public fields of Read, read.h:40-56) ------------------------------------- */
/* Per INPUT READ arrays (length n_reads); any pointer may be NULL. mean_q / window_q are the RAW
 * values of read.cpp:60-61; passed is the hard cut-off result of read.cpp:65-73. */
typedef struct fl_read_results {
    int32_t *length;
    double *mean_q, *window_q, *length_score;
    uint8_t *passed;
    int32_t *first_base_in_kmer, *last_base_in_kmer;   /* read.cpp:75-84 (-1 in Phred mode) */
    int32_t *n_bad, *n_child;                          /* sizes of m_bad_ranges / m_child_reads */
    uint64_t *row_start;                               /* first reads2 row of this read */
} fl_read_results;

/* Per reads2 ROW arrays (length n_rows): a row is an input read without children, or one child
 * (read.cpp:119-141). start/end are the range in the parent (child name = parent + "_" +
 * (start+1) + "-" + end, read.cpp:135-136). norm_* / final_score / passed_final are filled by
 * fl_finalize (main.cpp:202-212, 251-257); before it passed_final == passed. */
typedef struct fl_row_results {
    uint32_t *parent;
    int32_t *start, *end;
    double *mean_q, *window_q, *length_score;
    double *norm_mean, *norm_window, *final_score;
    uint8_t *passed, *passed_final;
} fl_row_results;

int fl_results_reads(fl_ctx *ctx, const fl_read_results *host_out);
int fl_results_rows(fl_ctx *ctx, const fl_row_results *host_out);
/* Device pointer + count of the final per-row pass flags (uint8), for callers that keep
 * everything on the GPU. */
int fl_results_pass_dev(fl_ctx *ctx, void **dev_passed_final, uint64_t *n_rows);
/* Copies only the final per-row pass flags to host memory (the per-step result a streaming
 * caller needs); *n_rows receives the row count, at most cap flags are written. */
int fl_results_pass(fl_ctx *ctx, uint8_t *host_out, uint64_t cap, uint64_t *n_rows);

/* ---- synthetic workloads (bench / tests only; deterministic, identical on host and device) -- */
/* SURVEY 8d's generators as integer-only counter-based functions (filtlong_b200/csrc/fl_synth.h). The
 * *_host flavours are also exported by the tiny libflsynth_host.so (no CUDA inside) for the CPU legs of
 * bench.py. */
/* Phred+33 quality string for padded arena `off/len`: per-base Q = clip(qbar[i] + z, 1, 50) with z
 * an integer-only approximately normal(0, 4) draw keyed by (seed, read index, position). */
int fl_synth_qual_device(fl_ctx *ctx, uint64_t seed, uint32_t n, const uint64_t *dev_off,
                         const int32_t *dev_len, const uint8_t *dev_qbar, uint64_t read_index_base,
                         uint8_t *dev_qual);
void fl_synth_qual_host(uint64_t seed, uint32_t n, const uint64_t *off, const int32_t *len,
                        const uint8_t *qbar, uint64_t read_index_base, uint8_t *qual);
/* Uniform random genome of n_bases (2-bit arena, one sequence at offset 0). */
int fl_synth_genome_device(fl_ctx *ctx, uint64_t seed, uint64_t n_bases, uint32_t *dev_seq2b);
void fl_synth_genome_host(uint64_t seed, uint64_t n_bases, uint32_t *seq2b);
/* Assembly of n_contigs contigs of contig_bases uniform random bases each (contig c at padded offset
 * c * fl_padded_len(contig_bases)), with n_ppm / 1e6 of its 1024-base blocks replaced by runs of N
 * (code 0 in seq2b, bit set in nmask; nmask may be NULL). BASELINE config 5: 1000 x 3 Mbp, 2 % N. */
int fl_synth_assembly_device(fl_ctx *ctx, uint64_t seed, uint32_t n_contigs, uint64_t contig_bases,
                             uint32_t n_ppm, uint32_t *dev_seq2b, uint32_t *dev_nmask);
void fl_synth_assembly_host(uint64_t seed, uint32_t n_contigs, uint64_t contig_bases, uint32_t n_ppm,
                            uint32_t *seq2b, uint32_t *nmask);
/* Reads sampled from that genome: read i is copied from the template genome[start[i], start[i] + span)
 * (span = len + len/8 + 64, fl_synth_span) on strand[i] (1 = reverse complement) with per-base errors at
 * rate err_ppm[i]/1e6 -- split 50/25/25 into substitutions / insertions / deletions when flags bit 0 is
 * set (ONT / PacBio model), substitutions only otherwise (Illumina model) -- and, overriding the template,
 * uniform random bases in [junk_pos[i], junk_pos[i]+junk_len[i]) (chimeric insert) and in the first
 * adap5[i] / last adap3[i] positions (adapters). adap5 / adap3 may be NULL. */
#define FL_SYNTH_INDELS 1u
typedef struct fl_synth_reads {
    uint32_t n;
    uint32_t flags;
    uint64_t genome_bases;
    const uint64_t *off;
    const int32_t *len;
    const uint64_t *start;
    const uint8_t *strand;
    const uint32_t *err_ppm;
    const int32_t *junk_pos, *junk_len;
    const int32_t *adap5, *adap3;
} fl_synth_reads;
int fl_synth_reads_device(fl_ctx *ctx, uint64_t seed, const uint32_t *dev_genome2b,
                          const fl_synth_reads *dev_desc, uint64_t read_index_base, uint32_t *dev_seq2b);
void fl_synth_reads_host(uint64_t seed, const uint32_t *genome2b, const fl_synth_reads *desc,
                         uint64_t read_index_base, uint32_t *seq2b);
/* 2-bit arena -> ASCII bases (one byte per padded base, 'N' where nmask is set, 0 in the padding):
 * what a caller holding text would hand to the char* boundary (read.h:32). */
int fl_synth_ascii_device(fl_ctx *ctx, uint32_t n, const uint64_t *dev_off, const int32_t *dev_len,
                          const uint32_t *dev_seq2b, const uint32_t *dev_nmask, uint8_t *dev_ascii);
void fl_synth_ascii_host(uint32_t n, const uint64_t *off, const int32_t *len, const uint32_t *seq2b,
                         const uint32_t *nmask, uint8_t *ascii);

/* ---- BGZF output (no reference counterpart: replaces the `| gzip > output.fastq.gz` pipe the reference README ends
 * its command lines with) ----------------------------------------------------------------------------------------------
 * The input is cut into blocks of FL_BGZF_BLOCK bytes (bgzip's block size; the last one may be shorter) and every
 * block becomes one BGZF member (SAM specification 4.1): a gzip member with MTIME 0, XFL 0, OS 255 and a 6-byte 'BC'
 * extra field holding the member size - 1, a raw deflate stream (one dynamic-Huffman block, or a stored block when that
 * is not larger) and the CRC-32 / ISIZE trailer. The members follow each other in input order, then, with append_eof,
 * the 28-byte empty member that ends a BGZF file. Any gzip reader reads the result; the same input always gives the
 * same bytes. Works on any context (one without reads or k-mers too) and leaves its scored reads and results as they
 * are. FL_ERANGE: cap is too small; *n_out then holds the size needed. */
#define FL_BGZF_BLOCK 65280u
/* Largest output n_bytes of input can give, the EOF member included. */
uint64_t fl_bgzf_bound(uint64_t n_bytes);
/* Host buffers (pinned ones copy fastest). */
int fl_bgzf_compress(fl_ctx *ctx, const void *host_in, uint64_t n, void *host_out, uint64_t cap, int append_eof,
                     uint64_t *n_out);
/* Device buffers on the context's device. */
int fl_bgzf_compress_device(fl_ctx *ctx, const void *dev_in, uint64_t n, void *dev_out, uint64_t cap, int append_eof,
                            uint64_t *n_out);

/* ---- gzip input inflated on the device (no reference counterpart: the reference reads .gz input through zlib's gzread)
 * An ordinary gzip file -- one member, or several back to back, with whatever bytes after the last member that do not
 * start a gzip header, as gzread reads it -- inflated in parallel on the context's device: chunks of the compressed
 * bytes are decoded speculatively from candidate block starts, the chain of chunk boundaries is checked and repaired,
 * back-references into a chunk's unknown 32 KiB window are resolved afterwards, and every member's CRC-32 and ISIZE are
 * checked. Output symbols take 2 bytes per output byte on the device, so a large file is done in rounds sized from the
 * free device memory. bin/filtlong uses it on its scoring context for gzip input that is not BGZF and has at least
 * 64 MiB of compressed bytes, and falls back to one host zlib thread on a decline.
 * FL_GUNZIP_OK: host_out[0, *n_out) holds exactly the bytes zlib inflates from host_in. FL_GUNZIP_DECLINED: anything
 * not handled here -- not gzip, truncated, corrupt, a bad CRC or ISIZE, more than cap bytes, a chunk whose output does
 * not fit its slot, too many repair passes, not enough device memory -- and nothing is promised about host_out.
 * chunk_bytes / max_device_bytes: 0 = the library's choice (max_device_bytes is then the free device memory).
 * Works on any context and leaves its reads and results as they are; every device buffer is freed before it returns.
 * A CUDA failure is FL_ECUDA. */
enum { FL_GUNZIP_OK = 0, FL_GUNZIP_DECLINED = 1 };
typedef struct fl_gunzip_stats {
    uint64_t members;      /* gzip members inflated */
    uint64_t chunks;       /* chunks decoded (a chunk without a candidate start is merged into the one before) */
    uint64_t redecoded;    /* chunks decoded again from where their predecessor really stopped */
    uint64_t rounds;       /* rounds of chunks the device memory allowed */
} fl_gunzip_stats;
/* Host buffers (the CLI's path: a mapped file into the reservation it is read from). */
int fl_gzip_inflate(fl_ctx *ctx, const void *host_in, uint64_t n, void *host_out, uint64_t cap, uint64_t chunk_bytes,
                    uint64_t max_device_bytes, uint64_t *n_out, int *status, fl_gunzip_stats *stats);
/* Device buffers on the context's device: the same, without the copies. */
int fl_gzip_inflate_device(fl_ctx *ctx, const void *dev_in, uint64_t n, void *dev_out, uint64_t cap, uint64_t chunk_bytes,
                           uint64_t max_device_bytes, uint64_t *n_out, int *status, fl_gunzip_stats *stats);

/* ---- misc ---------------------------------------------------------------------------------- */
const char *fl_version(void);
/* Phred look-up tables exactly as the device uses them (read.cpp:270-273 evaluated with the host
 * libm): q[b] = 1 - pow(10, -((int8_t)b - 33)/10.0), a[b] = q[b] / window_size. */
void fl_phred_luts(int32_t window_size, double *q256, double *a256);

#ifdef __cplusplus
}
#endif
#endif

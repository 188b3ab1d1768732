// filtlong_b200/csrc/host/bam.h -- BAM input, unaligned or (--aligned) aligned: the only code that knows the BAM record
// layout (SAM/BAM format specification, section 4.2).
//
// A BAM file is BGZF; it is inflated into memory like any gzip input (textsrc.h, gzmem.h), and an inflated input that
// starts with "BAM\1" is this format (MappedFile::format() == FL_FORMAT_BAM). The header is copied to the output as it
// is. The records are cut into chunks of whole records by walking the block_size chain once; each chunk's records are
// then checked and indexed on their own (the feeder does that on its reader threads) into the Records table the rest of
// the CLI uses: name_off at read_name, name_len without the NUL, no comment, seq_off at the first SEQ byte, qual_off at
// QUAL, len = l_seq. A record starts 36 bytes before its name, so the table needs no field of its own for it.
//
// A record stands for the record of its FASTQ equivalent: name = read_name, sequence = SEQ decoded with
// "=ACMGRSVTWYHKDBN", quality = each QUAL byte + 33, or no quality (a FASTA record) when QUAL starts with 0xFF.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "survivors.h"
#include "textsrc.h"

constexpr int FL_FORMAT_BAM = 3;

// the bytes start with the BAM magic "BAM\1"
inline bool bam_magic(const char *b, uint64_t size) { return size >= 4 && b[0] == 'B' && b[1] == 'A' && b[2] == 'M' && b[3] == 1; }
// the file is gzip / BGZF and its inflated stream starts with the BAM magic (only the first bytes are inflated)
bool bam_file_magic(const std::string &path);

// The header: magic, l_text, text, n_ref and the reference entries, all inside the input. *end: its size.
bool bam_header(const char *b, uint64_t size, uint64_t *end, std::string *why);

// The records after the header in chunks of whole records of at most `target` bytes; a record larger than that is a
// chunk of its own, and no chunk reaches 2 GiB. Checks the block_size chain: every block_size >= 32, every record ends
// inside the input. *max_chunk: the largest chunk; *max_record (when given): the largest record.
bool bam_plan_chunks(const char *b, uint64_t size, uint64_t header_end, uint64_t target, std::vector<Chunk> &out, uint64_t *max_chunk,
                     std::string *why, uint64_t *max_record = nullptr);

// One chunk's records, offsets relative to the chunk's first byte. seq32 / qual32: the same offsets as rec.seq_off /
// rec.qual_off, in the width fl_reads_push_bam takes.
struct BamChunkIndex {
    Records rec;
    std::vector<uint32_t> seq32, qual32;
    std::vector<uint8_t> reverse;         // aligned: per read record, 1 when it is reverse-complemented (flag 0x10)
    std::vector<Follower> followers;      // aligned: the secondary and supplementary records (`before` counts rec)
    std::string error;            // why the first record that failed a check failed (then the index stops there)
};

// Checks and indexes the records of chunk c of the inflated input b: fields inside the record, aux fields that parse up
// to its end, unaligned (flag 0x4 set, 0x10 / 0x100 / 0x800 clear, no CIGAR), l_seq >= 1, name bytes in '!'..'~'.
// false: ix.error says why, naming the record by its byte offset in the inflated input or by its read name.
//
// aligned (--aligned): records may be aligned. A record with flag & 0x900 == 0 is a read record, indexed in ix.rec with
// its reverse flag; it needs l_seq >= 1 and, when mapped (0x4 clear), a CIGAR without H whose query length (M I S = X)
// is l_seq, so that the record holds the whole read. Any other record is a follower (ix.followers): it is not scored
// and may have no SEQ. Both get the checks every record gets.
bool bam_index_chunk(const char *b, const Chunk &c, BamChunkIndex &ix, bool aligned = false);

// Appends chunk c's index to a part's tables, as file offsets: its read records to R (their reverse flags to rev when
// given), its followers to F, counted among R's reads.
void bam_append_chunk(const BamChunkIndex &ix, const Chunk &c, Records &R, std::vector<Follower> &F, std::vector<uint8_t> *rev = nullptr);

// Finds each follower's read record by name (names: the parts' Records, in order) and sets its owner; returns the
// number of orphans.
uint64_t bam_join_followers(const char *b, const NameIndex &names, std::vector<Follower> &F);

// the record whose read_name starts at `name`: its first byte (block_size) and its size
inline const char *bam_record_of(const char *name) { return name - 36; }
uint64_t bam_record_bytes(const char *rec);
uint32_t bam_l_seq(const char *rec);
// QUAL of the record starts with 0xFF: the record has no quality
inline bool bam_no_quality(const char *qual) { return (unsigned char)qual[0] == 0xFF; }

// Appends to `out` the record of a child [start, end) of `rec` (0 <= start < end <= l_seq): the parent's fixed fields,
// read_name name_<start+1>-<end>, SEQ and QUAL of the slice (QUAL all 0xFF when the parent has none), and of the aux
// fields the parent's RG; with keep_mods, when the parent's MM / ML / MN are valid, then its MM and ML re-based to the
// child (fl_bam_mods.h) and MN:I = end - start. Throws std::runtime_error when the child's name does not fit in a BAM
// record. Returns FL_BAM_MODS_KEPT, FL_BAM_MODS_INVALID (keep_mods, the parent has an MM tag and its tags are not
// valid) or 0.
int bam_child_record(const char *rec, int start, int end, std::string &out, bool keep_mods = false);

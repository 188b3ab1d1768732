// filtlong_b200/csrc/host/survivors.h -- pass 2 of the CLI: the surviving reads and child rows in input order, as the
// reference prints them (reference src/main.cpp:263-313), and the stderr blocks that lead up to it. The only code that
// knows that output layout and how the bytes reach the descriptor. Two sources feed it:
//   * random access: the mapped input (or an inflated BAM file) and a table of where each record sits (the device feeder's, one part per shard, or
//     the host reader's when every record was simple). To BGZF; to pwrite() groups written by a few threads when the
//     descriptor is a regular file not opened with O_APPEND; else to writev().
//   * sequential: the input parsed again by FastxReader (streamed gzip, CR LF, multi-line records), copied through a
//     buffer or into BGZF.
// Every writer writes the rows whose final pass flag equals `want`: stdout gets the survivors (true), `--failed FILE` the
// rest (false), with the same bytes a survivor would have. Every writer returns false when a write (or a compression)
// failed.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../../include/filtlong_b200.h"
#include "arguments.h"
#include "fastx.h"

// Where each record sits in the mapped input, as file offsets. A comment starts one byte after its name (the device and
// FastxReader both guarantee it).
struct Records {
    std::vector<uint64_t> name_off, seq_off, qual_off, name_hash;
    std::vector<uint32_t> name_len, comment_len;
    std::vector<int32_t> len;
    size_t n = 0;
    bool lead_checked = false;    // every name follows the format's lead character (the device checked it)
    void ensure(size_t cap) {
        if (name_off.size() >= cap) return;
        const size_t c = cap + cap / 2;
        name_off.resize(c); seq_off.resize(c); qual_off.resize(c); name_hash.resize(c);
        name_len.resize(c); comment_len.resize(c); len.resize(c);
    }
    void add(uint64_t name_o, uint32_t name_l, uint32_t comment_l, uint64_t seq_o, uint64_t qual_o, int32_t length) {
        ensure(n + 1);
        name_off[n] = name_o; name_len[n] = name_l; comment_len[n] = comment_l;
        seq_off[n] = seq_o; qual_off[n] = qual_o; len[n] = length;
        ++n;
    }
    bool within(uint64_t file_size, bool quality) const;   // every piece that is printed lies inside the file
};

// Read-only view of the results pass 2 needs. ReadSet and the feeder's shards hold these arrays under these names.
struct Results {
    const int32_t *n_child;
    const uint64_t *row_start;
    const int32_t *row_s, *row_e;
    const uint8_t *row_pfinal;
    template <class T> static Results of(const T &t) {
        return Results{t.n_child.data(), t.row_start.data(), t.row_s.data(), t.row_e.data(), t.row_pfinal.data()};
    }
};

struct Format {
    char lead;                    // '>' or '@'
    bool quality;                 // print "+" and the quality
    bool bam = false;             // BAM records (bam.h) instead of text; then lead and quality are not used
    uint64_t bam_header = 0;      // BAM: bytes [0, bam_header) of the input are the header, written first
    uint64_t bam_max_record = 0;  // BAM: the largest record of the input
    bool keep_mods = false;       // BAM, --keep_mods: children keep their parent's modification tags, re-based
};

// BAM --aligned: a secondary or supplementary record. It is not scored; it is written when its read record (the one of
// the same name) is, and an orphan (no read record has its name) only to --failed.
struct Follower {
    uint64_t off;                 // its first byte (block_size), a file offset
    uint64_t before;              // the index in its part's Records of the read record after it (Records::n: none)
    uint64_t name_hash;           // fl_name_hash of its read_name
    int32_t owner_part = -1;      // its read record: part, and index in that part's Records; -1: an orphan
    uint64_t owner = 0;
};

struct Part {                     // one part of the table, with its results
    const Records *rec;
    Results res;
    const std::vector<Follower> *followers = nullptr;   // BAM --aligned: in file order
};

// The read names of one or more tables: a flat open-addressing table over the 64-bit hashes computed with the records,
// names compared byte for byte in the input only when two hashes agree; no string is built.
class NameIndex {
public:
    // tables[t] in order; false: *dup is the first name met twice (the table is then incomplete)
    bool build(const std::vector<const Records *> &tables, const char *base, std::string *dup);
    // the record named name[0, len) whose hash is h: true, *table and *index set
    bool find(uint64_t h, const char *name, uint32_t len, int32_t *table, uint64_t *index) const;

private:
    std::vector<const Records *> tables_;
    const char *base_ = nullptr;
    std::vector<uint64_t> keys_, at_;          // at_: (table << 56 | index) + 1, 0 for a free slot
    size_t mask_ = 0;
};

// name_<start+1>-<end>, a child read's name (reference src/read.cpp:135-136), appended to `out`
inline void append_child_name(std::string &out, const char *name, size_t name_len, int start, int end) {
    out.append(name, name_len);
    out += '_';
    out += std::to_string(start + 1);
    out += '-';
    out += std::to_string(end);
}

// Random access: the survivors of `parts`, in order, from the input mapped at `base`; compressed on the context `bgzf`
// when it is given. The last two are the choices write_survivors makes, callable directly. BAM (fmt.bam): the header,
// then each kept read's record as it is and a new record for each kept child; the CLI always passes a context, without
// one the uncompressed BAM stream is written. A second output is a second call, on its descriptor with want = false.
// With the context the children are built on its device (bgzf_out.h). mods_counts, when given, gets the children that
// kept modification tags and those whose parent's tags are invalid (fmt.keep_mods).
bool write_survivors(int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, fl_ctx *bgzf, bool want = true,
                     uint64_t *mods_counts = nullptr);
bool write_survivors_writev(int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, bool want = true);
bool write_survivors_pwrite(int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, bool want = true);
// Both outputs of a random-access source: the survivors to fd, then, with --failed, the other rows to args.failed_fd (a
// failure there reported by report_failed_write). With fmt.keep_mods, then one stderr line with stdout's mods_counts.
// True when both were written.
bool write_outputs(const Arguments &args, int fd, const char *base, const std::vector<Part> &parts, const Format &fmt, fl_ctx *bgzf);
// Sequential: the survivors among the first n_reads records of `input` (a path, or bytes in memory), parsed again. With
// failed_fd >= 0 the same parse also writes the other rows to failed_fd (compressed too when bgzf is given), and
// *failed_ok (when given) tells whether that output was written; the return value is stdout's.
bool reparse_survivors(int fd, const FastxInput &input, const Results &res, size_t n_reads, const Format &fmt, fl_ctx *bgzf,
                       int failed_fd = -1, bool *failed_ok = nullptr);
// --failed: `ok`, after printing an error that names the file when it is false
bool report_failed_write(const Arguments &args, bool ok);

// "  after trimming / splitting: N reads (B bp)" when --trim or --split is on, then a blank line (main.cpp:157-167)
void log_after_trim_split(const Arguments &args, uint64_t n_rows, const fl_summary &summary);
// the "Filtering long reads" block, when a target is set (main.cpp:218-261)
void log_filtering(const Arguments &args, const fl_summary &summary);

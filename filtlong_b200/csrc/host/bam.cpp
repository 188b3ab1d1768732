// filtlong_b200/csrc/host/bam.cpp -- see bam.h.
#include "bam.h"

#include <string.h>
#include <zlib.h>

#include <algorithm>
#include <stdexcept>

#include "../fl_bam_mods.h"
#include "../fl_name_hash.h"

namespace {

// a record's fixed fields, offsets from its first byte (block_size)
constexpr uint64_t kFixed = 36;        // block_size + the 32 bytes up to read_name
constexpr int kLReadName = 12, kNCigar = 16, kFlag = 18, kLSeq = 20;

inline uint32_t u32(const char *p) {
    uint32_t v;
    memcpy(&v, p, 4);
    return v;
}
inline uint16_t u16(const char *p) {
    uint16_t v;
    memcpy(&v, p, 2);
    return v;
}

// the aux field at p (tag, type, value) ends at *next, not after `end`; false if it does not parse
bool aux_field(const char *p, const char *end, const char **next) {
    const uint8_t *n = fl_aux_next((const uint8_t *)p, (const uint8_t *)end);
    if (n) *next = (const char *)n;
    return n != nullptr;
}

std::string at_byte(uint64_t off) { return "record at byte " + std::to_string(off); }

}  // namespace

bool bam_file_magic(const std::string &path) {
    gzFile z = gzopen(path.c_str(), "rb");
    if (!z) return false;
    char m[4];
    const bool yes = !gzdirect(z) && gzread(z, m, 4) == 4 && bam_magic(m, 4);
    gzclose(z);
    return yes;
}

bool bam_header(const char *b, uint64_t size, uint64_t *end, std::string *why) {
    auto fail = [&](const char *what) { *why = std::string("malformed BAM header: ") + what; return false; };
    if (!bam_magic(b, size)) return fail("no BAM magic");
    if (size < 12) return fail("the header runs past the end of the file");
    uint64_t p = 8 + (uint64_t)u32(b + 4);                                   // l_text
    if (p + 4 > size) return fail("the header text runs past the end of the file");
    const uint32_t n_ref = u32(b + p);
    p += 4;
    for (uint32_t r = 0; r < n_ref; ++r) {
        if (p + 4 > size) return fail("the reference entries run past the end of the file");
        p += 4 + (uint64_t)u32(b + p) + 4;                                    // l_name, name, l_ref
        if (p > size) return fail("the reference entries run past the end of the file");
    }
    *end = p;
    return true;
}

bool bam_plan_chunks(const char *b, uint64_t size, uint64_t header_end, uint64_t target, std::vector<Chunk> &out, uint64_t *max_chunk,
                     std::string *why, uint64_t *max_record) {
    const uint64_t kMaxChunk = (1ull << 31) - 1;
    uint64_t p = header_end, lo = header_end, biggest = 0, biggest_record = 0;
    auto cut = [&](uint64_t e) {
        out.push_back(Chunk{lo, e});
        biggest = std::max(biggest, e - lo);
        lo = e;
    };
    while (p < size) {
        if (size - p < 4) { *why = "malformed BAM input: " + at_byte(p) + " runs past the end of the file"; return false; }
        const uint64_t bs = u32(b + p);
        if (bs < 32) { *why = "malformed BAM input: " + at_byte(p) + " has block_size < 32"; return false; }
        if (bs + 4 > size - p) { *why = "malformed BAM input: " + at_byte(p) + " runs past the end of the file"; return false; }
        if (bs + 4 > kMaxChunk) { *why = "BAM " + at_byte(p) + " is larger than 2 GiB"; return false; }
        const uint64_t e = p + 4 + bs;
        biggest_record = std::max(biggest_record, 4 + bs);
        if (e - lo > target && p > lo) cut(p);                              // the record starts the next chunk
        p = e;
    }
    if (p > lo) cut(p);
    *max_chunk = biggest;
    if (max_record) *max_record = biggest_record;
    return true;
}

bool bam_index_chunk(const char *b, const Chunk &c, BamChunkIndex &ix, bool aligned) {
    Records &R = ix.rec;
    R.n = 0;
    ix.seq32.clear();
    ix.qual32.clear();
    ix.reverse.clear();
    ix.followers.clear();
    ix.error.clear();
    const char *base = b + c.begin;
    uint64_t p = 0;
    const uint64_t n_bytes = c.end - c.begin;
    while (p < n_bytes) {
        const char *r = base + p;
        const uint64_t bs = u32(r), at = c.begin + p;                         // the chain itself was checked by bam_plan_chunks
        const char *end = r + 4 + bs;
        const uint64_t l_name = (uint8_t)r[kLReadName], n_cigar = u16(r + kNCigar), l_seq = u32(r + kLSeq);
        const unsigned flag = u16(r + kFlag);
        const char *name = r + kFixed;
        if (l_name < 2 || l_name > bs - 32 || name[l_name - 1] != 0) {
            ix.error = "malformed BAM input: the read name of the " + at_byte(at) + " does not end with its NUL";
            return false;
        }
        if (l_name + 4 * n_cigar + (l_seq + 1) / 2 + l_seq > bs - 32) {
            ix.error = "malformed BAM input: the fields of the " + at_byte(at) + " do not fit in its block_size";
            return false;
        }
        const char *seq = name + l_name + 4 * n_cigar, *qual = seq + (l_seq + 1) / 2;
        for (const char *a = qual + l_seq; a < end;) {
            if (!aux_field(a, end, &a)) {
                ix.error = "malformed BAM input: the aux fields of the " + at_byte(at) + " do not parse up to its end";
                return false;
            }
        }
        const std::string shown(name, l_name - 1);
        const bool follower = aligned && (flag & 0x900);
        if (!aligned && (!(flag & 0x4) || (flag & 0x910) || n_cigar != 0)) {
            ix.error = "BAM input must be unaligned: read " + shown + " has flag " + std::to_string(flag) + " and " +
                       std::to_string(n_cigar) + " CIGAR operations";
            return false;
        }
        if (!follower && l_seq < 1) {
            ix.error = "BAM read " + shown + " has no sequence";
            return false;
        }
        if (aligned && !follower && !(flag & 0x4)) {                           // mapped: the record must hold the whole read
            uint64_t query = 0;
            bool hard = false;
            for (uint64_t k = 0; k < n_cigar; ++k) {
                const uint32_t op = u32(name + l_name + 4 * k), code = op & 15u;
                if (code > 8) {
                    ix.error = "BAM read " + shown + " has a CIGAR operation of code " + std::to_string(code);
                    return false;
                }
                hard = hard || code == 5;
                if (code == 0 || code == 1 || code == 4 || code == 7 || code == 8) query += op >> 4;   // M I S = X
            }
            if (hard) {
                ix.error = "BAM read " + shown + ": its primary record is hard-clipped";
                return false;
            }
            if (query != l_seq) {
                ix.error = "BAM read " + shown + ": the query length of its CIGAR (" + std::to_string(query) + ") is not its l_seq (" +
                           std::to_string(l_seq) + ")";
                return false;
            }
        }
        for (uint64_t i = 0; i + 1 < l_name; ++i)
            if ((unsigned char)name[i] < '!' || (unsigned char)name[i] > '~') {
                ix.error = "BAM read name with a byte outside '!'..'~' in the " + at_byte(at);
                return false;
            }
        if (follower) {
            ix.followers.push_back(Follower{p, R.n, fl_name_hash((const unsigned char *)name, l_name - 1)});
            p += 4 + bs;
            continue;
        }
        const uint64_t name_off = (uint64_t)(name - base), seq_off = (uint64_t)(seq - base), qual_off = (uint64_t)(qual - base);
        R.add(name_off, (uint32_t)(l_name - 1), 0, seq_off, qual_off, (int32_t)l_seq);
        R.name_hash[R.n - 1] = fl_name_hash((const unsigned char *)name, l_name - 1);
        ix.seq32.push_back((uint32_t)seq_off);
        ix.qual32.push_back((uint32_t)qual_off);
        if (aligned) ix.reverse.push_back((flag & 0x10) ? 1 : 0);
        p += 4 + bs;
    }
    return true;
}

void bam_append_chunk(const BamChunkIndex &ix, const Chunk &c, Records &R, std::vector<Follower> &F, std::vector<uint8_t> *rev) {
    const Records &X = ix.rec;
    for (Follower f : ix.followers) {
        f.off += c.begin;
        f.before += R.n;
        F.push_back(f);
    }
    R.ensure(R.n + X.n);
    for (size_t j = 0; j < X.n; ++j, ++R.n) {
        R.name_off[R.n] = X.name_off[j] + c.begin; R.seq_off[R.n] = X.seq_off[j] + c.begin; R.qual_off[R.n] = X.qual_off[j] + c.begin;
        R.name_len[R.n] = X.name_len[j]; R.comment_len[R.n] = 0; R.len[R.n] = X.len[j]; R.name_hash[R.n] = X.name_hash[j];
    }
    if (rev) rev->insert(rev->end(), ix.reverse.begin(), ix.reverse.end());
}

uint64_t bam_join_followers(const char *b, const NameIndex &names, std::vector<Follower> &F) {
    uint64_t orphans = 0;
    for (Follower &f : F) {
        const char *rec = b + f.off;
        f.owner_part = -1;
        if (!names.find(f.name_hash, rec + kFixed, (uint32_t)(uint8_t)rec[kLReadName] - 1, &f.owner_part, &f.owner)) {
            f.owner_part = -1;
            ++orphans;
        }
    }
    return orphans;
}

uint64_t bam_record_bytes(const char *rec) { return 4 + (uint64_t)u32(rec); }
uint32_t bam_l_seq(const char *rec) { return u32(rec + kLSeq); }

int bam_child_record(const char *rec, int start, int end, std::string &out, bool keep_mods) {
    const uint64_t l_name = (uint8_t)rec[kLReadName], n_cigar = u16(rec + kNCigar), l_seq = u32(rec + kLSeq);
    const char *name = rec + kFixed, *seq = name + l_name + 4 * n_cigar, *qual = seq + (l_seq + 1) / 2, *rec_end = rec + bam_record_bytes(rec);
    std::string nm(name, l_name - 1);
    nm += '_';
    nm += std::to_string(start + 1);
    nm += '-';
    nm += std::to_string(end);
    if (nm.size() + 1 > 255) throw std::runtime_error("the name of child read " + nm + " is too long for a BAM record");
    const uint32_t n = (uint32_t)(end - start);
    const size_t at = out.size();
    out.append(rec, kFixed);                                                 // block_size (set below) and the fixed fields
    out[at + kLReadName] = (char)(nm.size() + 1);
    memcpy(&out[at + kLSeq], &n, 4);
    out.append(nm.data(), nm.size());
    out += '\0';
    const auto nib = [&](uint32_t i) -> unsigned { const unsigned char x = (unsigned char)seq[i >> 1]; return (i & 1) ? (x & 15u) : (x >> 4); };
    for (uint32_t j = 0; j < n; j += 2) {
        const unsigned hi = nib((uint32_t)start + j), lo = j + 1 < n ? nib((uint32_t)start + j + 1) : 0u;
        out += (char)((hi << 4) | lo);
    }
    if (bam_no_quality(qual)) out.append(n, (char)0xFF);
    else out.append(qual + start, n);
    for (const char *a = qual + l_seq; a < rec_end;) {                        // the RG fields, then the modification tags
        const char *next = rec_end;
        aux_field(a, rec_end, &next);
        if (a[0] == 'R' && a[1] == 'G') out.append(a, (size_t)(next - a));
        a = next;
    }
    int status = 0;
    FlModTags t;
    fl_mod_tags((const uint8_t *)qual + l_seq, (const uint8_t *)rec_end, (int64_t)l_seq, &t);
    if (keep_mods && t.has_mm) {
        uint64_t total[5] = {0, 0, 0, 0, l_seq}, before_s[5] = {0, 0, 0, 0, (uint64_t)start}, before_e[5] = {0, 0, 0, 0, (uint64_t)end};
        for (uint32_t i = 0; i < l_seq; ++i)
            for (int b = 0; b < 4; ++b)
                if (nib(i) == fl_mm_code(b)) {
                    ++total[b];
                    before_s[b] += i < (uint32_t)start;
                    before_e[b] += i < (uint32_t)end;
                }
        status = FL_BAM_MODS_INVALID;
        if (fl_mods_valid(t, total)) {
            status = FL_BAM_MODS_KEPT;
            std::string mm, ml;
            uint64_t ml_at = 0, calls;
            for (uint32_t p = 0; p < t.mm_len;) {
                uint32_t head, codes;
                int b;
                fl_mm_head(t.mm, t.mm_len, p, &head, &b, &codes);
                mm.append((const char *)t.mm + p, head);
                FlMMCursor cur = fl_mm_cursor(p + head);
                std::string deltas(t.mm_len, '\0');                                 // no longer than the parent's
                uint64_t k0, k1;
                deltas.resize(fl_mm_rebase(t.mm, t.mm_len, cur, before_s[b], before_e[b], (uint8_t *)&deltas[0], &k0, &k1));
                mm += deltas;
                mm += ';';
                if (t.has_ml) ml.append((const char *)t.ml + ml_at + k0 * codes, (size_t)((k1 - k0) * codes));
                p = fl_mm_group_end(t.mm, cur, &calls);
                ml_at += calls * codes;
            }
            std::string mm_field = "MMZ" + mm;
            mm_field += '\0';
            std::string ml_field;
            if (t.has_ml) {
                const uint32_t k = (uint32_t)ml.size();
                ml_field = "MLBC";
                ml_field.append((const char *)&k, 4);
                ml_field += ml;
            }
            out += t.ml_first ? ml_field + mm_field : mm_field + ml_field;
            out += "MNI";
            out.append((const char *)&n, 4);
        }
    }
    const uint32_t bs = (uint32_t)(out.size() - at - 4);
    memcpy(&out[at], &bs, 4);
    return status;
}

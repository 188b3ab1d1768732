// tests/stream_dump.cpp -- test helper for input read from a stream (filtlong_b200/csrc/host/streamsrc.cpp, textsrc.cpp):
// reads standard input the way the CLI reads `-`, cutting chunks with plan_next_chunk while the bytes arrive as the
// feeder's planner does, then finishes the stream (gzip is inflated) and writes what it holds:
//     stream_dump <budget_bytes> <target_bytes> <buffer_out>
// <buffer_out> gets the bytes held in memory. stdout: "CHUNK <begin> <end> <last>" per chunk cut while the stream
// arrived (plain text only; "NOPLAN" if the planner gave up), "EARLY <n>" (chunks cut before the end), then "HELD <size>
// <inflated> <stream_bytes>", "SAME <0|1>" (plan_chunks over the whole buffer cuts the same chunks), and one line per
// record the memory-backed FastxReader reads chunk by chunk: "REC <name>^A<comment>^A<seq>^A<qual>", then "END <code>".
// A stream that cannot be held: its message on stderr, exit 1.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../filtlong_b200/csrc/host/fastx.h"
#include "../filtlong_b200/csrc/host/streamsrc.h"
#include "../filtlong_b200/csrc/host/textsrc.h"

int main(int argc, char **argv) {
    if (argc < 4) return 64;
    const uint64_t budget = strtoull(argv[1], nullptr, 10), target = strtoull(argv[2], nullptr, 10);
    StreamInput s;
    s.start("-", budget);
    bool ended = false;
    uint64_t avail = s.wait_for(2, &ended);
    const char b0 = avail ? s.base()[0] : 0;
    const int format = b0 == '@' ? FL_TEXT_FASTQ : b0 == '>' ? FL_TEXT_FASTA : 0;
    std::vector<Chunk> plan;
    bool planned = format != 0, gave_up = false;
    size_t early = 0;
    for (uint64_t pos = 0; planned;) {                                   // the feeder's planner thread, inline
        Chunk c;
        int r;
        while ((r = plan_next_chunk(s.base(), avail, ended, format, target, target, pos, &c)) == 1) {
            pos = c.end;
            plan.push_back(c);
            if (!ended) ++early;
            printf("CHUNK %llu %llu %d\n", (unsigned long long)c.begin, (unsigned long long)c.end, (int)(ended && pos == avail));
        }
        if (r < 0) { gave_up = true; break; }
        if (ended) break;
        avail = s.wait_for(std::max(avail + 1, pos + target + 1), &ended);
    }
    if (gave_up) printf("NOPLAN\n");
    printf("EARLY %zu\n", early);
    std::string why;
    if (!s.finish(&why)) {
        fprintf(stderr, "%s\n", why.c_str());
        return 1;
    }
    const MappedFile &f = s.file();
    FILE *o = fopen(argv[3], "wb");
    if (!o || (f.size && fwrite(f.base, 1, (size_t)f.size, o) != f.size) || fclose(o) != 0) return 2;
    printf("HELD %llu %d %llu\n", (unsigned long long)f.size, (int)s.inflated(), (unsigned long long)s.stream_bytes());
    std::vector<Chunk> whole;
    const bool same = planned && !gave_up && plan_chunks(f.base, f.size, format, target, target, whole) && whole.size() == plan.size() &&
                      std::equal(plan.begin(), plan.end(), whole.begin(), [](const Chunk &a, const Chunk &b) { return a.begin == b.begin && a.end == b.end; });
    printf("SAME %d\n", (int)same);
    if (!planned || gave_up) plan.assign(1, Chunk{0, f.size});
    long long l = -1;
    for (const Chunk &c : plan) {
        FastxReader in(f.base + c.begin, c.end - c.begin);
        while ((l = in.next()) >= 0) printf("REC %s\x01%s\x01%s\x01%s\n", in.name.c_str(), in.comment.c_str(), in.seq.c_str(), in.qual.c_str());
        if (l != -1) break;
    }
    printf("END %lld\n", l);
    return 0;
}

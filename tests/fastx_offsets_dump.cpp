// tests/fastx_offsets_dump.cpp -- prints, for every record of each FASTA/FASTQ file named, what FastxReader parsed
// and where it says the pieces sit in the byte stream, so a test can check the slices against the file. The last
// three columns are FNV-1a hashes of the comment, the sequence and the quality, every byte of them.
#include <cstdio>

#include "../filtlong_b200/csrc/host/fastx.h"

static unsigned long long fnv(const std::string &s) {
    unsigned long long h = 0xCBF29CE484222325ull;
    for (unsigned char c : s) h = (h ^ c) * 0x100000001B3ull;
    return h;
}

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    for (int a = 1; a < argc; ++a) {
        FastxReader in(argv[a]);
        if (!in.ok()) return 3;
        long long l;
        while ((l = in.next()) >= 0)
            printf("%s\t%zu\t%zu\t%zu\t%d\t%llu\t%llu\t%llu\t%d\t%llu\t%016llx\t%016llx\t%016llx\n", in.name.c_str(), in.comment.size(),
                   in.seq.size(), in.qual.size(), (int)in.simple, (unsigned long long)in.comment_off, (unsigned long long)in.seq_off,
                   (unsigned long long)in.qual_off, (int)in.plain(), (unsigned long long)in.name_off, fnv(in.comment), fnv(in.seq), fnv(in.qual));
        printf("END %lld\n", l);
    }
    return 0;
}

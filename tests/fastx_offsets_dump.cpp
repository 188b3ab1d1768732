// tests/fastx_offsets_dump.cpp -- prints, for every record of a FASTA/FASTQ file, what FastxReader parsed
// and where it says the pieces sit in the byte stream, so a test can check the slices against the file.
#include <cstdio>

#include "../filtlong_b200/csrc/host/fastx.h"

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    FastxReader in(argv[1]);
    if (!in.ok()) return 3;
    long long l;
    while ((l = in.next()) >= 0)
        printf("%s\t%zu\t%zu\t%zu\t%d\t%llu\t%llu\t%llu\t%d\t%llu\n", in.name.c_str(), in.comment.size(), in.seq.size(), in.qual.size(),
               (int)in.simple, (unsigned long long)in.comment_off, (unsigned long long)in.seq_off, (unsigned long long)in.qual_off,
               (int)in.plain(), (unsigned long long)in.name_off);
    printf("END %lld\n", l);
    return 0;
}

// filtlong_b200/csrc/host/arguments.h -- command-line options of the `filtlong` drop-in.
// Same public surface as the reference's Arguments (reference src/arguments.h:50-96); the parser
// behind it is our own (no vendored args.h) and reproduces the option syntax, value readers,
// validation order and error strings the reference's tests pin (SURVEY Appendix B).
#pragma once
#include <string>
#include <vector>

enum ParsingResult { GOOD, BAD, HELP, VERSION };

class Arguments {
public:
    Arguments(int argc, char **argv);

    ParsingResult parsing_result;
    std::string input_reads;

    bool target_bases_set = false;
    long long target_bases = 0;
    bool keep_percent_set = false;
    double keep_percent = 0.0;
    bool min_length_set = false;
    int min_length = 0;
    bool max_length_set = false;
    int max_length = 0;
    bool min_mean_q_set = false;
    double min_mean_q = 0.0;
    bool min_window_q_set = false;
    double min_window_q = 0.0;

    bool assembly_set = false;
    std::string assembly;
    std::vector<std::string> short_reads;

    double length_weight = 1.0;
    double mean_q_weight = 1.0;
    double window_q_weight = 1.0;

    bool trim = false;
    bool split_set = false;
    int split = 0;
    int trim_q = 0;               // this build only: --trim / --split on Phred qualities without a reference (0 = off)
    // this build only: reads with more than max_contam percent of their bases in 16-mers of this file are removed
    bool contam_set = false;
    std::string contam;
    bool max_contam_set = false;
    double max_contam = 50.0;
    bool contam_k_set = false;
    int contam_k = 16;            // the length of the contaminant k-mers (16 to 32)

    int window_size = 250;
    bool verbose = false;
    int gpus = 1;                 // this build only: shard the read set across this many GPUs (one context + one thread each)
    bool bgzip = false;           // this build only: stdout compressed as BGZF on the GPU (bgzf_out.h)
    bool keep_mods = false;       // this build only: BAM children keep their parent's MM / ML tags, re-based (fl_bam_mods.h)
    bool aligned = false;         // this build only: BAM input may be aligned; secondary / supplementary records follow their read
    // this build only: the rows stdout does not get go to this file, opened (O_TRUNC) while the arguments are checked
    bool failed_set = false;
    std::string failed;
    int failed_fd = -1;

private:
    bool does_file_exist(const std::string &filename);
    bool reads_exist(const std::string &filename);
};

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

    int window_size = 250;
    bool verbose = false;
    int gpus = 1;                 // this build only: shard the read set across this many GPUs (one context + one thread each)

private:
    bool does_file_exist(const std::string &filename);
};

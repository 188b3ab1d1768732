// filtlong_b200/csrc/host/arguments.cpp -- see arguments.h. Behaviour follows reference
// src/arguments.cpp:28-400 (value readers 28-113, option table 152-222, validation 253-393).
#include "arguments.h"

#include <algorithm>
#include <cctype>
#include <climits>
#include <fstream>
#include <iostream>
#include <sstream>
#include <stdexcept>

namespace {

struct ParseError : std::runtime_error {
    using std::runtime_error::runtime_error;
};
struct HelpRequested {};

// arguments.cpp:28-39: only digits and dots, then std::stod
double read_double(const std::string &name, const std::string &value) {
    try {
        if (value.find_first_not_of("0123456789.") != std::string::npos) throw std::invalid_argument("");
        return std::stod(value);
    } catch (...) {
        throw ParseError("Error: argument '" + name + "' received invalid value type '" + value + "'");
    }
}

// arguments.cpp:53-97: optional sign, decimals, optional k|kb|m|mb|g|gb (case-insensitive)
long long parse_int_with_suffix(const std::string &value) {
    if (value.empty()) throw std::invalid_argument("Empty value");
    std::string lower = value;
    std::transform(lower.begin(), lower.end(), lower.begin(), ::tolower);
    size_t start = value[0] == '-' ? 1 : 0;
    size_t suffix_pos = lower.find_first_not_of("0123456789.", start);
    if (suffix_pos == std::string::npos) return static_cast<long long>(std::stod(value));
    std::string numeric = value.substr(0, suffix_pos), suffix = lower.substr(suffix_pos);
    if (numeric.empty() || (numeric.size() == 1 && numeric[0] == '-')) throw std::invalid_argument("No numeric value");
    double v = std::stod(numeric);
    long long mult;
    if (suffix == "k" || suffix == "kb") mult = 1000;
    else if (suffix == "m" || suffix == "mb") mult = 1000000;
    else if (suffix == "g" || suffix == "gb") mult = 1000000000;
    else throw std::invalid_argument("Unknown suffix");
    return static_cast<long long>(v * mult);
}

long long read_ll_suffix(const std::string &name, const std::string &value) {        // arguments.cpp:42-51
    try {
        return parse_int_with_suffix(value);
    } catch (...) {
        throw ParseError("Error: argument '" + name + "' received invalid value '" + value + "'");
    }
}

int read_int_suffix(const std::string &name, const std::string &value) {             // arguments.cpp:100-113
    try {
        long long r = parse_int_with_suffix(value);
        if (r > INT_MAX || r < INT_MIN) throw std::invalid_argument("range");
        return static_cast<int>(r);
    } catch (...) {
        throw ParseError("Error: argument '" + name + "' received invalid value '" + value + "'");
    }
}

long long read_plain_ll(const std::string &name, const std::string &value) {         // args.h default reader
    std::istringstream ss(value);
    long long v = 0;
    ss >> v;
    if (ss.rdbuf()->in_avail() > 0)
        throw ParseError("Error: argument '" + name + "' received invalid value type '" + value + "'");
    return v;
}

struct Opt {
    char short_name;            // 0 if none
    const char *long_name;
    bool takes_value;
    const char *placeholder;    // the name used in reader error messages
    const char *help;
};

const Opt kOpts[] = {
    {'t', "target_bases", true, "int", "keep only the best reads up to this many total bases (unit suffixes: k, kb, m, mb, g, gb)"},
    {'p', "keep_percent", true, "float", "keep only this percentage of the best reads (measured by bases)"},
    {'l', "min_length", true, "int", "minimum length threshold (unit suffixes: k, kb, m, mb, g, gb)"},
    {'L', "max_length", true, "int", "maximum length threshold (unit suffixes: k, kb, m, mb, g, gb)"},
    {'q', "min_mean_q", true, "float", "minimum mean quality threshold"},
    {0, "min_window_q", true, "float", "minimum window quality threshold"},
    {'a', "assembly", true, "file", "reference assembly in FASTA format"},
    {'1', "short_1", true, "file", "reference short reads in FASTQ format"},
    {'2', "short_2", true, "file", "reference short reads in FASTQ format"},
    {0, "length_weight", true, "float", "weight given to the length score (default: 1)"},
    {0, "mean_q_weight", true, "float", "weight given to the mean quality score (default: 1)"},
    {0, "window_q_weight", true, "float", "weight given to the window quality score (default: 1)"},
    {0, "trim", false, "trim", "trim non-k-mer-matching bases from start/end of reads"},
    {0, "split", true, "split", "split reads at this many (or more) consecutive non-k-mer-matching bases (unit suffixes: k, kb, m, mb, g, gb)"},
    {0, "window_size", true, "int", "size of sliding window used when measuring window quality (default: 250)"},
    {0, "gpus", true, "int", "number of GPUs to shard the read set across (default: 1; not a reference option)"},
    {0, "verbose", false, "verbose", "verbose output to stderr with info for each read"},
    {0, "version", false, "version", "display the program version and quit"},
    {'h', "help", false, "help", "display this help menu"},
};

void print_help(const char *prog) {
    std::ostream &o = std::cerr;
    o << "usage: " << prog << " {OPTIONS} [input_reads]\n\n"
      << "Filtlong: a quality filtering tool for Nanopore and PacBio reads\n\n"
      << "positional arguments:\n   input_reads                          input long reads to be filtered\n\n";
    struct Group { const char *title; int first, last; };
    const Group groups[] = {
        {"output thresholds:", 0, 5},
        {"external references (if provided, read quality will be determined using these instead of from the Phred scores):", 6, 8},
        {"score weights (control the relative contribution of each score to the final read score):", 9, 11},
        {"read manipulation:", 12, 13},
        {"other:", 14, 18},
    };
    for (const Group &g : groups) {
        o << g.title << "\n";
        for (int i = g.first; i <= g.last; ++i) {
            const Opt &p = kOpts[i];
            std::string flags = "   ";
            if (p.short_name) flags += std::string("-") + p.short_name + (p.takes_value ? std::string("[") + p.placeholder + "], " : ", ");
            flags += std::string("--") + p.long_name + (p.takes_value ? std::string(" [") + p.placeholder + "]" : "");
            if (flags.size() < 40) flags += std::string(40 - flags.size(), ' ');
            o << flags << p.help << "\n";
        }
        o << "\n";
    }
    o << "For more information, go to: https://github.com/rrwick/Filtlong\n";
}

}  // namespace

Arguments::Arguments(int argc, char **argv) {
    parsing_result = GOOD;
    bool version_flag = false;
    std::string short_1, short_2;
    bool short_1_set = false, short_2_set = false, positional_set = false;
    long long window_ll = 250;

    auto apply = [&](const Opt &o, const std::string &v) {
        const std::string ln = o.long_name, nm = o.placeholder;
        if (ln == "target_bases") { target_bases = read_ll_suffix(nm, v); target_bases_set = true; }
        else if (ln == "keep_percent") { keep_percent = read_double(nm, v); keep_percent_set = true; }
        else if (ln == "min_length") { min_length = read_int_suffix(nm, v); min_length_set = true; }
        else if (ln == "max_length") { max_length = read_int_suffix(nm, v); max_length_set = true; }
        else if (ln == "min_mean_q") { min_mean_q = read_double(nm, v); min_mean_q_set = true; }
        else if (ln == "min_window_q") { min_window_q = read_double(nm, v); min_window_q_set = true; }
        else if (ln == "assembly") { assembly = v; assembly_set = true; }
        else if (ln == "short_1") { short_1 = v; short_1_set = true; }
        else if (ln == "short_2") { short_2 = v; short_2_set = true; }
        else if (ln == "length_weight") length_weight = read_double(nm, v);
        else if (ln == "mean_q_weight") mean_q_weight = read_double(nm, v);
        else if (ln == "window_q_weight") window_q_weight = read_double(nm, v);
        else if (ln == "trim") trim = true;
        else if (ln == "split") { split = read_int_suffix(nm, v); split_set = true; }
        else if (ln == "window_size") window_ll = read_plain_ll(nm, v);
        else if (ln == "gpus") gpus = (int)read_plain_ll(nm, v);
        else if (ln == "verbose") verbose = true;
        else if (ln == "version") version_flag = true;
        else if (ln == "help") throw HelpRequested();
    };

    try {
        bool terminated = false;
        for (int i = 1; i < argc; ++i) {
            const std::string arg = argv[i];
            if (!terminated && arg == "--") { terminated = true; continue; }
            if (!terminated && arg.size() > 2 && arg[0] == '-' && arg[1] == '-') {
                // long option: the value is always the NEXT token, taken wholesale (LongSeparator " ")
                const std::string nm = arg.substr(2);
                const Opt *o = nullptr;
                for (const Opt &c : kOpts) if (nm == c.long_name) o = &c;
                if (!o) throw ParseError("Error: flag could not be matched: " + nm);
                if (o->takes_value) {
                    if (i + 1 >= argc) throw ParseError("Error: flag '" + nm + "' requires an argument but received none");
                    apply(*o, argv[++i]);
                } else apply(*o, "");
            } else if (!terminated && arg.size() > 1 && arg[0] == '-' && arg[1] != '-') {
                // short option bundle; a value-taking flag ends the bundle (joined value or next token)
                for (size_t k = 1; k < arg.size(); ++k) {
                    const Opt *o = nullptr;
                    for (const Opt &c : kOpts) if (c.short_name && c.short_name == arg[k]) o = &c;
                    if (!o) throw ParseError(std::string("Error: flag could not be matched: '") + arg[k] + "'");
                    if (!o->takes_value) { apply(*o, ""); continue; }
                    if (k + 1 < arg.size()) apply(*o, arg.substr(k + 1));
                    else {
                        if (i + 1 >= argc) throw ParseError(std::string("Error: flag '") + arg[k] + "' requires an argument but received none");
                        apply(*o, argv[++i]);
                    }
                    break;
                }
            } else {
                if (positional_set)
                    throw ParseError("Error: passed in argument, but no positional arguments were ready to receive it: " + arg);
                input_reads = arg;
                positional_set = true;
            }
        }
    } catch (const HelpRequested &) {
        print_help(argv[0]);
        parsing_result = HELP;
        return;
    } catch (const ParseError &e) {
        std::cerr << e.what() << "\n";
        parsing_result = BAD;
        return;
    }
    if (argc == 1) {                                                     // arguments.cpp:243-247
        print_help(argc > 0 ? argv[0] : "filtlong");
        parsing_result = HELP;
        return;
    }
    if (version_flag) { parsing_result = VERSION; return; }
    window_size = static_cast<int>(window_ll);                           // arguments.cpp:294 (long long -> int)
    if (short_1_set) short_reads.push_back(short_1);
    if (short_2_set) short_reads.push_back(short_2);

    auto fail = [&](const std::string &msg) {
        std::cerr << msg << "\n";
        parsing_result = BAD;
    };
#define FAIL(msg) do { fail(msg); return; } while (0)
    if (input_reads.empty()) FAIL("Error: input reads are required");
    const bool some_reference = !short_reads.empty() || assembly_set;
    if (trim && !some_reference) FAIL("Error: assembly or read reference is required to use --trim");
    if (split_set && !some_reference) FAIL("Error: assembly or read reference is required to use --split");
    std::vector<std::string> files{input_reads};
    for (const auto &f : short_reads) files.push_back(f);
    if (assembly_set) files.push_back(assembly);
    for (const auto &f : files)
        if (!does_file_exist(f)) FAIL("Error: cannot find file: " + f);
    if (!trim && !split_set && !target_bases_set && !keep_percent_set && !min_length_set && !max_length_set &&
        !min_mean_q_set && !min_window_q_set)
        FAIL("Error: no thresholds set, you must use one of the following options:\n"
             "target_bases, keep_percent, min_length, max_length, min_mean_q, min_window_q, trim, split");
    if (target_bases_set && target_bases <= 0) FAIL("Error: the value for --target_bases must be a positive integer");
    if (min_length_set && min_length <= 0) FAIL("Error: the value for --min_length must be a positive integer");
    if (max_length_set && max_length <= 0) FAIL("Error: the value for --max_length must be a positive integer");
    if (keep_percent_set && (keep_percent <= 0.0 || keep_percent >= 100.0))
        FAIL("Error: the value for --keep_percent must be greater than 0 and less than 100");
    if (min_mean_q_set && min_mean_q <= 0.0) FAIL("Error: the value for --min_mean_q must be greater than 0");
    if (min_window_q_set && min_window_q <= 0.0) FAIL("Error: the value for --min_window_q must be greater than 0");
    if (length_weight < 0.0 || mean_q_weight < 0.0 || window_q_weight < 0.0) FAIL("Error: weight values cannot be negative");
    if (split_set && split <= 0) FAIL("Error: the value for --split must be a positive integer");
    if (window_size <= 0) FAIL("Error: the value for --window_size must be a positive integer");
    if (gpus < 1 || gpus > 64) FAIL("Error: the value for --gpus must be between 1 and 64");
}

bool Arguments::does_file_exist(const std::string &filename) {
    std::ifstream infile(filename);
    return infile.good();
}

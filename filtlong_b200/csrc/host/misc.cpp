// filtlong_b200/csrc/host/misc.cpp -- see misc.h
#include "misc.h"

#include <iomanip>
#include <iostream>
#include <locale>
#include <sstream>

std::string double_to_string(double n) {                 // misc.cpp:24-32
    std::ostringstream ss;
    ss << std::fixed << std::setprecision(2) << n;
    std::string s = ss.str();
    return s.size() < 5 ? std::string(5 - s.size(), ' ') + s : s;
}

std::string int_to_string(long long n) {                 // misc.cpp:35-40
    std::ostringstream ss;
    try {
        ss.imbue(std::locale(""));
    } catch (const std::exception &) {
        // the reference aborts here when LANG names a locale that is not installed; fall back to "C"
    }
    ss << std::fixed << n;
    return ss.str();
}

void print_hash_progress(const std::string &filename, long long base_count) {
    std::cerr << "\r  " << filename << " (" << int_to_string(base_count) << " bp)";
}

void print_read_score_progress(long long read_count, long long base_count) {
    std::cerr << "\r  " << int_to_string(read_count) << " reads (" << int_to_string(base_count) << " bp)";
}

void print_contam_removal(double max_contam, long long reads, long long bases, int k) {
    std::ostringstream pct;
    pct << max_contam;
    std::cerr << "Removing contaminant reads\n";
    std::cerr << "  " << int_to_string(reads) << " reads (" << int_to_string(bases) << " bp) with more than " << pct.str()
              << "% of bases in contaminant " << k << "-mers\n\n";
}

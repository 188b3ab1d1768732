// filtlong_b200/csrc/host/misc.h -- formatting helpers of the reference's stderr log
// (reference src/misc.cpp:24-49), locale-safe: an uninstalled LANG no longer aborts the program.
#pragma once
#include <string>

std::string double_to_string(double n);          // "%.2f", left-padded to 5 characters
std::string int_to_string(long long n);          // digit grouping of the user's locale, "C" if unavailable
void print_hash_progress(const std::string &filename, long long base_count);
void print_read_score_progress(long long read_count, long long base_count);
// --contam: "Removing contaminant reads" and the removed reads and bases (nothing without --contam)
void print_contam_removal(double max_contam, long long reads, long long bases, int k);

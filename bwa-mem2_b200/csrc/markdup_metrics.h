// markdup_metrics.h — the duplication metrics file of bm2_mem --markdup-metrics and bm2_markdup: Picard's DuplicationMetrics per library, the
// library-size estimate and the ROI histogram, restated from Picard's formulas (the rule is markdup_device.cuh's; byte equality with Picard is not claimed).
//
//   ## htsjdk.samtools.metrics.StringHeader
//   # bm2_mem (or bm2_markdup) <the arguments after the program name, joined by spaces>
//   (blank)
//   ## METRICS CLASS	picard.sam.DuplicationMetrics
//   LIBRARY	UNPAIRED_READS_EXAMINED	...	ESTIMATED_LIBRARY_SIZE      (the ten columns, tab-separated)
//   <one row of values per library>
//   (when there is one library and its size is defined) a blank line, "## HISTOGRAM	java.lang.Double", "BIN	CoverageMult", rows 1.0 .. 100.0
//
// Doubles are printed as %.6f with trailing zeros and a trailing '.' removed; there is no timestamp, so the file is deterministic.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

struct DupMetrics {
    std::string library = "Unknown Library";
    int64_t unpaired_reads = 0, read_pairs = 0, secondary_or_supplementary = 0, unmapped = 0, unpaired_dups = 0, pair_dups = 0, optical_pairs = 0;
};

// %.6f without trailing zeros and without a trailing '.'
inline std::string dup_metrics_double(double v) {
    char b[64];
    snprintf(b, sizeof b, "%.6f", v);
    std::string s(b);
    while (!s.empty() && s.back() == '0') s.pop_back();
    if (!s.empty() && s.back() == '.') s.pop_back();
    return s;
}

// Picard's estimateLibrarySize(pairs, unique): -1 (undefined) when pairs <= 0 or pairs - unique <= 0
inline int64_t dup_library_size(int64_t pairs, int64_t unique) {
    if (pairs <= 0 || pairs - unique <= 0) return -1;
    const double c = (double) unique, n = (double) pairs;
    auto f = [&](double x) { return c / x - 1 + std::exp(-n / x); };
    double m = 1.0, M = 100.0;
    while (f(M * c) > 0) M *= 10.0;
    for (int i = 0; i < 40; ++i) {
        const double r = (m + M) / 2.0, u = f(r * c);
        if (u == 0) break;
        if (u > 0) m = r; else M = r;
    }
    return (int64_t) (c * (m + M) / 2.0);
}

inline double dup_percent_duplication(const DupMetrics &x) {
    const int64_t den = x.unpaired_reads + 2 * x.read_pairs;
    return den ? (double) (x.unpaired_dups + 2 * x.pair_dups) / (double) den : 0.0;
}

// the file of one or more libraries' rows (in the order given) under "# <program> <args>"; the histogram only when there is exactly one row
// and its library size is defined
inline std::string dup_metrics_file(const std::vector<DupMetrics> &rows, const std::string &program, const std::string &args) {
    std::string o = "## htsjdk.samtools.metrics.StringHeader\n# " + program + (args.empty() ? std::string() : " " + args) + "\n\n";
    o += "## METRICS CLASS\tpicard.sam.DuplicationMetrics\n";
    o += "LIBRARY\tUNPAIRED_READS_EXAMINED\tREAD_PAIRS_EXAMINED\tSECONDARY_OR_SUPPLEMENTARY_RDS\tUNMAPPED_READS\tUNPAIRED_READ_DUPLICATES\t"
         "READ_PAIR_DUPLICATES\tREAD_PAIR_OPTICAL_DUPLICATES\tPERCENT_DUPLICATION\tESTIMATED_LIBRARY_SIZE\n";
    for (const DupMetrics &x : rows) {
        const int64_t L = dup_library_size(x.read_pairs - x.optical_pairs, x.read_pairs - x.pair_dups);
        o += x.library;
        for (int64_t v : { x.unpaired_reads, x.read_pairs, x.secondary_or_supplementary, x.unmapped, x.unpaired_dups, x.pair_dups, x.optical_pairs })
            o += "\t" + std::to_string(v);
        o += "\t" + dup_metrics_double(dup_percent_duplication(x)) + "\t" + (L >= 0 ? std::to_string(L) : std::string()) + "\n";
    }
    const int64_t L = rows.size() == 1 ? dup_library_size(rows[0].read_pairs - rows[0].optical_pairs, rows[0].read_pairs - rows[0].pair_dups) : -1;
    if (L >= 0) {
        const DupMetrics &x = rows[0];
        o += "\n## HISTOGRAM\tjava.lang.Double\nBIN\tCoverageMult\n";
        for (int k = 1; k <= 100; ++k) {
            const double v = (double) L * (1 - std::exp(-((double) k * (double) x.read_pairs) / (double) L)) / (double) (x.read_pairs - x.pair_dups);
            o += std::to_string(k) + ".0\t" + dup_metrics_double(v) + "\n";
        }
    }
    return o;
}

// bm2_mem's file: its one library
inline std::string dup_metrics_text(const DupMetrics &x, const std::string &args) { return dup_metrics_file({x}, "bm2_mem", args); }

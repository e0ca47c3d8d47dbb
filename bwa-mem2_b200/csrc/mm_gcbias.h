// mm_gcbias.h — the host side of bm2_multiplemetrics' GC bias: Picard's GcBiasDetailMetrics and GcBiasSummaryMetrics formulas and file
// text over bm2_mm_gc_finish's counts (the per-window and per-record rule is mm_device.cuh's).  Recalled from Picard's
// GcBiasMetricsCollector, not checked against Picard; byte equality with Picard is not claimed.
//
//   m          the mean coverage: sum READ_STARTS / sum WINDOWS over all bins
//   detail     one row per GC 0..100, empty bins included (our choice): WINDOWS, READ_STARTS; MEAN_BASE_QUALITY the integer
//              round(-10 log10(errors / bases)) when errors > 0, else 0; NORMALIZED_COVERAGE (READ_STARTS / WINDOWS) / m; ERROR_BAR_WIDTH
//              (sqrt(READ_STARTS) / WINDOWS) / m
//   summary    over the bins with WINDOWS >= 1e-5 * total windows, d = 100 WINDOWS / total windows - 100 READ_STARTS / total read starts; a
//              positive d adds to AT_DROPOUT when GC <= 50 and to GC_DROPOUT when GC >= 50.  GC_NC_a_b over the bins a..b with READ_STARTS > 0:
//              sum READ_STARTS / (sum WINDOWS * m), 0 without such a bin.
//   zero       a zero denominator gives 0, as in the tool's other files
//   file       mm_header's lines, the columns and the rows; doubles as dup_metrics_double prints them; no timestamp
#pragma once
#include "mm_metrics.h"
#include <cmath>
#include <string>

struct MmGcCounts {
    int64_t windows[MM_GC_BINS] = {}, reads[MM_GC_BINS] = {}, bases[MM_GC_BINS] = {}, errors[MM_GC_BINS] = {};
    int64_t clusters = 0, aligned = 0;
};

inline double mm_gc_ratio(double a, double b) { return b != 0 ? a / b : 0.0; }

// m: sum READ_STARTS / sum WINDOWS
inline double mm_gc_mean(const MmGcCounts &x) {
    int64_t r = 0, w = 0;
    for (int k = 0; k < MM_GC_BINS; ++k) { r += x.reads[k]; w += x.windows[k]; }
    return mm_gc_ratio((double) r, (double) w);
}

inline std::string mm_gc_detail_text(const MmGcCounts &x, const std::string &args) {
    std::string o = mm_header(args, "picard.analysis.GcBiasDetailMetrics");
    o += "ACCUMULATION_LEVEL\tREADS_USED\tGC\tWINDOWS\tREAD_STARTS\tMEAN_BASE_QUALITY\tNORMALIZED_COVERAGE\tERROR_BAR_WIDTH\tSAMPLE\tLIBRARY\tREAD_GROUP\n";
    const double m = mm_gc_mean(x);
    for (int k = 0; k < MM_GC_BINS; ++k) {
        const int64_t q = x.errors[k] > 0 ? (int64_t) std::floor(-10.0 * std::log10((double) x.errors[k] / (double) x.bases[k]) + 0.5) : 0;
        const double cov = mm_gc_ratio(mm_gc_ratio((double) x.reads[k], (double) x.windows[k]), m);
        const double bar = mm_gc_ratio(mm_gc_ratio(std::sqrt((double) x.reads[k]), (double) x.windows[k]), m);
        o += "All Reads\tALL\t" + std::to_string(k) + "\t" + std::to_string(x.windows[k]) + "\t" + std::to_string(x.reads[k]) + "\t" + std::to_string(q) +
             "\t" + dup_metrics_double(cov) + "\t" + dup_metrics_double(bar) + "\t\t\t\n";
    }
    return o;
}

inline std::string mm_gc_summary_text(const MmGcCounts &x, const std::string &args) {
    std::string o = mm_header(args, "picard.analysis.GcBiasSummaryMetrics");
    o += "ACCUMULATION_LEVEL\tREADS_USED\tWINDOW_SIZE\tTOTAL_CLUSTERS\tALIGNED_READS\tAT_DROPOUT\tGC_DROPOUT\tGC_NC_0_19\tGC_NC_20_39\tGC_NC_40_59\t"
         "GC_NC_60_79\tGC_NC_80_100\tSAMPLE\tLIBRARY\tREAD_GROUP\n";
    int64_t tw = 0, tr = 0;
    for (int k = 0; k < MM_GC_BINS; ++k) { tw += x.windows[k]; tr += x.reads[k]; }
    double at = 0, gc = 0;
    for (int k = 0; k < MM_GC_BINS; ++k) {
        if ((double) x.windows[k] < 1e-5 * (double) tw) continue;       // MINIMUM_GENOME_FRACTION
        const double d = mm_gc_ratio(100.0 * (double) x.windows[k], (double) tw) - mm_gc_ratio(100.0 * (double) x.reads[k], (double) tr);
        if (d > 0 && k <= 50) at += d;
        if (d > 0 && k >= 50) gc += d;
    }
    const double m = mm_gc_mean(x);
    o += "All Reads\tALL\t" + std::to_string(MM_GC_W) + "\t" + std::to_string(x.clusters) + "\t" + std::to_string(x.aligned) + "\t" + dup_metrics_double(at) +
         "\t" + dup_metrics_double(gc);
    static const int kRange[5][2] = {{0, 19}, {20, 39}, {40, 59}, {60, 79}, {80, 100}};
    for (const auto &rg : kRange) {
        int64_t r = 0, w = 0;
        for (int k = rg[0]; k <= rg[1]; ++k) if (x.reads[k] > 0) { r += x.reads[k]; w += x.windows[k]; }
        o += "\t" + dup_metrics_double(mm_gc_ratio((double) r, (double) w * m));
    }
    return o + "\t\t\t\n";
}

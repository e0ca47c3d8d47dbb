// bqsr_report.h — the host side of bm2_mem --recal-file: the empirical quality of a table row and the recalibration report's text, from the
// dense tables of bm2_bqsr_tables.  Restated in Python in tests/bqsr_util.py.
//
//   empirical quality   GATK's RecalDatum.bayesianEstimateOfEmpiricalQuality: with N = n + 2 observations and E = e + 1 errors (N above
//                       2^31 - 2: both scaled down to N = 2^31 - 2, E rounded half up), the argmax, lowest first, over Q = 0..60 of
//                       log10(0.9 exp(-d^2 / 0.5)), d = min(|(int) (Q - prior)|, 40), plus the binomial log10-likelihood of E errors in N at
//                       the error rate 10^(-Q/10) (an infinite or NaN likelihood counts as -DBL_MAX), capped at 93.  The binomial coefficient
//                       is the same for every Q, so it is left out: the argmax does not change.
//   report              GATKReport v1.1: Arguments (GATK 4's defaults), Quantized (qualities 0..93 mapped to themselves), RecalTable0 (the
//                       read group), RecalTable1 (quality), RecalTable2 (quality and context, then quality and cycle), event M only, the
//                       rows with at least one observation.  Each cell is padded to its column's widest, strings left, numbers right, two
//                       spaces apart.  No timestamp.
#pragma once
#include "bqsr_device.cuh"
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

inline int bqsr_empirical_q(int64_t n, int64_t e, double prior) {
    const int64_t kMax = 2147483646;
    int64_t N = n + 2, E = e + 1;
    if (N > kMax) { const double frac = (double) kMax / (double) N; E = (int64_t) std::floor((double) E * frac + 0.5); N = kMax; }
    double best = 0; int arg = 0;
    for (int Q = 0; Q <= 60; ++Q) {
        int d = std::abs((int) ((double) Q - prior));
        if (d > 40) d = 40;
        const double lp = std::log10(0.9 * std::exp(-(double) (d * d) / 0.5));
        const double l10p = (double) Q / -10.0, l10q = std::log10(1.0 - std::pow(10.0, l10p));
        double ll = (double) E * l10p + (double) (N - E) * l10q;
        if (!std::isfinite(ll)) ll = -DBL_MAX;
        const double v = lp + ll;
        if (Q == 0 || v > best) { best = v; arg = Q; }
    }
    return arg < 93 ? arg : 93;
}

// the read group covariate of a read group line: its PU, else its ID
inline std::string bqsr_read_group(const std::string &rg_line) {
    auto field = [&](const char *tag) {
        const size_t at = rg_line.find(std::string("\t") + tag);
        if (at == std::string::npos) return std::string();
        const size_t b = at + 4, e = rg_line.find_first_of("\t\n", b);
        return rg_line.substr(b, (e == std::string::npos ? rg_line.size() : e) - b);
    };
    const std::string pu = field("PU:");
    return pu.empty() ? field("ID:") : pu;
}

// one GATKReport table: cols are (name, format); rows hold the cells' text
struct BqsrTable {
    std::string name, desc;
    std::vector<std::pair<std::string, std::string>> cols;
    std::vector<std::vector<std::string>> rows;
    std::string text() const {
        std::string o = "#:GATKTable:" + std::to_string(cols.size()) + ":" + std::to_string(rows.size());
        for (const auto &c : cols) o += ":" + c.second;
        o += ":;\n#:GATKTable:" + name + ":" + desc + "\n";
        std::vector<size_t> w(cols.size());
        for (size_t c = 0; c < cols.size(); ++c) {
            w[c] = cols[c].first.size();
            for (const auto &r : rows) if (r[c].size() > w[c]) w[c] = r[c].size();
        }
        auto line = [&](const std::vector<std::string> &cells) {
            for (size_t c = 0; c < cols.size(); ++c) {
                const std::string pad(w[c] - cells[c].size(), ' ');
                if (c) o += "  ";
                o += cols[c].second == "%s" ? cells[c] + pad : pad + cells[c];
            }
            o += "\n";
        };
        std::vector<std::string> hdr;
        for (const auto &c : cols) hdr.push_back(c.first);
        line(hdr);
        for (const auto &r : rows) line(r);
        return o + "\n";
    }
};

inline std::string bqsr_fmt(const char *f, double v) { char b[64]; snprintf(b, sizeof b, f, v); return b; }

// the report of the dense tables: qual [94], ctx [94 * 16], cyc [94 * 1001], observations and errors
inline std::string bqsr_report_text(const std::string &rg, const int64_t *qo, const int64_t *qe, const int64_t *co, const int64_t *ce,
                                    const int64_t *yo, const int64_t *ye) {
    std::string o = "#:GATKReport.v1.1:5\n";
    BqsrTable a{"Arguments", "Recalibration argument collection values used in this run", {{"Argument", "%s"}, {"Value", "%s"}}, {}};
    static const char *const args[17][2] = {
        {"binary_tag_name", "null"}, {"covariate", "ReadGroupCovariate,QualityScoreCovariate,ContextCovariate,CycleCovariate"},
        {"default_platform", "null"}, {"deletions_default_quality", "45"}, {"force_platform", "null"}, {"indels_context_size", "3"},
        {"insertions_default_quality", "45"}, {"low_quality_tail", "2"}, {"maximum_cycle_value", "500"}, {"mismatches_context_size", "2"},
        {"mismatches_default_quality", "-1"}, {"no_standard_covs", "false"}, {"quantizing_levels", "16"}, {"recalibration_report", "null"},
        {"run_without_dbsnp", "false"}, {"solid_nocall_strategy", "THROW_EXCEPTION"}, {"solid_recal_mode", "SET_Q_ZERO"}};
    for (const auto &r : args) a.rows.push_back({r[0], r[1]});
    o += a.text();
    BqsrTable qz{"Quantized", "Quality quantization map", {{"QualityScore", "%d"}, {"Count", "%d"}, {"QuantizedScore", "%d"}}, {}};
    for (int q = 0; q < BQSR_NQ; ++q) qz.rows.push_back({std::to_string(q), std::to_string((long long) qo[q]), std::to_string(q)});
    o += qz.text();
    int64_t N = 0, E = 0; double s = 0;
    for (int q = 0; q < BQSR_NQ; ++q) { N += qo[q]; E += qe[q]; s += (double) qo[q] * std::pow(10.0, (double) q / -10.0); }
    BqsrTable t0{"RecalTable0", "", {{"ReadGroup", "%s"}, {"EventType", "%s"}, {"EmpiricalQuality", "%.4f"}, {"EstimatedQReported", "%.4f"},
                                     {"Observations", "%d"}, {"Errors", "%.2f"}}, {}};
    if (N > 0) {
        const double qr = -10.0 * std::log10(s / (double) N);
        t0.rows.push_back({rg, "M", bqsr_fmt("%.4f", bqsr_empirical_q(N, E, qr)), bqsr_fmt("%.4f", qr), std::to_string((long long) N),
                           bqsr_fmt("%.2f", (double) E)});
    }
    o += t0.text();
    BqsrTable t1{"RecalTable1", "", {{"ReadGroup", "%s"}, {"QualityScore", "%d"}, {"EventType", "%s"}, {"EmpiricalQuality", "%.4f"},
                                     {"Observations", "%d"}, {"Errors", "%.2f"}}, {}};
    BqsrTable t2{"RecalTable2", "", {{"ReadGroup", "%s"}, {"QualityScore", "%d"}, {"CovariateValue", "%s"}, {"CovariateName", "%s"},
                                     {"EventType", "%s"}, {"EmpiricalQuality", "%.4f"}, {"Observations", "%d"}, {"Errors", "%.2f"}}, {}};
    static const char L[] = "ACGT";
    for (int q = 0; q < BQSR_NQ; ++q) {
        if (qo[q]) t1.rows.push_back({rg, std::to_string(q), "M", bqsr_fmt("%.4f", bqsr_empirical_q(qo[q], qe[q], q)), std::to_string((long long) qo[q]),
                                      bqsr_fmt("%.2f", (double) qe[q])});
        for (int c = 0; c < BQSR_NCTX; ++c) {
            const int64_t n = co[q * BQSR_NCTX + c], e = ce[q * BQSR_NCTX + c];
            if (n) t2.rows.push_back({rg, std::to_string(q), std::string{L[c >> 2], L[c & 3]}, "Context", "M", bqsr_fmt("%.4f", bqsr_empirical_q(n, e, q)),
                                      std::to_string((long long) n), bqsr_fmt("%.2f", (double) e)});
        }
        for (int y = 0; y < BQSR_NCYC; ++y) {
            const int64_t n = yo[q * BQSR_NCYC + y], e = ye[q * BQSR_NCYC + y];
            if (n) t2.rows.push_back({rg, std::to_string(q), std::to_string(y - BQSR_MAX_CYCLE), "Cycle", "M", bqsr_fmt("%.4f", bqsr_empirical_q(n, e, q)),
                                      std::to_string((long long) n), bqsr_fmt("%.2f", (double) e)});
        }
    }
    return o + t1.text() + t2.text();
}

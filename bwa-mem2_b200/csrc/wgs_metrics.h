// wgs_metrics.h — the host side of bm2_wgsmetrics: the reference (<prefix>.ann and .amb only), the checks on the BAM header and record
// order, and Picard's WgsMetrics formulas and file text (the per-locus rule is wgs_device.cuh's; byte equality with Picard is not claimed).
//
//   reference  .ann: "l_pac n_seqs seed", then per contig "gi name[ anno]" and "offset len n_ambs"; .amb: "l_pac n_seqs n_holes", then
//              "offset len char" per hole.  The holes of N, n and . are the no-call loci; every hole is kept with its letter as well.
//   header     @HD must say SO:coordinate; the binary reference list must equal the .ann contigs in order, names and lengths
//              (wgs_check_refs, which bm2_multiplemetrics calls alone)
//   order      bam_coord_key never decreases from one record to the next
//   metrics    T = sum H[d], C = sum d H[d]; MEAN = C / T; SD = sqrt(sum H[d] (d - MEAN)^2 / (T - 1)); MEDIAN of the multiset of depths (even T:
//              the mean of the T/2-th and T/2+1-th smallest, odd T: the ceil(T/2)-th); MAD the same median over |d - MEDIAN|;
//              PCT_EXC_x = EXC_x / (the six exclusions + C), PCT_EXC_TOTAL = the six exclusions / that; PCT_kX = sum_{d >= k} H[d] / T.
//              A zero denominator gives 0.  HET_SNP_SENSITIVITY and HET_SNP_Q are empty: Picard draws them by Monte-Carlo sampling.
//   file       ## htsjdk.samtools.metrics.StringHeader, "# bm2_wgsmetrics <arguments>", a blank line, "## METRICS CLASS	picard.analysis.WgsMetrics",
//              the columns and one row, a blank line, "## HISTOGRAM	java.lang.Integer", "coverage	high_quality_coverage_count", rows 0..cap.
//              Doubles as dup_metrics_double prints them; no timestamp, so the file is deterministic.
#pragma once
#include "markdup_metrics.h"
#include "wgs_device.cuh"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <utility>
#include <vector>

struct WgsReference {
    int64_t l_pac = 0;
    std::vector<std::string> names;
    std::vector<int64_t> off;
    std::vector<int32_t> len;
    std::vector<int64_t> nocall;          // [beg, end) pairs, sorted
    std::vector<int64_t> holes;           // every hole as [beg, end) pairs, in .amb order
    std::vector<char> hole_char;          // each hole's letter
};

inline std::string wgs_read_reference(const std::string &prefix, WgsReference &r) {
    FILE *f = fopen((prefix + ".ann").c_str(), "r");
    if (!f) return "cannot open " + prefix + ".ann";
    long long l_pac = 0, seed = 0;
    int n = 0;
    if (fscanf(f, "%lld %d %lld", &l_pac, &n, &seed) != 3 || l_pac < 0 || n < 0) { fclose(f); return prefix + ".ann: a bad header line"; }
    r.l_pac = l_pac;
    for (int k = 0; k < n; ++k) {
        long long gi, o; int ln, nh;
        char name[8192];
        if (fscanf(f, "%lld %8191s", &gi, name) != 2) { fclose(f); return prefix + ".ann: a bad contig line"; }
        for (int c = fgetc(f); c != '\n' && c != EOF; c = fgetc(f)) {}
        if (fscanf(f, "%lld %d %d", &o, &ln, &nh) != 3 || o < 0 || ln < 0 || o + ln > l_pac) { fclose(f); return prefix + ".ann: a bad contig line"; }
        r.names.push_back(name); r.off.push_back(o); r.len.push_back(ln);
    }
    fclose(f);
    f = fopen((prefix + ".amb").c_str(), "r");
    if (!f) return "cannot open " + prefix + ".amb";
    long long a, b, nh;
    if (fscanf(f, "%lld %lld %lld", &a, &b, &nh) != 3 || a != l_pac || nh < 0) { fclose(f); return prefix + ".amb: a bad header line"; }
    for (long long h = 0; h < nh; ++h) {
        char c;
        if (fscanf(f, "%lld %lld %c", &a, &b, &c) != 3 || a < 0 || b < 0 || a + b > l_pac) { fclose(f); return prefix + ".amb: a bad hole line"; }
        r.holes.push_back(a); r.holes.push_back(a + b); r.hole_char.push_back(c);
        if (c != 'N' && c != 'n' && c != '.') continue;
        if (!r.nocall.empty() && a < r.nocall.back()) { fclose(f); return prefix + ".amb: the holes are not sorted"; }
        r.nocall.push_back(a); r.nocall.push_back(a + b);
    }
    fclose(f);
    return "";
}

// the header's reference list against the index: the first difference
inline std::string wgs_check_refs(const std::vector<std::pair<std::string, int32_t>> &refs, const WgsReference &r) {
    for (size_t k = 0; k < std::max(refs.size(), r.names.size()); ++k) {
        if (k >= refs.size()) return "the header has " + std::to_string(refs.size()) + " references, the index " + std::to_string(r.names.size()) + " contigs";
        if (k >= r.names.size()) return "the header has " + std::to_string(refs.size()) + " references, the index " + std::to_string(r.names.size()) + " contigs";
        if (refs[k].first != r.names[k] || refs[k].second != r.len[k])
            return "reference " + std::to_string(k) + " is " + refs[k].first + " of length " + std::to_string(refs[k].second) + " in the header, " +
                   r.names[k] + " of length " + std::to_string(r.len[k]) + " in the index";
    }
    return "";
}

// the header's sort order and reference list against the index
inline std::string wgs_check_header(const std::string &text, const std::vector<std::pair<std::string, int32_t>> &refs, const WgsReference &r) {
    std::string so;
    if (text.compare(0, 4, "@HD\t") == 0) {
        const size_t e = text.find('\n'), at = text.find("\tSO:");
        if (at != std::string::npos && at < e) so = text.substr(at + 4, std::min(text.find('\t', at + 4), e) - at - 4);
    }
    if (so != "coordinate") return "the input is not coordinate-sorted (@HD SO:" + (so.empty() ? std::string("<none>") : so) + ")";
    return wgs_check_refs(refs, r);
}

// the coordinate order, record by record; the error names the read
struct WgsOrder {
    uint64_t prev = 0;
    bool any = false;
    std::string check(const uint8_t *rec) {
        const BamFixed f = bam_fixed(rec);
        const uint64_t k = bam_coord_key(f.rid, f.pos, f.flag);
        if (any && k < prev) return "read " + std::string((const char *) rec + 36) + " is out of coordinate order";
        prev = k; any = true;
        return "";
    }
};

struct WgsCounts {
    std::vector<int64_t> hist;                // [cap + 1]
    int64_t exc[WGS_NEXC] = {0, 0, 0, 0, 0, 0};
};

// the median of a multiset given as (value, count) pairs sorted by value, with n = the sum of the counts
inline double wgs_median(const std::vector<std::pair<double, int64_t>> &v, int64_t n) {
    if (n <= 0) return 0;
    auto kth = [&](int64_t k) {                   // the k-th smallest, 1-based
        int64_t s = 0;
        for (const auto &p : v) { s += p.second; if (s >= k) return p.first; }
        return v.back().first;
    };
    return n % 2 ? kth((n + 1) / 2) : (kth(n / 2) + kth(n / 2 + 1)) / 2.0;
}

inline std::string wgs_metrics_text(const WgsCounts &x, const std::string &args) {
    const int cap = (int) x.hist.size() - 1;
    int64_t T = 0, C = 0;
    for (int d = 0; d <= cap; ++d) { T += x.hist[d]; C += (int64_t) d * x.hist[d]; }
    const double mean = T ? (double) C / (double) T : 0.0;
    double ss = 0;
    for (int d = 0; d <= cap; ++d) ss += (double) x.hist[d] * (((double) d - mean) * ((double) d - mean));
    const double sd = T > 1 ? std::sqrt(ss / (double) (T - 1)) : 0.0;
    std::vector<std::pair<double, int64_t>> v, dev;
    for (int d = 0; d <= cap; ++d) if (x.hist[d]) v.push_back({(double) d, x.hist[d]});
    const double median = wgs_median(v, T);
    for (const auto &p : v) dev.push_back({std::fabs(p.first - median), p.second});
    std::sort(dev.begin(), dev.end());
    const double mad = wgs_median(dev, T);
    int64_t excl = 0;
    for (int k = 0; k < WGS_NEXC; ++k) excl += x.exc[k];
    const int64_t den = excl + C;
    auto pct = [&](int64_t a, int64_t b) { return b ? (double) a / (double) b : 0.0; };
    static const int kX[] = {1, 5, 10, 15, 20, 25, 30, 40, 50, 60, 70, 80, 90, 100};
    std::string o = "## htsjdk.samtools.metrics.StringHeader\n# bm2_wgsmetrics" + (args.empty() ? std::string() : " " + args) + "\n\n";
    o += "## METRICS CLASS\tpicard.analysis.WgsMetrics\n";
    o += "GENOME_TERRITORY\tMEAN_COVERAGE\tSD_COVERAGE\tMEDIAN_COVERAGE\tMAD_COVERAGE\tPCT_EXC_MAPQ\tPCT_EXC_DUPE\tPCT_EXC_UNPAIRED\tPCT_EXC_BASEQ\t"
         "PCT_EXC_OVERLAP\tPCT_EXC_CAPPED\tPCT_EXC_TOTAL";
    for (int k : kX) o += "\tPCT_" + std::to_string(k) + "X";
    o += "\tHET_SNP_SENSITIVITY\tHET_SNP_Q\n";
    o += std::to_string(T);
    for (double d : {mean, sd, median, mad}) o += "\t" + dup_metrics_double(d);
    for (int k = 0; k < WGS_NEXC; ++k) o += "\t" + dup_metrics_double(pct(x.exc[k], den));
    o += "\t" + dup_metrics_double(pct(excl, den));
    for (int k : kX) {
        int64_t s = 0;
        for (int d = k; d <= cap; ++d) s += x.hist[d];
        o += "\t" + dup_metrics_double(pct(s, T));
    }
    o += "\t\t\n\n## HISTOGRAM\tjava.lang.Integer\ncoverage\thigh_quality_coverage_count\n";
    for (int d = 0; d <= cap; ++d) o += std::to_string(d) + "\t" + std::to_string(x.hist[d]) + "\n";
    return o;
}

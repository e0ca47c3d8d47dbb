// mm_metrics.h — the host side of bm2_multiplemetrics: the reference (<prefix>.ann, .amb and .pac), the default adapters, and Picard's
// AlignmentSummaryMetrics and InsertSizeMetrics formulas and file text (the per-record rule is mm_device.cuh's; byte equality with Picard is
// not claimed).
//
//   reference  wgs_read_reference's contigs and holes (sorted and disjoint), and the .pac: (l_pac + 3) / 4 packed bytes, a 0 byte when
//              l_pac % 4 == 0, then l_pac % 4 (fasta_pack.cpp's layout)
//   histogram  htsjdk's Histogram rules over (key, count): MEAN = sum k c / n; SD = sqrt(sum c (k - MEAN)^2 / (n - 1)); MEDIAN and MAD as
//              wgs_median; MODE the smallest of the keys with the largest count.  n <= 1 gives SD 0, n = 0 gives 0 everywhere.
//   summary    rows FIRST_OF_PAIR, SECOND_OF_PAIR and PAIR (their sums) when a first-of-pair read was counted; UNPAIRED when an unpaired
//              read was, or no first-of-pair read; ratios as mm_summary_row states them; a zero denominator gives 0.  BAD_CYCLES: the
//              cycles whose no-calls / TOTAL_READS >= 0.8 (PAIR: the first and second rows' sum).
//   insert     the orientations (FR, RF, TANDEM) with at least 5 % of all pairs; per orientation, on its histogram: READ_PAIRS, MIN, MAX,
//              MEDIAN, MODE, MAD and the widths by Picard's loop (mm_insert_row); then trimmed to keys <= (int) (MEDIAN + 10 MAD): MEAN and
//              SD.  The file's histogram is the trimmed one, one row per key of the reported orientations' union.
//   file       ## htsjdk.samtools.metrics.StringHeader, "# bm2_multiplemetrics <arguments>", a blank line, "## METRICS CLASS	<class>", the
//              columns and the rows; for insert sizes a blank line, "## HISTOGRAM	java.lang.Integer" and the histogram.  Doubles as
//              dup_metrics_double prints them; no timestamp.
#pragma once
#include "markdup_metrics.h"
#include "mm_device.cuh"
#include "wgs_metrics.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <map>
#include <string>
#include <utility>
#include <vector>

// Picard's default ADAPTER_SEQUENCE: the 5' and 3' adapters of IlluminaUtil.IlluminaAdapterPair SINGLE_END, PAIRED_END and INDEXED.
// Restated from Picard's public source, not checked against Picard here.  Only the first 16 bases take part.
inline const char *const kMmAdapters[6] = {
    "AATGATACGGCGACCACCGACAGGTTCAGAGTTCTACAGTCCGACGATC",                     // SINGLE_END 5'
    "AGATCGGAAGAGCTCGTATGCCGTCTTCTGCTTG",                                    // SINGLE_END 3'
    "AATGATACGGCGACCACCGAGATCTACACTCTTTCCCTACACGACGCTCTTCCGATCT",            // PAIRED_END 5'
    "AGATCGGAAGAGCGGTTCAGCAGGAATGCCGAGACCGATCTCGTATGCCGTCTTCTGCTTG",         // PAIRED_END 3'
    "AATGATACGGCGACCACCGAGATCTACACTCTTTCCCTACACGACGCTCTTCCGATCT",            // INDEXED 5'
    "AGATCGGAAGAGCACACGTCTGAACTCCAGTCACNNNNNNNNATCTCGTATGCCGTCTTCTGCTTG",    // INDEXED 3'
};

// the kmers the adapter test compares with: each adapter's first 16 bases, then their reverse complement
inline void mm_adapter_kmers(char out[MM_N_ADAPTER_KMERS][MM_ADAPTER_LEN]) {
    for (int a = 0; a < 6; ++a)
        for (int k = 0; k < MM_ADAPTER_LEN; ++k) {
            const char c = kMmAdapters[a][k];
            out[2 * a][k] = c;
            out[2 * a + 1][MM_ADAPTER_LEN - 1 - k] = c == 'A' ? 'T' : c == 'C' ? 'G' : c == 'G' ? 'C' : c == 'T' ? 'A' : c;
        }
}

struct MmReference : WgsReference {
    std::vector<uint8_t> pac;                 // (l_pac + 3) / 4 bytes
};

inline std::string mm_read_reference(const std::string &prefix, MmReference &r) {
    std::string e = wgs_read_reference(prefix, r);
    if (!e.empty()) return e;
    for (size_t h = 1; h < r.hole_char.size(); ++h)
        if (r.holes[2 * h] < r.holes[2 * h - 1]) return prefix + ".amb: the holes are not sorted";
    FILE *f = fopen((prefix + ".pac").c_str(), "rb");
    if (!f) return "cannot open " + prefix + ".pac";
    const int64_t packed = (r.l_pac + 3) / 4, want = packed + (r.l_pac % 4 == 0 ? 1 : 0) + 1;
    std::vector<uint8_t> all;
    uint8_t buf[1 << 16];
    for (size_t k; (k = fread(buf, 1, sizeof buf, f)) > 0;) {
        all.insert(all.end(), buf, buf + k);
        if ((int64_t) all.size() > want) break;
    }
    const bool bad = ferror(f) != 0;
    fclose(f);
    if (bad) return "cannot read " + prefix + ".pac";
    if ((int64_t) all.size() != want || all.back() != (uint8_t) (r.l_pac % 4))
        return prefix + ".pac: its size does not fit the " + std::to_string(r.l_pac) + " bases of " + prefix + ".ann";
    all.resize((size_t) packed);
    r.pac.swap(all);
    return "";
}

// the counters and histograms of bm2_mm_finish, on the host
struct MmCounts {
    int64_t c[MM_NCAT][MM_NCOUNT] = {};
    std::vector<int64_t> len[MM_NCAT], mism[MM_NCAT], nocall[MM_NCAT];   // by l_seq, by mismatch count, by cycle
    std::map<int64_t, int64_t> ins[MM_NORIENT];                           // insert size -> pairs
};

// from bm2_mm_result_t's arrays (max_len + 1 per category; insert bins max_insert + 1 per orientation; big as orientation << 32 | size)
inline MmCounts mm_counts(const int64_t (*counts)[MM_NCOUNT], int32_t max_len, const int64_t *len, const int64_t *mism, const int64_t *nocall,
                          int32_t max_insert, const int64_t *ins, const uint64_t *big, int64_t n_big) {
    MmCounts x;
    const size_t L = (size_t) max_len + 1;
    for (int c = 0; c < MM_NCAT; ++c) {
        for (int k = 0; k < MM_NCOUNT; ++k) x.c[c][k] = counts[c][k];
        x.len[c].assign(len + c * L, len + (c + 1) * L);
        x.mism[c].assign(mism + c * L, mism + (c + 1) * L);
        x.nocall[c].assign(nocall + c * L, nocall + (c + 1) * L);
    }
    for (int o = 0; o < MM_NORIENT; ++o)
        for (int32_t k = 0; k <= max_insert; ++k)
            if (ins[(size_t) o * ((size_t) max_insert + 1) + (size_t) k]) x.ins[o][k] = ins[(size_t) o * ((size_t) max_insert + 1) + (size_t) k];
    for (int64_t i = 0; i < n_big; ++i) x.ins[big[i] >> 32][(int64_t) (big[i] & 0xFFFFFFFFu)] += 1;
    return x;
}

// htsjdk's Histogram statistics of (key, count) pairs sorted by key
struct MmHist {
    int64_t n = 0;
    double mean = 0, sd = 0, median = 0, mad = 0, mode = 0;
    int64_t min = 0, max = 0;
};
inline MmHist mm_hist(const std::vector<std::pair<int64_t, int64_t>> &v) {
    MmHist h;
    double s = 0;
    int64_t best = 0;
    for (const auto &p : v) {
        h.n += p.second; s += (double) p.first * (double) p.second;
        if (p.second > best) { best = p.second; h.mode = (double) p.first; }
    }
    if (!h.n) return h;
    h.min = v.front().first; h.max = v.back().first;
    h.mean = s / (double) h.n;
    double ss = 0;
    for (const auto &p : v) ss += (double) p.second * (((double) p.first - h.mean) * ((double) p.first - h.mean));
    h.sd = h.n > 1 ? std::sqrt(ss / (double) (h.n - 1)) : 0.0;
    std::vector<std::pair<double, int64_t>> d, dev;
    for (const auto &p : v) d.push_back({(double) p.first, p.second});
    h.median = wgs_median(d, h.n);
    for (const auto &p : d) dev.push_back({std::fabs(p.first - h.median), p.second});
    std::sort(dev.begin(), dev.end());
    h.mad = wgs_median(dev, h.n);
    return h;
}

inline std::vector<std::pair<int64_t, int64_t>> mm_nonzero(const std::vector<int64_t> &a) {
    std::vector<std::pair<int64_t, int64_t>> v;
    for (size_t k = 0; k < a.size(); ++k) if (a[k]) v.push_back({(int64_t) k, a[k]});
    return v;
}

inline int64_t mm_bad_cycles(const std::vector<int64_t> &nocall, int64_t total) {
    int64_t n = 0;
    for (int64_t v : nocall) n += total > 0 && (double) v / (double) total >= 0.8;
    return n;
}

inline std::string mm_header(const std::string &args, const char *cls) {
    return "## htsjdk.samtools.metrics.StringHeader\n# bm2_multiplemetrics" + (args.empty() ? std::string() : " " + args) + "\n\n## METRICS CLASS\t" +
           cls + "\n";
}

// one AlignmentSummaryMetrics row from a category's counters, histograms and BAD_CYCLES
inline std::string mm_summary_row(const char *name, const int64_t *c, const std::vector<int64_t> &len, const std::vector<int64_t> &mism,
                                  int64_t bad_cycles) {
    auto r = [](int64_t a, int64_t b) { return dup_metrics_double(b ? (double) a / (double) b : 0.0); };
    const MmHist L = mm_hist(mm_nonzero(len)), M = mm_hist(mm_nonzero(mism));
    std::string o = name;
    auto i = [&](int64_t v) { o += "\t" + std::to_string(v); };
    auto d = [&](const std::string &v) { o += "\t" + v; };
    i(c[MM_TOTAL]); i(c[MM_PF]); d(r(c[MM_PF], c[MM_TOTAL])); i(c[MM_NOISE]); i(c[MM_ALIGNED]); d(r(c[MM_ALIGNED], c[MM_PF]));
    i(c[MM_ALIGNED_BASES]); i(c[MM_HQ_READS]); i(c[MM_HQ_BASES]); i(c[MM_HQ_Q20]); d(dup_metrics_double(M.median));
    d(r(c[MM_MISMATCH], c[MM_ALIGNED_BASES])); d(r(c[MM_HQ_MISMATCH], c[MM_HQ_BASES])); d(r(c[MM_INDELS], c[MM_ALIGNED_BASES]));
    d(dup_metrics_double(L.mean)); d(dup_metrics_double(L.sd)); d(dup_metrics_double(L.median)); d(dup_metrics_double(L.mad)); i(L.min); i(L.max);
    i(c[MM_IN_PAIRS]); d(r(c[MM_IN_PAIRS], c[MM_ALIGNED])); i(c[MM_IMPROPER]); d(r(c[MM_IMPROPER], c[MM_ALIGNED])); i(bad_cycles);
    d(r(c[MM_FORWARD], c[MM_ALIGNED])); d(r(c[MM_CHIM], c[MM_CHIM_DEN])); d(r(c[MM_ADAPTER], c[MM_PF])); d(r(c[MM_SOFTCLIP], c[MM_ALIGNED_BASES]));
    d(r(c[MM_HARDCLIP], c[MM_ALIGNED_BASES])); d(r(c[MM_SC3_SUM], c[MM_SC3_READS]));
    return o + "\t\t\t\n";
}

inline std::string mm_summary_text(const MmCounts &x, const std::string &args) {
    std::string o = mm_header(args, "picard.analysis.AlignmentSummaryMetrics");
    o += "CATEGORY\tTOTAL_READS\tPF_READS\tPCT_PF_READS\tPF_NOISE_READS\tPF_READS_ALIGNED\tPCT_PF_READS_ALIGNED\tPF_ALIGNED_BASES\t"
         "PF_HQ_ALIGNED_READS\tPF_HQ_ALIGNED_BASES\tPF_HQ_ALIGNED_Q20_BASES\tPF_HQ_MEDIAN_MISMATCHES\tPF_MISMATCH_RATE\tPF_HQ_ERROR_RATE\t"
         "PF_INDEL_RATE\tMEAN_READ_LENGTH\tSD_READ_LENGTH\tMEDIAN_READ_LENGTH\tMAD_READ_LENGTH\tMIN_READ_LENGTH\tMAX_READ_LENGTH\t"
         "READS_ALIGNED_IN_PAIRS\tPCT_READS_ALIGNED_IN_PAIRS\tPF_READS_IMPROPER_PAIRS\tPCT_PF_READS_IMPROPER_PAIRS\tBAD_CYCLES\tSTRAND_BALANCE\t"
         "PCT_CHIMERAS\tPCT_ADAPTER\tPCT_SOFTCLIP\tPCT_HARDCLIP\tAVG_POS_3PRIME_SOFTCLIP_LENGTH\tSAMPLE\tLIBRARY\tREAD_GROUP\n";
    const bool paired = x.c[MM_FIRST][MM_TOTAL] > 0;
    if (paired) {
        const int64_t b0 = mm_bad_cycles(x.nocall[MM_FIRST], x.c[MM_FIRST][MM_TOTAL]);
        const int64_t b1 = mm_bad_cycles(x.nocall[MM_SECOND], x.c[MM_SECOND][MM_TOTAL]);
        o += mm_summary_row("FIRST_OF_PAIR", x.c[MM_FIRST], x.len[MM_FIRST], x.mism[MM_FIRST], b0);
        o += mm_summary_row("SECOND_OF_PAIR", x.c[MM_SECOND], x.len[MM_SECOND], x.mism[MM_SECOND], b1);
        int64_t c[MM_NCOUNT];
        for (int k = 0; k < MM_NCOUNT; ++k) c[k] = x.c[MM_FIRST][k] + x.c[MM_SECOND][k];
        auto sum = [](const std::vector<int64_t> &a, const std::vector<int64_t> &b) {
            std::vector<int64_t> s(std::max(a.size(), b.size()), 0);
            for (size_t k = 0; k < a.size(); ++k) s[k] += a[k];
            for (size_t k = 0; k < b.size(); ++k) s[k] += b[k];
            return s;
        };
        o += mm_summary_row("PAIR", c, sum(x.len[MM_FIRST], x.len[MM_SECOND]), sum(x.mism[MM_FIRST], x.mism[MM_SECOND]), b0 + b1);
    }
    if (x.c[MM_UNPAIRED][MM_TOTAL] > 0 || !paired)
        o += mm_summary_row("UNPAIRED", x.c[MM_UNPAIRED], x.len[MM_UNPAIRED], x.mism[MM_UNPAIRED],
                            mm_bad_cycles(x.nocall[MM_UNPAIRED], x.c[MM_UNPAIRED][MM_TOTAL]));
    return o;
}

// one InsertSizeMetrics row of an orientation's histogram; trimmed receives the histogram trimmed to (int) (MEDIAN + 10 MAD)
inline std::string mm_insert_row(const char *orient, const std::map<int64_t, int64_t> &h, std::map<int64_t, int64_t> &trimmed) {
    const std::vector<std::pair<int64_t, int64_t>> v(h.begin(), h.end());
    const MmHist s = mm_hist(v);
    static const double kPct[] = {0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 0.95, 0.99};
    int64_t width[11] = {};
    double low = s.median, high = s.median, covered = 0;
    while (low >= (double) s.min || high <= (double) s.max) {
        auto at = [&](double k) { const auto it = h.find((int64_t) k); return it == h.end() ? 0.0 : (double) it->second; };
        covered += at(low);
        if (low != high) covered += at(high);
        const double pct = covered / (double) s.n;
        const int64_t distance = (int64_t) (high - low) + 1;
        for (int k = 0; k < 11; ++k) if (pct >= kPct[k] && width[k] == 0) width[k] = distance;
        --low; ++high;
    }
    const int64_t top = (int64_t) (s.median + 10 * s.mad);
    std::vector<std::pair<int64_t, int64_t>> tv;
    for (const auto &p : v) if (p.first <= top) { tv.push_back(p); trimmed[p.first] = p.second; }
    const MmHist t = mm_hist(tv);
    std::string o = dup_metrics_double(s.median) + "\t" + dup_metrics_double(s.mode) + "\t" + dup_metrics_double(s.mad) + "\t" + std::to_string(s.min) +
                    "\t" + std::to_string(s.max) + "\t" + dup_metrics_double(t.mean) + "\t" + dup_metrics_double(t.sd) + "\t" + std::to_string(s.n) +
                    "\t" + orient;
    for (int64_t w : width) o += "\t" + std::to_string(w);
    return o + "\t\t\t\n";
}

// the insert size file; pairs receives the number of pairs counted
inline std::string mm_insert_text(const MmCounts &x, const std::string &args, int64_t *pairs) {
    static const char *const kOrient[3] = {"FR", "RF", "TANDEM"}, *const kCol[3] = {"fr", "rf", "tandem"};
    std::string o = mm_header(args, "picard.analysis.InsertSizeMetrics");
    o += "MEDIAN_INSERT_SIZE\tMODE_INSERT_SIZE\tMEDIAN_ABSOLUTE_DEVIATION\tMIN_INSERT_SIZE\tMAX_INSERT_SIZE\tMEAN_INSERT_SIZE\tSTANDARD_DEVIATION\t"
         "READ_PAIRS\tPAIR_ORIENTATION\tWIDTH_OF_10_PERCENT\tWIDTH_OF_20_PERCENT\tWIDTH_OF_30_PERCENT\tWIDTH_OF_40_PERCENT\tWIDTH_OF_50_PERCENT\t"
         "WIDTH_OF_60_PERCENT\tWIDTH_OF_70_PERCENT\tWIDTH_OF_80_PERCENT\tWIDTH_OF_90_PERCENT\tWIDTH_OF_95_PERCENT\tWIDTH_OF_99_PERCENT\tSAMPLE\t"
         "LIBRARY\tREAD_GROUP\n";
    int64_t n[3] = {0, 0, 0}, total = 0;
    for (int k = 0; k < 3; ++k) { for (const auto &p : x.ins[k]) n[k] += p.second; total += n[k]; }
    *pairs = total;
    if (!total) return o;
    std::vector<int> shown;
    std::map<int64_t, int64_t> trimmed[3];
    for (int k = 0; k < 3; ++k)
        if ((double) n[k] / (double) total >= 0.05) { shown.push_back(k); o += mm_insert_row(kOrient[k], x.ins[k], trimmed[k]); }
    o += "\n## HISTOGRAM\tjava.lang.Integer\ninsert_size";
    std::map<int64_t, int> keys;
    for (int k : shown) { o += std::string("\tAll_Reads.") + kCol[k] + "_count"; for (const auto &p : trimmed[k]) keys[p.first] = 1; }
    o += "\n";
    for (const auto &kv : keys) {
        o += std::to_string(kv.first);
        for (int k : shown) { const auto it = trimmed[k].find(kv.first); o += "\t" + std::to_string(it == trimmed[k].end() ? 0 : it->second); }
        o += "\n";
    }
    return o;
}

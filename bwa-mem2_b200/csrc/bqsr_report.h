// bqsr_report.h — the host side of bm2_mem --recal-file: the empirical quality of a table row and the recalibration report's text, from the
// dense tables of bm2_bqsr_tables; and of bm2_applybqsr: the report parsed back into the dense tables the apply kernel reads.  Restated in
// Python in tests/bqsr_util.py and tests/applybqsr_util.py.
//
//   empirical quality   GATK's RecalDatum.bayesianEstimateOfEmpiricalQuality: with N = n + 2 observations and E = e + 1 errors (N above
//                       2^31 - 2: both scaled down to N = 2^31 - 2, E rounded half up), the argmax, lowest first, over Q = 0..60 of
//                       log10(0.9 exp(-d^2 / 0.5)), d = min(|(int) (Q - prior)|, 40), plus the binomial log10-likelihood of E errors in N at
//                       the error rate 10^(-Q/10) (an infinite or NaN likelihood counts as -DBL_MAX), capped at 93.  The binomial coefficient
//                       is the same for every Q, so it is left out: the argmax does not change.
//   report              GATKReport v1.1: Arguments (GATK 4's defaults), Quantized (qualities 0..93 mapped to themselves), RecalTable0 (the
//                       read group), RecalTable1 (quality), RecalTable2 (quality and context, then quality and cycle), event M only, the
//                       rows with at least one observation.  Several read group covariates: each one's rows in turn, in the order given.  Each cell is padded to its column's widest, strings left, numbers right, two
//                       spaces apart.  No timestamp.
#pragma once
#include "bqsr_device.cuh"
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
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

// the value of a header line's tag ("ID:"), empty without it
inline std::string bqsr_rg_tag(const std::string &line, const char *tag) {
    const size_t at = line.find(std::string("\t") + tag);
    if (at == std::string::npos) return std::string();
    const size_t b = at + 4, e = line.find_first_of("\t\n", b);
    return line.substr(b, (e == std::string::npos ? line.size() : e) - b);
}

// the read group covariate of a read group line: its PU, else its ID
inline std::string bqsr_read_group(const std::string &rg_line) {
    const std::string pu = bqsr_rg_tag(rg_line, "PU:");
    return pu.empty() ? bqsr_rg_tag(rg_line, "ID:") : pu;
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

// one covariate's dense tables: qual [94], ctx [94 * 16], cyc [94 * 1001], observations and errors
struct BqsrCovTables {
    std::string rg;
    const int64_t *qo, *qe, *co, *ce, *yo, *ye;
};

// the report of several covariates (bm2_baserecalibrator, in the byte order of their strings): RecalTable0 one row per covariate,
// RecalTable1 and RecalTable2 the rows of each covariate in turn, the Quantized table's Count summed over them
inline std::string bqsr_report_text(const std::vector<BqsrCovTables> &covs) {
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
    for (int q = 0; q < BQSR_NQ; ++q) {
        int64_t n = 0;
        for (const BqsrCovTables &c : covs) n += c.qo[q];
        qz.rows.push_back({std::to_string(q), std::to_string((long long) n), std::to_string(q)});
    }
    o += qz.text();
    BqsrTable t0{"RecalTable0", "", {{"ReadGroup", "%s"}, {"EventType", "%s"}, {"EmpiricalQuality", "%.4f"}, {"EstimatedQReported", "%.4f"},
                                     {"Observations", "%d"}, {"Errors", "%.2f"}}, {}};
    BqsrTable t1{"RecalTable1", "", {{"ReadGroup", "%s"}, {"QualityScore", "%d"}, {"EventType", "%s"}, {"EmpiricalQuality", "%.4f"},
                                     {"Observations", "%d"}, {"Errors", "%.2f"}}, {}};
    BqsrTable t2{"RecalTable2", "", {{"ReadGroup", "%s"}, {"QualityScore", "%d"}, {"CovariateValue", "%s"}, {"CovariateName", "%s"},
                                     {"EventType", "%s"}, {"EmpiricalQuality", "%.4f"}, {"Observations", "%d"}, {"Errors", "%.2f"}}, {}};
    static const char L[] = "ACGT";
    for (const BqsrCovTables &c : covs) {
        const std::string &rg = c.rg;
        int64_t N = 0, E = 0; double s = 0;
        for (int q = 0; q < BQSR_NQ; ++q) { N += c.qo[q]; E += c.qe[q]; s += (double) c.qo[q] * std::pow(10.0, (double) q / -10.0); }
        if (N > 0) {
            const double qr = -10.0 * std::log10(s / (double) N);
            t0.rows.push_back({rg, "M", bqsr_fmt("%.4f", bqsr_empirical_q(N, E, qr)), bqsr_fmt("%.4f", qr), std::to_string((long long) N),
                               bqsr_fmt("%.2f", (double) E)});
        }
        for (int q = 0; q < BQSR_NQ; ++q) {
            if (c.qo[q]) t1.rows.push_back({rg, std::to_string(q), "M", bqsr_fmt("%.4f", bqsr_empirical_q(c.qo[q], c.qe[q], q)),
                                            std::to_string((long long) c.qo[q]), bqsr_fmt("%.2f", (double) c.qe[q])});
            for (int x = 0; x < BQSR_NCTX; ++x) {
                const int64_t n = c.co[q * BQSR_NCTX + x], e = c.ce[q * BQSR_NCTX + x];
                if (n) t2.rows.push_back({rg, std::to_string(q), std::string{L[x >> 2], L[x & 3]}, "Context", "M", bqsr_fmt("%.4f", bqsr_empirical_q(n, e, q)),
                                          std::to_string((long long) n), bqsr_fmt("%.2f", (double) e)});
            }
            for (int y = 0; y < BQSR_NCYC; ++y) {
                const int64_t n = c.yo[q * BQSR_NCYC + y], e = c.ye[q * BQSR_NCYC + y];
                if (n) t2.rows.push_back({rg, std::to_string(q), std::to_string(y - BQSR_MAX_CYCLE), "Cycle", "M", bqsr_fmt("%.4f", bqsr_empirical_q(n, e, q)),
                                          std::to_string((long long) n), bqsr_fmt("%.2f", (double) e)});
            }
        }
    }
    return o + t0.text() + t1.text() + t2.text();
}

// the report of one covariate's dense tables (bm2_mem --recal-file)
inline std::string bqsr_report_text(const std::string &rg, const int64_t *qo, const int64_t *qe, const int64_t *co, const int64_t *ce,
                                    const int64_t *yo, const int64_t *ye) {
    return bqsr_report_text(std::vector<BqsrCovTables>{{rg, qo, qe, co, ce, yo, ye}});
}

// ---- the apply side (bm2_applybqsr): a GATKReport v1.1 recalibration table read back into the dense tables of bqsr_device.cuh's rule ----
//   parse    the tables by name (Arguments, RecalTable0, RecalTable1, RecalTable2; any other is skipped), the columns by their header names,
//            the cells split on runs of spaces; rows with EventType M only.  Arguments must hold covariate = ReadGroupCovariate,
//            QualityScoreCovariate,ContextCovariate,CycleCovariate, mismatches_context_size 2, low_quality_tail 2 and maximum_cycle_value 500,
//            the keys the kernel is fixed to.  A missing table, column or argument, a quality outside 0..93, a context that is not two of
//            ACGT, a cycle outside +-1..500, a number that does not parse or a repeated row is an error naming the file and the line.  Rows of
//            a read group without a RecalTable0 row are ignored: such reads are written unchanged.  The Quantized table is not read (no
//            quantization).
//   deltas   per read group r (EQ(n, e, prior) = bqsr_empirical_q(n, (int64) (e + 0.5), prior), n the Observations, e the Errors as double):
//            E its RecalTable0 EstimatedQReported, G = EQ(row r, E) - E, D_q = EQ(row (r, q), E + G) - (E + G), P = (E + G) + D_q,
//            D_ctx = EQ(row (r, q, ctx), P) - P, D_cyc = EQ(row (r, q, cyc), P) - P, each 0.0 without its row; IEEE double in this order
struct BqsrApplyTables {
    std::vector<std::string> rgs;          // the read group covariates with a RecalTable0 row, in table order
    std::vector<double> P, ctx, cyc;       // per read group: [94], [94 * 16], [94 * 1001]
};

inline std::string bqsr_parse_report(const std::string &text, const std::string &path, BqsrApplyTables &out) {
    struct Tab { int line = 0; std::vector<std::string> cols; std::vector<std::pair<int, std::vector<std::string>>> rows; };
    std::map<std::string, Tab> tabs;
    std::vector<std::string> lines;
    for (size_t b = 0; b <= text.size();) {
        size_t e = text.find('\n', b);
        if (e == std::string::npos) e = text.size();
        std::string l = text.substr(b, e - b);
        if (!l.empty() && l.back() == '\r') l.pop_back();
        lines.push_back(l);
        b = e + 1;
    }
    auto err = [&](int line, const std::string &m) { return path + ":" + std::to_string(line) + ": " + m; };
    auto cells = [](const std::string &l) {
        std::vector<std::string> v;
        for (size_t b = 0;;) {
            b = l.find_first_not_of(' ', b);
            if (b == std::string::npos) break;
            const size_t e = l.find(' ', b);
            v.push_back(l.substr(b, e == std::string::npos ? e : e - b));
            if (e == std::string::npos) break;
            b = e;
        }
        return v;
    };
    if (lines.empty() || lines[0].compare(0, 18, "#:GATKReport.v1.1:") != 0) return err(1, "not a GATKReport v1.1 file");
    for (size_t i = 1; i < lines.size(); ++i) {
        if (lines[i].compare(0, 12, "#:GATKTable:") != 0) continue;
        const int at = (int) i + 1;
        long long nc = 0, nr = 0;
        if (sscanf(lines[i].c_str() + 12, "%lld:%lld", &nc, &nr) != 2 || nc < 1 || nr < 0) return err(at, "a table's format line does not parse");
        if (i + 2 >= lines.size() || lines[i + 1].compare(0, 12, "#:GATKTable:") != 0) return err(at + 1, "a table without its name line");
        const std::string name = lines[i + 1].substr(12, lines[i + 1].find(':', 12) == std::string::npos ? std::string::npos : lines[i + 1].find(':', 12) - 12);
        Tab t;
        t.line = at + 2;
        t.cols = cells(lines[i + 2]);
        if ((long long) t.cols.size() != nc) return err(at + 2, "the header has " + std::to_string(t.cols.size()) + " columns, the table " + std::to_string(nc));
        for (long long r = 0; r < nr; ++r) {
            const size_t k = i + 3 + (size_t) r;
            if (k >= lines.size()) return err((int) lines.size(), "table " + name + " ends before its " + std::to_string(nr) + " rows");
            std::vector<std::string> c = cells(lines[k]);
            if ((long long) c.size() != nc) return err((int) k + 1, "a row of " + std::to_string(c.size()) + " cells, the header has " + std::to_string(nc));
            t.rows.push_back({(int) k + 1, std::move(c)});
        }
        if (!tabs.count(name)) tabs[name] = std::move(t);
        i += 2 + (size_t) nr;
    }
    const int last = (int) lines.size();
    for (const char *n : {"Arguments", "RecalTable0", "RecalTable1", "RecalTable2"})
        if (!tabs.count(n)) return err(last, std::string("no table ") + n);
    auto col = [&](const Tab &t, const char *tab, const char *c, int &k) -> std::string {
        for (k = 0; k < (int) t.cols.size(); ++k) if (t.cols[(size_t) k] == c) return "";
        return err(t.line, std::string("table ") + tab + " has no column " + c);
    };
    std::string e;
    {   // the arguments the kernel's keys are fixed to
        const Tab &a = tabs["Arguments"];
        int ka, kv;
        if (!(e = col(a, "Arguments", "Argument", ka)).empty() || !(e = col(a, "Arguments", "Value", kv)).empty()) return e;
        static const char *const want[4][2] = {{"covariate", "ReadGroupCovariate,QualityScoreCovariate,ContextCovariate,CycleCovariate"},
                                               {"mismatches_context_size", "2"}, {"low_quality_tail", "2"}, {"maximum_cycle_value", "500"}};
        for (const auto &w : want) {
            bool found = false;
            for (const auto &r : a.rows)
                if (r.second[(size_t) ka] == w[0]) {
                    found = true;
                    if (r.second[(size_t) kv] != w[1]) return err(r.first, std::string("argument ") + w[0] + " is " + r.second[(size_t) kv] + ", not " + w[1]);
                }
            if (!found) return err(a.line, std::string("no argument ") + w[0]);
        }
    }
    auto num = [](const std::string &s, double &v) { char *x; v = strtod(s.c_str(), &x); return !s.empty() && !*x && std::isfinite(v) && v >= 0; };
    auto obs = [](const std::string &s, int64_t &v) { char *x; v = strtoll(s.c_str(), &x, 10); return !s.empty() && !*x && v >= 0; };
    struct Row { bool has = false; int64_t n = 0; double e = 0; };
    struct Rg { double E = 0; Row r; std::vector<Row> q, c, y; };
    std::map<std::string, size_t> rg_of;
    std::vector<Rg> rgs;
    {
        const Tab &t = tabs["RecalTable0"];
        int kr, ke, kq, kn, kx;
        if (!(e = col(t, "RecalTable0", "ReadGroup", kr)).empty() || !(e = col(t, "RecalTable0", "EventType", ke)).empty() ||
            !(e = col(t, "RecalTable0", "EstimatedQReported", kq)).empty() || !(e = col(t, "RecalTable0", "Observations", kn)).empty() ||
            !(e = col(t, "RecalTable0", "Errors", kx)).empty()) return e;
        for (const auto &r : t.rows) {
            const std::vector<std::string> &c = r.second;
            if (c[(size_t) ke] != "M") continue;
            if (rg_of.count(c[(size_t) kr])) return err(r.first, "a second row of read group " + c[(size_t) kr]);
            Rg g;
            if (!num(c[(size_t) kq], g.E) || !obs(c[(size_t) kn], g.r.n) || !num(c[(size_t) kx], g.r.e)) return err(r.first, "a number does not parse");
            g.r.has = true;
            g.q.resize(BQSR_NQ); g.c.resize(BQSR_NQ * BQSR_NCTX); g.y.resize(BQSR_NQ * BQSR_NCYC);
            rg_of[c[(size_t) kr]] = rgs.size();
            out.rgs.push_back(c[(size_t) kr]);
            rgs.push_back(std::move(g));
        }
    }
    auto qual = [](const std::string &s, int &q) { char *x; const long v = strtol(s.c_str(), &x, 10); q = (int) v; return !s.empty() && !*x && v >= 0 && v < BQSR_NQ; };
    auto put = [&](Row &w, int line, const std::string &n, const std::string &x) -> std::string {
        if (w.has) return err(line, "a repeated row");
        if (!obs(n, w.n) || !num(x, w.e)) return err(line, "a number does not parse");
        w.has = true;
        return "";
    };
    {
        const Tab &t = tabs["RecalTable1"];
        int kr, kq, ke, kn, kx;
        if (!(e = col(t, "RecalTable1", "ReadGroup", kr)).empty() || !(e = col(t, "RecalTable1", "QualityScore", kq)).empty() ||
            !(e = col(t, "RecalTable1", "EventType", ke)).empty() || !(e = col(t, "RecalTable1", "Observations", kn)).empty() ||
            !(e = col(t, "RecalTable1", "Errors", kx)).empty()) return e;
        for (const auto &r : t.rows) {
            const std::vector<std::string> &c = r.second;
            if (c[(size_t) ke] != "M") continue;
            int q;
            if (!qual(c[(size_t) kq], q)) return err(r.first, "quality " + c[(size_t) kq] + " is not in 0..93");
            const auto g = rg_of.find(c[(size_t) kr]);
            if (g == rg_of.end()) continue;
            if (!(e = put(rgs[g->second].q[(size_t) q], r.first, c[(size_t) kn], c[(size_t) kx])).empty()) return e;
        }
    }
    {
        const Tab &t = tabs["RecalTable2"];
        int kr, kq, kv, kc, ke, kn, kx;
        if (!(e = col(t, "RecalTable2", "ReadGroup", kr)).empty() || !(e = col(t, "RecalTable2", "QualityScore", kq)).empty() ||
            !(e = col(t, "RecalTable2", "CovariateValue", kv)).empty() || !(e = col(t, "RecalTable2", "CovariateName", kc)).empty() ||
            !(e = col(t, "RecalTable2", "EventType", ke)).empty() || !(e = col(t, "RecalTable2", "Observations", kn)).empty() ||
            !(e = col(t, "RecalTable2", "Errors", kx)).empty()) return e;
        for (const auto &r : t.rows) {
            const std::vector<std::string> &c = r.second;
            if (c[(size_t) ke] != "M") continue;
            int q;
            if (!qual(c[(size_t) kq], q)) return err(r.first, "quality " + c[(size_t) kq] + " is not in 0..93");
            const std::string &v = c[(size_t) kv], &name = c[(size_t) kc];
            Row *w = nullptr;
            const auto g = rg_of.find(c[(size_t) kr]);
            if (name == "Context") {
                static const char L[] = "ACGT";
                const char *a = v.size() == 2 ? strchr(L, v[0]) : nullptr, *b = v.size() == 2 ? strchr(L, v[1]) : nullptr;
                if (!a || !b || !v[0] || !v[1]) return err(r.first, "context " + v + " is not two of ACGT");
                if (g != rg_of.end()) w = &rgs[g->second].c[(size_t) (q * BQSR_NCTX + (a - L) * 4 + (b - L))];
            } else if (name == "Cycle") {
                char *x;
                const long y = strtol(v.c_str(), &x, 10);
                if (v.empty() || *x || y == 0 || y < -BQSR_MAX_CYCLE || y > BQSR_MAX_CYCLE) return err(r.first, "cycle " + v + " is not in +-1..500");
                if (g != rg_of.end()) w = &rgs[g->second].y[(size_t) (q * BQSR_NCYC + y + BQSR_MAX_CYCLE)];
            } else return err(r.first, "covariate " + name + " is neither Context nor Cycle");
            if (w && !(e = put(*w, r.first, c[(size_t) kn], c[(size_t) kx])).empty()) return e;
        }
    }
    auto EQ = [](const Row &w, double prior) { return (double) bqsr_empirical_q(w.n, (int64_t) (w.e + 0.5), prior); };
    out.P.assign(rgs.size() * BQSR_NQ, 0.0); out.ctx.assign(rgs.size() * BQSR_NQ * BQSR_NCTX, 0.0); out.cyc.assign(rgs.size() * BQSR_NQ * BQSR_NCYC, 0.0);
    for (size_t k = 0; k < rgs.size(); ++k) {
        const Rg &g = rgs[k];
        const double G = EQ(g.r, g.E) - g.E, EG = g.E + G;
        for (int q = 0; q < BQSR_NQ; ++q) {
            const Row &wq = g.q[(size_t) q];
            const double Dq = wq.has ? EQ(wq, EG) - EG : 0.0, P = EG + Dq;
            out.P[k * BQSR_NQ + (size_t) q] = P;
            for (int c = 0; c < BQSR_NCTX; ++c) {
                const Row &w = g.c[(size_t) (q * BQSR_NCTX + c)];
                if (w.has) out.ctx[k * BQSR_NQ * BQSR_NCTX + (size_t) (q * BQSR_NCTX + c)] = EQ(w, P) - P;
            }
            for (int y = 0; y < BQSR_NCYC; ++y) {
                const Row &w = g.y[(size_t) (q * BQSR_NCYC + y)];
                if (w.has) out.cyc[k * BQSR_NQ * BQSR_NCYC + (size_t) (q * BQSR_NCYC + y)] = EQ(w, P) - P;
            }
        }
    }
    return "";
}

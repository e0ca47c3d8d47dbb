// baserecalibrator_emul.cpp — test-only: bm2_baserecalibrator compiled for the host: bqsr_device.cuh's rule one record at a time with the
// read-group lookup the kernel calls (bqsr_rg_lookup), bqsr_recal.h's read groups, map and placement check, bqsr_report.h's report of
// several covariates, and the tool's loop over the inputs' windows (bam_window.h), for tests/test_baserecalibrator_cpu.py and the GPU tests.
#include "bam_window.h"
#include "bqsr_recal.h"
#include "known_sites.h"
#include "mm_metrics.h"
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

const char *const kErrText[5] = {"has no base qualities", "is longer than 500 cycles after clipping", "has a base quality above 93",
                                 "has no RG tag", "has an RG tag that is not an @RG ID of the headers"};

// counts the records into cnt (n_cov * kBqsrCounts, the device layout); returns "" or the error of the first malformed or read-error record
// (err: its index and kind 1..5, or -1 and 0)
std::string count(const uint8_t *recs, const int64_t *starts, int64_t n_recs, const BqsrView &v, const int32_t *contig_len, const uint8_t *map,
                  int32_t n_ids, int64_t *cnt, int64_t *err) {
    err[0] = -1; err[1] = 0;
    for (int64_t i = 0; i < n_recs; ++i)
        if (bqsr_outside_contig(recs + starts[i], contig_len, v.n_seqs)) {
            const uint8_t *r = recs + starts[i];
            return "read " + std::string((const char *) r + 36, r[12] - 1) + " is malformed: its alignment is not inside contig " + std::to_string(bqsr_le32(r + 4));
        }
    for (int64_t i = 0; i < n_recs; ++i) {
        const uint8_t *rec = recs + starts[i];
        BqsrRec r;
        bqsr_prep(rec, v, r);
        int cov = 0;
        if (n_ids && r.status != BQSR_FILTERED) {
            int32_t len = 0;
            const int32_t at = bqsr_aux_rg(rec, &len);
            const int j = at >= 0 ? bqsr_rg_lookup((const BqsrRgEntry *) map, n_ids, rec, at, len) : -1;
            if (j >= 0) cov = ((const BqsrRgEntry *) map)[j].val;
            else r.status = at < 0 ? BQSR_ERR_NORG : BQSR_ERR_BADRG;
        }
        if (r.status == BQSR_COUNT) bqsr_tails(r);
        if (r.status >= BQSR_ERR_NOQUAL) {
            if (err[0] < 0) { err[0] = i; err[1] = r.status - BQSR_ERR_NOQUAL + 1; }
            continue;
        }
        if (r.status != BQSR_COUNT) continue;
        int64_t *t = cnt + (int64_t) cov * kBqsrCounts;
        ++t[kBqsrReads];
        bqsr_walk(r, [&](int32_t k, bool ins, int64_t g) {
            int q, cx, cyc, e = 0;
            if (!bqsr_base(r, v, k, ins, g, q, cx, cyc, e)) return;
            ++t[kBqsrBases];
            if (cx >= 0) { t[kBqsrCxObs + q * BQSR_NCTX + cx] += 1; t[kBqsrCxErr + q * BQSR_NCTX + cx] += e; }
            t[kBqsrCyObs + q * BQSR_NCYC + cyc + BQSR_MAX_CYCLE] += 1; t[kBqsrCyErr + q * BQSR_NCYC + cyc + BQSR_MAX_CYCLE] += e;
        });
    }
    if (err[0] < 0) return "";
    const uint8_t *r = recs + starts[err[0]];
    return "read " + std::string((const char *) r + 36, r[12] - 1) + " " + kErrText[err[1] - 1];
}

// the report of n_cov covariates (names) from the device-layout counts
std::string report(const std::vector<std::string> &names, const int64_t *cnt, std::vector<int64_t> &qual) {
    const size_t n = names.size();
    qual.assign(n * 2 * BQSR_NQ, 0);
    std::vector<BqsrCovTables> covs;
    for (size_t c = 0; c < n; ++c) {
        const int64_t *t = cnt + (int64_t) c * kBqsrCounts;
        int64_t *qo = qual.data() + c * 2 * BQSR_NQ, *qe = qo + BQSR_NQ;
        for (int q = 0; q < BQSR_NQ; ++q)
            for (int y = 0; y < BQSR_NCYC; ++y) { qo[q] += t[kBqsrCyObs + q * BQSR_NCYC + y]; qe[q] += t[kBqsrCyErr + q * BQSR_NCYC + y]; }
        covs.push_back({names[c], qo, qe, t + kBqsrCxObs, t + kBqsrCxErr, t + kBqsrCyObs, t + kBqsrCyErr});
    }
    return bqsr_report_text(covs);
}

std::vector<std::string> split(const char *s) {
    std::vector<std::string> v;
    std::string x;
    for (const char *p = s;; ++p) {
        if (!*p || *p == '\n') { v.push_back(x); x.clear(); if (!*p) break; }
        else x += *p;
    }
    return v;
}

int64_t give(const std::string &s, char *out, int64_t cap) {
    if (out && cap > (int64_t) s.size()) memcpy(out, s.c_str(), s.size() + 1);
    return (int64_t) s.size();
}

}  // namespace

extern "C" {

// the rule over records: n_ids map entries (blob from bqsr_rg_map, bre_map), n_cov covariates of kBqsrCounts counters at cnt (zeroed by
// the caller); returns 0, or 1 with the message in msg (a malformed record: err[0] -1; a read error: err = index, kind)
int32_t bre_count(const uint8_t *recs, const int64_t *starts, int64_t n_recs, const uint8_t *pac, int64_t l_pac, const int64_t *off, const int32_t *len,
                  int32_t n_seqs, const uint64_t *covered, const uint64_t *junction, const int64_t *holes, int64_t n_holes, const uint8_t *map, int32_t n_ids,
                  int64_t *cnt, int64_t *err, char *msg, int64_t cap) {
    BqsrView v{nullptr, off, n_seqs, l_pac, covered, junction, holes, n_holes, pac};
    const std::string e = count(recs, starts, n_recs, v, len, map, n_ids, cnt, err);
    give(e, msg, cap);
    return !e.empty();
}

// the read-group map of ids ('\n'-separated, n of them) with their values into blob (cap bytes); returns its size, or -1 when too large
int64_t bre_map(const char *ids, int32_t n, const int32_t *vals, uint8_t *blob, int64_t cap) {
    std::vector<std::string> v = n ? split(ids) : std::vector<std::string>();
    std::vector<uint8_t> b;
    if (!bqsr_rg_map(v, std::vector<int32_t>(vals, vals + n), b).empty() || (int64_t) b.size() > cap) return -1;
    memcpy(blob, b.data(), b.size());
    return (int64_t) b.size();
}

// the report of n covariates (names: '\n'-separated) from counts in the device layout; returns its length, written to out when it fits
int64_t bre_report(const char *names, int32_t n, const int64_t *cnt, char *out, int64_t cap) {
    std::vector<int64_t> qual;
    return give(report(n ? split(names) : std::vector<std::string>(), cnt, qual), out, cap);
}

// the read groups of headers (texts: NUL-separated, n of them; input names '\n'-separated): "ids\ncovariates\n" with each ID's covariate
// index in id_cov (cap entries), or the error; returns 0 or 1
int32_t bre_read_groups(const char *texts, int32_t n, const char *names, char *out, int64_t cap, int32_t *id_cov, int32_t id_cap, int32_t *counts) {
    std::vector<std::string> t;
    for (int32_t i = 0; i < n; ++i) { t.push_back(texts); texts += t.back().size() + 1; }
    BqsrReadGroups g;
    const std::string e = bqsr_read_groups(t, split(names), g);
    if (!e.empty()) { give(e, out, cap); return 1; }
    std::string o;
    for (const std::string &s : g.ids) o += s + "\t";
    o += "\n";
    for (const std::string &s : g.covs) o += s + "\t";
    give(o, out, cap);
    for (size_t i = 0; i < g.id_cov.size() && (int32_t) i < id_cap; ++i) id_cov[i] = g.id_cov[i];
    counts[0] = (int32_t) g.ids.size(); counts[1] = (int32_t) g.covs.size();
    return 0;
}

// the tool: prefix, inputs and VCFs ('\n'-separated), window and threads; returns 0 with the table in out, or 1 with the error.
// stats: records, windows, counted reads, counted bases, covariates, known sites
int32_t bre_run(const char *prefix, const char *inputs, const char *vcfs, int64_t window, int32_t threads, char *out, int64_t cap, int64_t *stats) {
    MmReference ref;
    std::string e = mm_read_reference(prefix, ref);
    if (!e.empty()) { give(e, out, cap); return 1; }
    const std::vector<std::string> paths = split(inputs);
    std::vector<BamWindowReader> rds(paths.size());
    std::vector<std::string> texts, names;
    auto close_all = [&] { for (BamWindowReader &rd : rds) if (rd.f) fclose(rd.f); };
    for (size_t i = 0; i < paths.size() && e.empty(); ++i) {
        BamWindowReader &rd = rds[i];
        rd.name = paths[i]; rd.threads = threads; rd.window = 0;
        rd.f = fopen(paths[i].c_str(), "rb");
        if (!rd.f) { e = "cannot open " + paths[i]; break; }
        std::string text;
        std::vector<std::pair<std::string, int32_t>> refs;
        e = rd.header(text, refs);
        if (e.empty()) { e = wgs_check_refs(refs, ref); if (!e.empty()) e = rd.where() + e; }
        rd.window = window;
        texts.push_back(text); names.push_back(rd.name);
    }
    BqsrReadGroups g;
    std::vector<uint8_t> blob;
    if (e.empty()) e = bqsr_read_groups(texts, names, g);
    if (e.empty()) e = bqsr_rg_map(g.ids, g.id_cov, blob);
    KnownSites ks;
    if (e.empty()) e = read_known_sites(split(vcfs), ref.names, ref.off, std::vector<int64_t>(ref.len.begin(), ref.len.end()), ref.l_pac, ks);
    if (!e.empty()) { close_all(); give(e, out, cap); return 1; }
    BqsrView v{nullptr, ref.off.data(), (int32_t) ref.names.size(), ref.l_pac, ks.covered.data(), ks.junction.data(), ref.holes.data(),
               (int64_t) ref.hole_char.size(), ref.pac.data()};
    std::vector<int64_t> cnt(g.covs.size() * (size_t) kBqsrCounts, 0);
    int64_t n_records = 0, n_windows = 0, err[2];
    std::vector<uint8_t> w;
    std::vector<int64_t> st;
    for (size_t i = 0; i < rds.size() && e.empty(); ++i)
        for (;;) {
            e = rds[i].next(w, st);
            if (!e.empty() || st.empty()) break;
            e = count(w.data(), st.data(), (int64_t) st.size(), v, ref.len.data(), blob.data(), (int32_t) g.ids.size(), cnt.data(), err);
            if (!e.empty()) break;
            n_records += (int64_t) st.size(); ++n_windows;
        }
    close_all();
    if (!e.empty()) { give(e, out, cap); return 1; }
    std::vector<int64_t> qual;
    const std::string text = report(g.covs, cnt.data(), qual);
    stats[0] = n_records; stats[1] = n_windows; stats[2] = stats[3] = 0;
    for (size_t c = 0; c < g.covs.size(); ++c) { stats[2] += cnt[c * kBqsrCounts + kBqsrReads]; stats[3] += cnt[c * kBqsrCounts + kBqsrBases]; }
    stats[4] = (int64_t) g.covs.size(); stats[5] = ks.records;
    if ((int64_t) text.size() >= cap) { give("output buffer too small", out, cap); return 1; }
    give(text, out, cap);
    return 0;
}

}

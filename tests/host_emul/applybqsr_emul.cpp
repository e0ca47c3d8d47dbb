// applybqsr_emul.cpp — test-only: bm2_applybqsr's rule compiled for the host (bqsr_report.h's table parser and deltas, bqsr_device.cuh's
// per-record apply rule one base at a time, bam_window.h's window reader), for tests/test_applybqsr_cpu.py and the GPU tests.
#include "bqsr_report.h"
#include "bam_window.h"
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

extern "C" {

// the report (text, named path in errors) -> the read groups' dense tables (at most max_rg; P [94], ctx [94 * 16], cyc [94 * 1001] each)
// and their names '\n'-joined; returns the read group count, or -1 with the error in err
int32_t aq_parse(const char *text, const char *path, int32_t max_rg, double *P, double *ctx, double *cyc, char *names, int64_t names_cap, char *err,
                 int64_t cap) {
    BqsrApplyTables t;
    const std::string e = bqsr_parse_report(text, path, t);
    if (!e.empty()) { snprintf(err, (size_t) cap, "%s", e.c_str()); return -1; }
    if ((int32_t) t.rgs.size() > max_rg) { snprintf(err, (size_t) cap, "more than %d read groups", max_rg); return -1; }
    memcpy(P, t.P.data(), t.P.size() * 8); memcpy(ctx, t.ctx.data(), t.ctx.size() * 8); memcpy(cyc, t.cyc.data(), t.cyc.size() * 8);
    std::string n;
    for (size_t k = 0; k < t.rgs.size(); ++k) n += (k ? "\n" : "") + t.rgs[k];
    snprintf(names, (size_t) names_cap, "%s", n.c_str());
    return (int32_t) t.rgs.size();
}

// the records at starts rewritten in place; ids: the header's @RG IDs '\n'-joined, id_table their table indices; cnt: recalibrated, kept,
// bases changed; err: the first read error's index and kind (1 over 500 bases, 2 a quality above 93), or -1 and 0
void aq_apply(uint8_t *recs, const int64_t *starts, int64_t n_recs, const char *ids, const int32_t *id_table, int32_t n_ids, int32_t n_rg,
              const double *P, const double *ctx, const double *cyc, int64_t *cnt, int64_t *err) {
    std::vector<std::string> id(1);
    for (const char *p = ids; *p; ++p) { if (*p == '\n') id.emplace_back(); else id.back() += *p; }
    err[0] = -1; err[1] = 0;
    for (int64_t i = 0; i < n_recs; ++i) {
        uint8_t *rec = recs + starts[i];
        int32_t len = 0;
        const int32_t at = bqsr_aux_rg(rec, &len);
        int rg = -1;
        if (at >= 0)
            for (int32_t j = 0; j < n_ids; ++j)
                if (id[(size_t) j] == std::string((const char *) rec + at, (size_t) len)) { rg = id_table[j]; break; }
        BqsrRec r;
        bqsr_apply_prep(rec, r);
        if (rg < 0 || rg >= n_rg) r.status = BQSR_KEEP;
        if (r.status == BQSR_APPLY) bqsr_tails(r);
        if (r.status >= BQSR_ERR_NOQUAL) {
            if (err[0] < 0) { err[0] = i; err[1] = r.status - BQSR_ERR_CYCLES + 1; }
            continue;
        }
        if (r.status == BQSR_KEEP) { ++cnt[1]; continue; }
        ++cnt[0];
        const BqsrApplyView t{P + (size_t) rg * BQSR_NQ, ctx + (size_t) rg * BQSR_NQ * BQSR_NCTX, cyc + (size_t) rg * BQSR_NQ * BQSR_NCYC};
        uint8_t *qual = (uint8_t *) r.qual;
        for (int32_t k = 0; k < r.hi; ++k) {
            int cx, cy;
            bqsr_covariates(r, k, cx, cy);
            const int nq = bqsr_recal_q(t, qual[k], cx, cy);
            if (nq != qual[k]) { qual[k] = (uint8_t) nq; ++cnt[2]; }
        }
    }
}

// the window reader over the file at path: the header text and all the records, concatenated (malloc'd: aq_free), and the window count;
// returns 0, or 1 with the error in err.  warn gets the reader's warning.
int32_t aq_read(const char *path, int64_t window, int32_t threads, uint8_t **recs, int64_t *n, char **text, int64_t *n_windows, char *err, char *warn,
                int64_t cap) {
    BamWindowReader rd;
    rd.name = path; rd.window = window; rd.threads = threads;
    rd.f = fopen(path, "rb");
    *recs = nullptr; *text = nullptr; *n = 0; *n_windows = 0; warn[0] = 0;
    if (!rd.f) { snprintf(err, (size_t) cap, "cannot open %s", path); return 1; }
    std::string t;
    std::vector<std::pair<std::string, int32_t>> refs;
    std::string e = rd.header(t, refs);
    std::vector<uint8_t> all, w;
    std::vector<int64_t> st;
    while (e.empty()) {
        e = rd.next(w, st);
        if (!e.empty() || st.empty()) break;
        for (size_t i = 0; i < st.size(); ++i) if (st[i] != (i ? st[i - 1] + 4 + bam_le32(w.data() + st[i - 1]) : 0)) e = "records not contiguous";
        all.insert(all.end(), w.begin(), w.end());
        ++*n_windows;
    }
    fclose(rd.f);
    snprintf(warn, (size_t) cap, "%s", rd.warning.c_str());
    if (!e.empty()) { snprintf(err, (size_t) cap, "%s", e.c_str()); return 1; }
    *recs = (uint8_t *) malloc(all.size() + 1);
    memcpy(*recs, all.data(), all.size());
    *n = (int64_t) all.size();
    *text = strdup(t.c_str());
    return 0;
}

void aq_free(void *p) { free(p); }

}

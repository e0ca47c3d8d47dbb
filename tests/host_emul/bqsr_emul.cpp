// bqsr_emul.cpp — test-only: the rule of bm2_mem --recal-file compiled for the host (bqsr_device.cuh's per-record logic, bqsr_report.h's
// empirical quality and report text, known_sites.h's VCF reader), one base at a time, for tests/test_bqsr_cpu.py and the GPU tests.
#include "bqsr_report.h"
#include "known_sites.h"
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

extern "C" {

// counts the records at starts into the dense tables (int64, zeroed by the caller): qo/qe [94], co/ce [94 * 16], yo/ye [94 * 1001];
// rb: reads, bases; err: the first read error's index and kind (1 no qualities, 2 cycles, 3 quality), or -1 and 0
void bqsr_emul_count(const uint8_t *recs, const int64_t *starts, int64_t n_recs, const uint8_t *ref, int64_t l_pac, const int64_t *ann_off, int32_t n_seqs,
                     const uint64_t *covered, const uint64_t *junction, const int64_t *holes, int64_t n_holes, int64_t *qo, int64_t *qe, int64_t *co,
                     int64_t *ce, int64_t *yo, int64_t *ye, int64_t *rb, int64_t *err) {
    BqsrView v{ref, ann_off, n_seqs, l_pac, covered, junction, holes, n_holes};
    err[0] = -1; err[1] = 0;
    for (int64_t i = 0; i < n_recs; ++i) {
        BqsrRec r;
        bqsr_prep(recs + starts[i], v, r);
        if (r.status == BQSR_COUNT) bqsr_tails(r);
        if (r.status >= BQSR_ERR_NOQUAL) {
            if (err[0] < 0) { err[0] = i; err[1] = r.status - BQSR_ERR_NOQUAL + 1; }
            continue;
        }
        if (r.status != BQSR_COUNT) continue;
        ++rb[0];
        bqsr_walk(r, [&](int32_t k, bool ins, int64_t g) {
            int q, cx, cyc, e = 0;
            if (!bqsr_base(r, v, k, ins, g, q, cx, cyc, e)) return;
            ++rb[1];
            qo[q] += 1; qe[q] += e;
            if (cx >= 0) { co[q * BQSR_NCTX + cx] += 1; ce[q * BQSR_NCTX + cx] += e; }
            yo[q * BQSR_NCYC + cyc + BQSR_MAX_CYCLE] += 1; ye[q * BQSR_NCYC + cyc + BQSR_MAX_CYCLE] += e;
        });
    }
}

int bqsr_emul_empirical(int64_t n, int64_t e, double prior) { return bqsr_empirical_q(n, e, prior); }

// the report text (malloc'd, the caller frees it with bqsr_emul_free)
char *bqsr_emul_report(const char *rg, const int64_t *qo, const int64_t *qe, const int64_t *co, const int64_t *ce, const int64_t *yo, const int64_t *ye) {
    const std::string t = bqsr_report_text(rg, qo, qe, co, ce, yo, ye);
    char *o = (char *) malloc(t.size() + 1);
    memcpy(o, t.c_str(), t.size() + 1);
    return o;
}

char *bqsr_emul_read_group(const char *line) {
    const std::string t = bqsr_read_group(line);
    return strdup(t.c_str());
}

// the VCFs (paths: '\n'-separated) over the contigs (names: '\n'-separated) into covered / junction ((l_pac + 63) / 64 words each);
// returns the record count, or -1 with the error in err (cap bytes)
int64_t bqsr_emul_sites(const char *paths, const char *names, const int64_t *off, const int64_t *len, int32_t n_seqs, int64_t l_pac, uint64_t *covered,
                        uint64_t *junction, char *err, int64_t cap) {
    auto split = [](const char *s) { std::vector<std::string> v; std::string x; for (const char *p = s; ; ++p) { if (!*p || *p == '\n') { v.push_back(x); x.clear(); if (!*p) break; } else x += *p; } return v; };
    const std::vector<std::string> ps = split(paths), ns = split(names);
    KnownSites ks;
    const std::string e = read_known_sites(ps, std::vector<std::string>(ns.begin(), ns.begin() + n_seqs), std::vector<int64_t>(off, off + n_seqs),
                                           std::vector<int64_t>(len, len + n_seqs), l_pac, ks);
    if (!e.empty()) { snprintf(err, (size_t) cap, "%s", e.c_str()); return -1; }
    memcpy(covered, ks.covered.data(), ks.covered.size() * 8);
    memcpy(junction, ks.junction.data(), ks.junction.size() * 8);
    return ks.records;
}

void bqsr_emul_free(void *p) { free(p); }

}

// wgsmetrics_emul.cpp — test-only: bm2_wgsmetrics compiled for the host.  wgs.cu's phases (check, count, overlap by (name hash, file order)
// with the carry between windows, finish) one base at a time over wgs_device.cuh's rule, wgs_metrics.h's reference reader, header and order
// checks and file text, and the tool's window loop over bam_window.h's reader; for tests/test_wgsmetrics_cpu.py and the GPU tests.
#include "bam_window.h"
#include "wgs_metrics.h"
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

struct Emul {
    std::vector<int64_t> off;
    std::vector<int32_t> len;
    int64_t l_pac = 0;
    std::vector<uint32_t> nocall, pile;
    bm2_wgs_params_t p{};
    int64_t exc[WGS_NEXC] = {0, 0, 0, 0, 0, 0};
    int64_t seen = 0, counted = 0, carried_max = 0;
    std::vector<uint8_t> carry;
    std::vector<int64_t> cst;
    WgsOrder order;
};

const char *const kErrText[3] = {"has no base qualities (l_seq 0 or QUAL '*')", "does not lie inside a contig of the reference",
                                 "has a CIGAR that does not match its record"};

void set_err(char *err, int64_t cap, const std::string &m) { snprintf(err, (size_t) cap, "%s", m.c_str()); }

// wgs.cu's bm2_wgs_add: 0, 1 (the tool's order check failed) or 2 (a read error) with the message in err
int add(Emul &E, const uint8_t *recs, const int64_t *starts, int64_t n_recs, bool check_order, char *err, int64_t cap) {
    if (check_order)
        for (int64_t i = 0; i < n_recs; ++i) {
            const std::string e = E.order.check(recs + starts[i]);
            if (!e.empty()) { set_err(err, cap, e); return 1; }
        }
    if (!n_recs) return 0;
    const int64_t n_carry = (int64_t) E.cst.size(), n_all = n_carry + n_recs;
    std::vector<const uint8_t *> R;
    for (int64_t i = 0; i < n_carry; ++i) R.push_back(E.carry.data() + E.cst[(size_t) i]);
    for (int64_t i = 0; i < n_recs; ++i) R.push_back(recs + starts[i]);
    // check
    std::vector<WgsInfo> info((size_t) n_all);
    std::vector<uint64_t> keys((size_t) n_all);
    for (int64_t w = 0; w < n_all; ++w) {
        const uint8_t *r = R[(size_t) w];
        const DupCigar c = dup_cigar(r);
        const bool inside = wgs_cigar_inside(r, c);
        int64_t s[3] = {0, 0, 0};
        if (inside) wgs_cigar_part(c, 0, 1, s);
        const int st = wgs_status(r, s, inside, E.off.data(), E.len.data(), (int32_t) E.off.size(), E.p, info[(size_t) w]);
        keys[(size_t) w] = wgs_key(r, info[(size_t) w]);
        if (st >= WGS_ERR_NOQUAL && w >= n_carry) {
            set_err(err, cap, "bm2_wgs_add: read " + std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0) + " (record " +
                                  std::to_string(E.seen + w - n_carry) + ") " + kErrText[st - WGS_ERR_NOQUAL]);
            return 2;
        }
    }
    // count
    for (int64_t w = n_carry; w < n_all; ++w) {
        const WgsInfo &in = info[(size_t) w];
        if (in.status <= WGS_FILT_UNPAIRED) { E.exc[in.status] += in.aligned; continue; }
        if (in.status != WGS_PASS) continue;
        ++E.counted;
        const uint8_t *r = R[(size_t) w];
        const DupCigar c = dup_cigar(r);
        const WgsSeq sq = wgs_seq(r);
        int64_t k = 0, g = in.g0;
        for (int64_t i = 0; i < c.n; ++i) {
            const uint32_t op = dup_op(c, i), ln = op >> 4;
            if (wgs_aligned_op(op))
                for (uint32_t b = 0; b < ln; ++b) {
                    if (wgs_nocall(E.nocall.data(), g + b)) continue;
                    if (wgs_hq(sq, k + b, E.p.min_baseq)) ++E.pile[(size_t) (g + b)];
                    else ++E.exc[WGS_EXC_BASEQ];
                }
            if (dup_consumes_ref(op)) g += ln;
            if (wgs_query_op(op)) k += ln;
        }
    }
    // overlap
    std::vector<int64_t> ord((size_t) n_all);
    for (int64_t i = 0; i < n_all; ++i) ord[(size_t) i] = i;
    std::stable_sort(ord.begin(), ord.end(), [&](int64_t a, int64_t b) { return keys[(size_t) a] < keys[(size_t) b]; });
    for (int64_t i = 0; i < n_all;) {
        const uint64_t key = keys[(size_t) ord[(size_t) i]];
        int64_t e = i + 1;
        while (e < n_all && keys[(size_t) ord[(size_t) e]] == key) ++e;
        if (key & WGS_NOT_CANDIDATE) break;
        for (int64_t j = i + 1; j < e; ++j) {
            const int64_t x = ord[(size_t) j];
            if (x < n_carry) continue;
            const WgsInfo &in = info[(size_t) x];
            const uint8_t *r = R[(size_t) x];
            const DupCigar c = dup_cigar(r);
            const WgsSeq sq = wgs_seq(r);
            int64_t k = 0, g = in.g0;
            for (int64_t oi = 0; oi < c.n; ++oi) {
                const uint32_t op = dup_op(c, oi), ln = op >> 4;
                if (wgs_aligned_op(op))
                    for (uint32_t b = 0; b < ln; ++b) {
                        const int64_t gg = g + b;
                        if (wgs_nocall(E.nocall.data(), gg) || !wgs_hq(sq, k + b, E.p.min_baseq)) continue;
                        bool cov = false;
                        for (int64_t m = i; m < j && !cov; ++m) {
                            const int64_t y = ord[(size_t) m];
                            const WgsInfo &im = info[(size_t) y];
                            if (wgs_spans_overlap(im, in) && wgs_same_name(R[(size_t) y], r)) cov = wgs_hq_at(R[(size_t) y], dup_cigar(R[(size_t) y]), im.g0, gg, E.p.min_baseq);
                        }
                        if (cov) { --E.pile[(size_t) gg]; ++E.exc[WGS_EXC_OVERLAP]; }
                    }
                if (dup_consumes_ref(op)) g += ln;
                if (wgs_query_op(op)) k += ln;
            }
        }
        i = e;
    }
    // carry
    const BamFixed lf = bam_fixed(recs + starts[n_recs - 1]);
    const int64_t last_g = lf.rid >= 0 && lf.rid < (int32_t) E.off.size() ? E.off[(size_t) lf.rid] + lf.pos : 0;
    std::vector<uint8_t> carry;
    std::vector<int64_t> cst;
    for (int64_t i = 0; i < n_all; ++i) {
        if (!wgs_carried(info[(size_t) i], lf.rid, last_g)) continue;
        const uint8_t *r = R[(size_t) i];
        cst.push_back((int64_t) carry.size());
        carry.insert(carry.end(), r, r + 4 + bam_le32(r));
    }
    E.carry.swap(carry); E.cst.swap(cst);
    E.carried_max = std::max<int64_t>(E.carried_max, (int64_t) E.cst.size());
    E.seen += n_recs;
    return 0;
}

WgsCounts finish(const Emul &E) {
    WgsCounts x;
    x.hist.assign((size_t) E.p.coverage_cap + 1, 0);
    for (int k = 0; k < WGS_NEXC; ++k) x.exc[k] = E.exc[k];
    x.exc[WGS_EXC_CAPPED] = 0;
    for (int64_t g = 0; g < E.l_pac; ++g) {
        if (wgs_nocall(E.nocall.data(), g)) continue;
        const uint32_t d = E.pile[(size_t) g];
        if (d > (uint32_t) E.p.coverage_cap) x.exc[WGS_EXC_CAPPED] += d - (uint32_t) E.p.coverage_cap;
        ++x.hist[std::min<uint32_t>(d, (uint32_t) E.p.coverage_cap)];
    }
    return x;
}

}  // namespace

extern "C" {

void *wm_new(const int64_t *off, const int32_t *len, int32_t n_contigs, int64_t l_pac, const int64_t *nocall, int64_t n_nocall, int32_t min_mapq,
             int32_t min_baseq, int32_t cap, int32_t count_unpaired) {
    Emul *E = new Emul();
    E->off.assign(off, off + n_contigs); E->len.assign(len, len + n_contigs);
    E->l_pac = l_pac;
    E->nocall.assign((size_t) (l_pac + 31) / 32 + 1, 0);
    for (int64_t h = 0; h < n_nocall; ++h)
        for (int64_t g = nocall[2 * h]; g < nocall[2 * h + 1]; ++g) E->nocall[(size_t) (g >> 5)] |= 1u << (g & 31);
    E->pile.assign((size_t) l_pac, 0);
    E->p = bm2_wgs_params_t{min_mapq, min_baseq, cap, count_unpaired};
    return E;
}

int32_t wm_add(void *h, const uint8_t *recs, const int64_t *starts, int64_t n_recs, int32_t check_order, char *err, int64_t cap) {
    return add(*(Emul *) h, recs, starts, n_recs, check_order != 0, err, cap);
}

// hist [cap + 1], exc [6], stats: records, counted records, carried max
void wm_finish(void *h, int64_t *hist, int64_t *exc, int64_t *stats) {
    const Emul &E = *(Emul *) h;
    const WgsCounts x = finish(E);
    memcpy(hist, x.hist.data(), x.hist.size() * 8);
    memcpy(exc, x.exc, sizeof x.exc);
    stats[0] = E.seen; stats[1] = E.counted; stats[2] = E.carried_max;
}

void wm_free(void *h) { delete (Emul *) h; }

// the metrics file of (hist [cap + 1], exc [6]) for the arguments args; returns its length, written to out when it fits
int64_t wm_text(const int64_t *hist, int32_t cap, const int64_t *exc, const char *args, char *out, int64_t out_cap) {
    WgsCounts x;
    x.hist.assign(hist, hist + cap + 1);
    for (int k = 0; k < WGS_NEXC; ++k) x.exc[k] = exc[k];
    const std::string t = wgs_metrics_text(x, args);
    if ((int64_t) t.size() < out_cap) memcpy(out, t.c_str(), t.size() + 1);
    return (int64_t) t.size();
}

// the tool over a file: reference, header checks, windows with the order check, finish, text.  Returns 0 with the text in out, or 1 with
// the error in out.  stats: records, counted records, windows, carried max.
int32_t wm_run(const char *prefix, const char *bam, int64_t window, int32_t threads, int32_t min_mapq, int32_t min_baseq, int32_t cap,
               int32_t count_unpaired, const char *args, char *out, int64_t out_cap, int64_t *stats) {
    WgsReference ref;
    std::string e = wgs_read_reference(prefix, ref);
    if (!e.empty()) { set_err(out, out_cap, e); return 1; }
    BamWindowReader rd;
    rd.name = bam; rd.window = window; rd.threads = threads;
    rd.f = fopen(bam, "rb");
    if (!rd.f) { set_err(out, out_cap, std::string("cannot open ") + bam); return 1; }
    std::string text;
    std::vector<std::pair<std::string, int32_t>> refs;
    e = rd.header(text, refs);
    if (e.empty()) { e = wgs_check_header(text, refs, ref); if (!e.empty()) e = rd.where() + e; }
    if (!e.empty()) { fclose(rd.f); set_err(out, out_cap, e); return 1; }
    Emul *E = (Emul *) wm_new(ref.off.data(), ref.len.data(), (int32_t) ref.off.size(), ref.l_pac, ref.nocall.data(), (int64_t) ref.nocall.size() / 2,
                              min_mapq, min_baseq, cap, count_unpaired);
    std::vector<uint8_t> w;
    std::vector<int64_t> st;
    int64_t n_windows = 0;
    char err[4096];
    for (;;) {
        e = rd.next(w, st);
        if (!e.empty() || st.empty()) break;
        const int rc = add(*E, w.data(), st.data(), (int64_t) st.size(), true, err, sizeof err);
        if (rc) { e = rc == 1 ? rd.where() + err : std::string(err); break; }
        ++n_windows;
    }
    fclose(rd.f);
    if (!e.empty()) { wm_free(E); set_err(out, out_cap, e); return 1; }
    const std::string t = wgs_metrics_text(finish(*E), args);
    stats[0] = E->seen; stats[1] = E->counted; stats[2] = n_windows; stats[3] = E->carried_max;
    wm_free(E);
    set_err(out, out_cap, t);
    return 0;
}

}

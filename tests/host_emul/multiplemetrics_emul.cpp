// multiplemetrics_emul.cpp — test-only: bm2_multiplemetrics compiled for the host.  mm.cu's check and count kernels one record and one base
// at a time over mm_device.cuh's rule, mm_metrics.h's reference reader, formulas and file text, and the tool's window loop over
// bam_window.h's reader; for tests/test_multiplemetrics_cpu.py and the GPU tests.
#include "bam_window.h"
#include "mm_metrics.h"
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

struct Emul {
    std::vector<int64_t> off;
    std::vector<int32_t> len;
    int64_t l_pac = 0;
    std::vector<uint8_t> pac;
    std::vector<uint32_t> hole_bits;
    std::vector<int64_t> holes;
    std::vector<char> hole_char;
    char kmers[MM_N_ADAPTER_KMERS][MM_ADAPTER_LEN];
    MmCounts x;
    int64_t seen = 0;
};

const char *const kErrText[3] = {"has l_seq 0 or above 1048576", "does not lie inside a contig of the reference",
                                 "has a CIGAR that does not match its record"};

void set_err(char *err, int64_t cap, const std::string &m) { snprintf(err, (size_t) cap, "%s", m.c_str()); }

void bump(std::vector<int64_t> &v, int64_t k) {
    if ((int64_t) v.size() <= k) v.resize((size_t) k + 1, 0);
    ++v[(size_t) k];
}

// mm.cu's bm2_mm_add: 0, or 2 (a read error) with the message in err
int add(Emul &E, const uint8_t *recs, const int64_t *starts, int64_t n_recs, char *err, int64_t cap) {
    std::vector<MmInfo> info((size_t) n_recs);
    for (int64_t w = 0; w < n_recs; ++w) {                                        // check
        const uint8_t *r = recs + starts[w];
        const DupCigar c = dup_cigar(r);
        const bool inside = wgs_cigar_inside(r, c);
        int64_t s[3] = {0, 0, 0}, t[3] = {0, 0, 0};
        if (inside) { wgs_cigar_part(c, 0, 1, s); mm_clip_part(c, 0, 1, t); }
        mm_classify(r, s, t, inside, E.off.data(), E.len.data(), (int32_t) E.off.size(), E.kmers, info[(size_t) w]);
        if (info[(size_t) w].err) {
            set_err(err, cap, "bm2_mm_add: read " + std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0) + " (record " +
                                  std::to_string(E.seen + w) + ") " + kErrText[info[(size_t) w].err - 1]);
            return 2;
        }
    }
    for (int64_t w = 0; w < n_recs; ++w) {                                        // count
        const MmInfo &in = info[(size_t) w];
        if (!(in.bits & MMB_COUNTED)) continue;
        const uint8_t *r = recs + starts[w];
        const WgsSeq sq = wgs_seq(r);
        for (int32_t k = 0; k < in.l_seq; ++k)
            if (mm_nibble(sq.seq, k) == 15) bump(E.x.nocall[in.cat], (in.bits & MMB_REV) ? in.l_seq - 1 - k : k);
        uint32_t mism = 0, q20 = 0;
        if (in.bits & MMB_ALIGNED) {
            const DupCigar c = dup_cigar(r);
            int64_t k = 0, g = in.g0;
            for (int64_t i = 0; i < c.n; ++i) {
                const uint32_t op = dup_op(c, i), ln = op >> 4;
                if (wgs_aligned_op(op))
                    for (uint32_t b = 0; b < ln; ++b)
                        mm_base(sq, in.bits & MMB_NOQUAL, k + b, g + b, E.pac.data(), E.hole_bits.data(), E.holes.data(), E.hole_char.data(),
                                (int64_t) E.hole_char.size(), mism, q20);
                if (dup_consumes_ref(op)) g += ln;
                if (wgs_query_op(op)) k += ln;
            }
        }
        int64_t v[MM_NCOUNT];
        mm_record_counts(in, mism, q20, v);
        for (int k = 0; k < MM_NCOUNT; ++k) E.x.c[in.cat][k] += v[k];
        bump(E.x.len[in.cat], in.l_seq);
        if (in.bits & MMB_HQ) bump(E.x.mism[in.cat], mism);
        if (in.bits & MMB_INSERT) E.x.ins[in.orient][in.insert] += 1;
    }
    E.seen += n_recs;
    return 0;
}

Emul *make(const int64_t *off, const int32_t *len, int32_t n_contigs, int64_t l_pac, const uint8_t *pac, const int64_t *holes, const char *hole_char,
           int64_t n_holes) {
    Emul *E = new Emul();
    E->off.assign(off, off + n_contigs); E->len.assign(len, len + n_contigs);
    E->l_pac = l_pac;
    E->pac.assign(pac, pac + (l_pac + 3) / 4);
    E->holes.assign(holes, holes + 2 * n_holes); E->hole_char.assign(hole_char, hole_char + n_holes);
    E->holes.push_back(0); E->holes.push_back(0);                                 // never read: keeps data() valid when there is no hole
    E->hole_bits.assign((size_t) (l_pac + 31) / 32 + 1, 0);
    for (size_t w = 0; w < E->hole_bits.size(); ++w) E->hole_bits[w] = wgs_range_word(E->holes.data(), n_holes, (int64_t) w);
    mm_adapter_kmers(E->kmers);
    return E;
}

int64_t give(const std::string &t, char *out, int64_t out_cap) {
    if ((int64_t) t.size() < out_cap) memcpy(out, t.c_str(), t.size() + 1);
    return (int64_t) t.size();
}

}  // namespace

extern "C" {

void *mme_new(const int64_t *off, const int32_t *len, int32_t n_contigs, int64_t l_pac, const uint8_t *pac, const int64_t *holes, const char *hole_char,
              int64_t n_holes) {
    return make(off, len, n_contigs, l_pac, pac, holes, hole_char, n_holes);
}

int32_t mme_add(void *h, const uint8_t *recs, const int64_t *starts, int64_t n_recs, char *err, int64_t cap) {
    return add(*(Emul *) h, recs, starts, n_recs, err, cap);
}

// the counters [3][21], and the largest key of each histogram kind (len, mism, nocall) and the insert pairs per orientation [3]
void mme_counts(void *h, int64_t *counts, int64_t *pairs) {
    const Emul &E = *(Emul *) h;
    for (int c = 0; c < MM_NCAT; ++c) for (int k = 0; k < MM_NCOUNT; ++k) counts[c * MM_NCOUNT + k] = E.x.c[c][k];
    for (int o = 0; o < MM_NORIENT; ++o) { pairs[o] = 0; for (const auto &p : E.x.ins[o]) pairs[o] += p.second; }
}

// the file `which` (0 the alignment summary, 1 the insert sizes) for the arguments args; returns its length, written to out when it fits
int64_t mme_text(void *h, int32_t which, const char *args, char *out, int64_t out_cap) {
    const Emul &E = *(Emul *) h;
    int64_t pairs = 0;
    return give(which ? mm_insert_text(E.x, args, &pairs) : mm_summary_text(E.x, args), out, out_cap);
}

void mme_free(void *h) { delete (Emul *) h; }

// the tool over a file: reference, header check, windows, text.  Returns 0 with the two files in out (separated by a NUL), or 1 with the
// error in out.  stats: records, windows.
int32_t mme_run(const char *prefix, const char *bam, int64_t window, int32_t threads, const char *args, char *out, int64_t out_cap, int64_t *stats) {
    MmReference ref;
    std::string e = mm_read_reference(prefix, ref);
    if (!e.empty()) { set_err(out, out_cap, e); return 1; }
    BamWindowReader rd;
    rd.name = bam; rd.window = window; rd.threads = threads;
    rd.f = fopen(bam, "rb");
    if (!rd.f) { set_err(out, out_cap, std::string("cannot open ") + bam); return 1; }
    std::string text;
    std::vector<std::pair<std::string, int32_t>> refs;
    e = rd.header(text, refs);
    if (e.empty()) { e = wgs_check_refs(refs, ref); if (!e.empty()) e = rd.where() + e; }
    if (!e.empty()) { fclose(rd.f); set_err(out, out_cap, e); return 1; }
    Emul *E = make(ref.off.data(), ref.len.data(), (int32_t) ref.off.size(), ref.l_pac, ref.pac.data(), ref.holes.data(), ref.hole_char.data(),
                   (int64_t) ref.hole_char.size());
    std::vector<uint8_t> w;
    std::vector<int64_t> st;
    int64_t n_windows = 0;
    char err[4096];
    for (;;) {
        e = rd.next(w, st);
        if (!e.empty() || st.empty()) break;
        if (add(*E, w.data(), st.data(), (int64_t) st.size(), err, sizeof err)) { e = err; break; }
        ++n_windows;
    }
    fclose(rd.f);
    if (!e.empty()) { delete E; set_err(out, out_cap, e); return 1; }
    int64_t pairs = 0;
    const std::string a = mm_summary_text(E->x, args), b = mm_insert_text(E->x, args, &pairs);
    stats[0] = E->seen; stats[1] = n_windows;
    delete E;
    if ((int64_t) (a.size() + b.size() + 2) > out_cap) { set_err(out, out_cap, "output buffer too small"); return 1; }
    memcpy(out, a.c_str(), a.size() + 1);
    memcpy(out + a.size() + 1, b.c_str(), b.size() + 1);
    return 0;
}

}

// gcbias_emul.cpp — test-only: bm2_multiplemetrics' GC bias compiled for the host.  mm.cu's reference scan one window at a time (the
// letters by mm_ref_letter, counted afresh for every window), the check and count kernels with GC on one record and one base at a time over
// mm_device.cuh's rule, and mm_gcbias.h's formulas and text; for tests/test_gcbias_cpu.py and the GPU tests.
#include "mm_gcbias.h"
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
    MmGcCounts x;
    int64_t seen = 0;
};

const char *const kErrText[3] = {"has l_seq 0 or above 1048576", "does not lie inside a contig of the reference",
                                 "has a CIGAR that does not match its record"};

char letter(const Emul &E, int64_t g) {
    return mm_ref_letter(E.pac.data(), E.hole_bits.data(), E.holes.data(), E.hole_char.data(), (int64_t) E.hole_char.size(), g);
}

// the bin of the window at locus g, or -1
int window_bin(const Emul &E, int64_t g) {
    int gc = 0, n = 0;
    for (int k = 0; k < MM_GC_W; ++k) {
        const int c = mm_gc_class(letter(E, g + k));
        gc += c == 1; n += c == 2;
    }
    return mm_gc_bin(gc, n);
}

// mm.cu's scan
void scan(Emul &E) {
    for (size_t c = 0; c < E.off.size(); ++c)
        for (int64_t i = 1; i < (int64_t) E.len[c] - MM_GC_W; ++i) {
            const int bin = window_bin(E, E.off[c] + i);
            if (bin >= 0) E.x.windows[bin] += 1;
        }
}

// mm.cu's bm2_mm_add with GC on: 0, or 2 (a read error) with the message in err
int add(Emul &E, const uint8_t *recs, const int64_t *starts, int64_t n_recs, char *err, int64_t cap) {
    std::vector<MmInfo> info((size_t) n_recs);
    std::vector<MmGc> gi((size_t) n_recs);
    for (int64_t w = 0; w < n_recs; ++w) {                                        // check
        const uint8_t *r = recs + starts[w];
        const DupCigar c = dup_cigar(r);
        const bool inside = wgs_cigar_inside(r, c);
        int64_t s[3] = {0, 0, 0}, t[3] = {0, 0, 0}, idlen = 0;
        if (inside) { wgs_cigar_part(c, 0, 1, s); mm_clip_part(c, 0, 1, t); idlen = mm_gc_idlen_part(c, 0, 1); }
        MmInfo &in = info[(size_t) w];
        mm_classify(r, s, t, inside, E.off.data(), E.len.data(), (int32_t) E.off.size(), E.kmers, in, true);
        if (in.err) {
            snprintf(err, (size_t) cap, "%s", ("bm2_mm_add: read " + std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0) + " (record " +
                                               std::to_string(E.seen + w) + ") " + kErrText[in.err - 1]).c_str());
            return 2;
        }
        gi[(size_t) w] = MmGc{(in.bits & MMB_PLACED) ? mm_gc_window(r, s[1], E.off.data(), E.len.data()) : -1, idlen};
    }
    for (int64_t w = 0; w < n_recs; ++w) {                                        // count
        const MmInfo &in = info[(size_t) w];
        if (!(in.bits & MMB_COUNTED)) continue;
        const uint8_t *r = recs + starts[w];
        uint32_t mism = 0, q20 = 0;
        if (in.bits & MMB_PLACED) {
            const WgsSeq sq = wgs_seq(r);
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
        E.x.clusters += in.cat != MM_SECOND;
        E.x.aligned += (in.bits & MMB_PLACED) != 0;
        const int bin = gi[(size_t) w].gw >= 0 ? window_bin(E, gi[(size_t) w].gw) : -1;
        if (bin >= 0) { E.x.reads[bin] += 1; E.x.bases[bin] += in.l_seq; E.x.errors[bin] += (int64_t) mism + gi[(size_t) w].idlen; }
    }
    E.seen += n_recs;
    return 0;
}

int64_t give(const std::string &t, char *out, int64_t out_cap) {
    if ((int64_t) t.size() < out_cap) memcpy(out, t.c_str(), t.size() + 1);
    return (int64_t) t.size();
}

}  // namespace

extern "C" {

// a reference (as bm2_mm_set takes it); scans its windows
void *gce_new(const int64_t *off, const int32_t *len, int32_t n_contigs, int64_t l_pac, const uint8_t *pac, const int64_t *holes, const char *hole_char,
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
    scan(*E);
    return E;
}

int32_t gce_add(void *h, const uint8_t *recs, const int64_t *starts, int64_t n_recs, char *err, int64_t cap) {
    return add(*(Emul *) h, recs, starts, n_recs, err, cap);
}

// windows, reads, bases, errors [4][101], then total clusters and aligned reads [2]
void gce_counts(void *h, int64_t *bins, int64_t *totals) {
    const MmGcCounts &x = ((Emul *) h)->x;
    for (int k = 0; k < MM_GC_BINS; ++k) {
        bins[k] = x.windows[k]; bins[MM_GC_BINS + k] = x.reads[k]; bins[2 * MM_GC_BINS + k] = x.bases[k]; bins[3 * MM_GC_BINS + k] = x.errors[k];
    }
    totals[0] = x.clusters; totals[1] = x.aligned;
}

// the file `which` (0 the detail, 1 the summary) of counts given as gce_counts returns them; returns its length, written to out when it fits
int64_t gce_text(const int64_t *bins, const int64_t *totals, int32_t which, const char *args, char *out, int64_t out_cap) {
    MmGcCounts x;
    for (int k = 0; k < MM_GC_BINS; ++k) {
        x.windows[k] = bins[k]; x.reads[k] = bins[MM_GC_BINS + k]; x.bases[k] = bins[2 * MM_GC_BINS + k]; x.errors[k] = bins[3 * MM_GC_BINS + k];
    }
    x.clusters = totals[0]; x.aligned = totals[1];
    return give(which ? mm_gc_summary_text(x, args) : mm_gc_detail_text(x, args), out, out_cap);
}

// mm_gc_word of locus word w, for the test of the scan's bitsets against the letters
void gce_word(void *h, int64_t w, uint32_t *gcm, uint32_t *nm) {
    const Emul &E = *(Emul *) h;
    mm_gc_word(E.pac.data(), E.hole_bits.data(), E.holes.data(), E.hole_char.data(), (int64_t) E.hole_char.size(), E.l_pac, w, *gcm, *nm);
}

void gce_free(void *h) { delete (Emul *) h; }

}

// ext_device.cuh — extension-job construction, result folding, post-filter and the tail of
// mem_kernel2_core for ONE read / ONE job (device logic).
//
// Replaces mem_chain2aln_across_reads_V2 (reference src/bwamem.cpp:2069-2994: job build :2108-2438,
// band retry + fold :2472-2880, post-filter :2895-2989), cal_max_gap (:66-76), bns_fetch_seq_v2
// (:1890-1924), and the tail of mem_kernel2_core (:1141-1169) incl. mem_sort_dedup_patch (:292-353),
// mem_patch_reg (:175-234), bwa_gen_cigar2's score path (src/bwa.cpp:260-347) and the score-only
// ksw_global2 (src/ksw.cpp:558-668).
#pragma once
#include <string.h>
#include "hd.h"
#include "bm2_b200.h"
#include "chain_device.cuh"

#define BM2_H0 (-99)     // H0_, src/macro.h:44

struct ExtParams {
    int a, b, o_del, e_del, o_ins, e_ins, w, pen_clip5, pen_clip3, max_chain_gap;
    float mask_level_redun;
    int8_t mat[25];
};

struct ExtJobRec {       // one extension job; mirrors BswJob + the reg it belongs to
    int64_t toff; int64_t qoff; int32_t tlen, qlen; int32_t h0; int8_t tstride, qstride; int16_t _pad;
};

BM2_HD int cal_max_gap_d(const ExtParams &p, int qlen) {
    int l_del = (int) ((double) (qlen * p.a - p.o_del) / p.e_del + 1.);
    int l_ins = (int) ((double) (qlen * p.a - p.o_ins) / p.e_ins + 1.);
    int l = l_del > l_ins ? l_del : l_ins;
    l = l > 1 ? l : 1;
    return l < p.w << 1 ? l : p.w << 1;
}

BM2_HD int reg_n_comp_d(const bm2_alnreg_t &a) { return (a.n_comp_is_alt << 2) >> 2; }
BM2_HD void reg_set_n_comp_d(bm2_alnreg_t &a, int v) { a.n_comp_is_alt = (a.n_comp_is_alt & ~0x3FFFFFFF) | (v & 0x3FFFFFFF); }
BM2_HD void reg_set_is_alt_d(bm2_alnreg_t &a, int v) { a.n_comp_is_alt = (a.n_comp_is_alt & 0x3FFFFFFF) | ((v & 3) << 30); }

// Whole-record copy as seven 16-byte words: a member-wise struct assignment may skip the padding bytes, which are part of
// the output (callers compare / checksum records as bytes).  Records are 16-byte aligned (112 = 7 x 16, buffers from cudaMalloc).
static_assert(sizeof(bm2_alnreg_t) == 112, "bm2_alnreg_t layout");
BM2_HD void reg_copy(bm2_alnreg_t *dst, const bm2_alnreg_t *src) {
#if defined(__CUDA_ARCH__)
    const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
    uint4 *d4 = reinterpret_cast<uint4 *>(dst);
    uint4 v[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) v[k] = s4[k];
#pragma unroll
    for (int k = 0; k < 7; ++k) d4[k] = v[k];
#else
    memcpy(dst, src, sizeof(bm2_alnreg_t));
#endif
}

BM2_HD void seedcov_d(bm2_alnreg_t &a, const bm2_seed *seeds, int n) {
    if (a.rb != BM2_H0 && a.qb != BM2_H0 && a.qe != BM2_H0 && a.re != BM2_H0) {
        int cov = 0;
        for (int i = 0; i < n; ++i) {
            const bm2_seed &t = seeds[i];
            if (t.qbeg >= a.qb && t.qbeg + t.len <= a.qe && t.rbeg >= a.rb && t.rbeg + t.len <= a.re) cov += t.len;
        }
        a.seedcov = cov;
    }
}

// Per-reg extension state of the lazy extension (one byte per reg; see ext_walk_read_d):
enum : uint8_t {
    EXT_TODO = 0,       // not extended, not decided
    EXT_DONE = 1,       // extended (or needs no extension: the seed spans the read)
    EXT_SKIP = 2,       // not extended, and the walk proved the seed purged: never extended
    EXT_NEED = 3        // to be extended by the next wave: the first seed of a chain, or the seed a walk stopped at
};

// Builds regs + jobs of one read.  chains/seeds: the read's finalized chains; regs, reg_chain,
// reg_seed: the read's output stripe (one entry per seed, creation order); left/right jobs and their
// reg ids (GLOBAL reg index = reg_base + local).  srt: scratch of >= max chain length uint64.
// state (may be null): the regs' extension states for the lazy extension (EXT_NEED for the first seed of each chain).
BM2_HD void ext_build_read_d(const ContigView &cv, const ExtParams &p, const bm2_chain *chains, int n_chain, const bm2_seed *seeds,
                             int l_query, int64_t read_code_off, int64_t chain_base, int64_t reg_base, bm2_alnreg_t *regs,
                             int32_t *reg_chain, int32_t *reg_seed, ExtJobRec *left, int32_t *left_reg, ExtJobRec *right,
                             int32_t *right_reg, uint64_t *srt, uint8_t *state = nullptr)
{
    const int64_t l_pac = cv.l_pac;
    int n_reg = 0, nl = 0, nr = 0;
    for (int ci = 0; ci < n_chain; ++ci) {
        const bm2_chain &c = chains[ci];
        const bm2_seed *cs = seeds + c.seed_off;
        const int n = c.n_seeds;
        if (n == 0) continue;
        int64_t rmax0 = l_pac << 1, rmax1 = 0;
        for (int i = 0; i < n; ++i) {
            const bm2_seed &t = cs[i];
            const int64_t b = t.rbeg - (t.qbeg + cal_max_gap_d(p, t.qbeg));
            const int64_t e = t.rbeg + t.len + ((l_query - t.qbeg - t.len) + cal_max_gap_d(p, l_query - t.qbeg - t.len));
            rmax0 = rmax0 < b ? rmax0 : b;
            rmax1 = rmax1 > e ? rmax1 : e;
        }
        rmax0 = rmax0 > 0 ? rmax0 : 0;
        rmax1 = rmax1 < l_pac << 1 ? rmax1 : l_pac << 1;
        if (rmax0 < l_pac && l_pac < rmax1) { if (cs[0].rbeg < l_pac) rmax1 = l_pac; else rmax0 = l_pac; }
        {   // bns_fetch_seq_v2: clip the window to the contig of seeds[0].rbeg
            const int64_t mid = cs[0].rbeg;
            const int is_rev = mid >= l_pac;
            const int rid = bns_pos2rid_d(cv, bns_depos_d(cv, mid));
            int64_t far_beg = cv.ann_off[rid], far_end = far_beg + cv.ann_len[rid];
            if (is_rev) { const int64_t tmp = far_beg; far_beg = (l_pac << 1) - far_end; far_end = (l_pac << 1) - tmp; }
            rmax0 = rmax0 > far_beg ? rmax0 : far_beg;
            rmax1 = rmax1 < far_end ? rmax1 : far_end;
        }
        // seeds in ascending (score, index); keys are unique so any sorting algorithm gives the
        // order of ks_introsort_64 (src/bwamem.cpp:2188-2192)
        for (int i = 0; i < n; ++i) srt[i] = (uint64_t) cs[i].score << 32 | (uint32_t) i;
        for (int i = 1; i < n; ++i) { uint64_t v = srt[i]; int j = i; while (j > 0 && srt[j - 1] > v) { srt[j] = srt[j - 1]; --j; } srt[j] = v; }
        for (int k = n - 1; k >= 0; --k) {
            const int si = (int) (uint32_t) srt[k];
            const bm2_seed &s = cs[si];
            alignas(16) bm2_alnreg_t a = bm2_alnreg_t();   // value-initialised: the padding bytes are part of the output too
            a.rb = a.re = BM2_H0; a.qb = a.qe = BM2_H0; a.rid = c.rid; a.c = 0;
            a.score = a.truesc = -1; a.sub = a.alt_sc = a.csub = a.sub_n = 0; a.w = p.w; a.seedcov = 0;
            a.secondary = a.secondary_all = 0; a.seedlen0 = s.len; a.n_comp_is_alt = 0; a.frac_rep = c.frac_rep; a.hash = 0; a.flg = 0;
            a.pad0_ = a.pad1_ = a.pad2_ = 0;
            const int ai = n_reg;
            if (s.qbeg) {
                ExtJobRec j; j.qlen = s.qbeg; j.tlen = (int) (s.rbeg - rmax0); j.toff = s.rbeg - 1; j.qoff = read_code_off + s.qbeg - 1;
                j.h0 = s.len * p.a; j.tstride = -1; j.qstride = -1; j._pad = 0;
                left[nl] = j; left_reg[nl] = (int32_t) (reg_base + ai); ++nl;
                a.qb = s.qbeg; a.rb = s.rbeg;
            } else { a.score = a.truesc = s.len * p.a; a.qb = 0; a.rb = s.rbeg; }
            if (s.qbeg + s.len != l_query) {
                const int64_t qe = s.qbeg + s.len, re = s.rbeg + s.len - rmax0;
                ExtJobRec j; j.qlen = (int) (l_query - qe); j.tlen = (int) (rmax1 - rmax0 - re); j.toff = rmax0 + re; j.qoff = read_code_off + qe;
                j.h0 = BM2_H0; j.tstride = 1; j.qstride = 1; j._pad = 0;
                right[nr] = j; right_reg[nr] = (int32_t) (reg_base + ai); ++nr;
                a.qe = (int) qe; a.re = rmax0 + re;
            } else {
                a.qe = l_query; a.re = s.rbeg + s.len;
                seedcov_d(a, cs, n);
            }
            reg_copy(&regs[ai], &a); reg_chain[ai] = (int32_t) (chain_base + ci); reg_seed[ai] = si;
            if (state) state[ai] = (!s.qbeg && s.qbeg + s.len == l_query) ? EXT_DONE : (k == n - 1 ? EXT_NEED : EXT_TODO);
            ++n_reg;
        }
    }
}

// Fold of one finished extension (src/bwamem.cpp:2485-2521 left, :2705-2740 right).
// Returns true when accepted; false => the job must be re-run with the doubled band.
BM2_HD bool ext_fold_d(const ExtParams &p, bm2_alnreg_t &a, int is_right, int h0, int score, int qle, int tle, int gtle, int gscore,
                       int max_off, int w, int last_try, int l_query, const bm2_seed *chain_seeds, int n_chain_seeds)
{
    const int prev = a.score;
    a.score = score;
    if (!(a.score == prev || max_off < (w >> 1) + (w >> 2) || last_try)) return false;
    if (!is_right) {
        if (gscore <= 0 || gscore <= a.score - p.pen_clip5) { a.qb -= qle; a.rb -= tle; a.truesc = a.score; }
        else { a.qb = 0; a.rb -= gtle; a.truesc = gscore; }
    } else {
        if (gscore <= 0 || gscore <= a.score - p.pen_clip3) { a.qe += qle; a.re += tle; a.truesc += a.score - h0; }
        else { a.qe = l_query; a.re += gtle; a.truesc += gscore - h0; }
    }
    a.w = a.w > w ? a.w : w;
    seedcov_d(a, chain_seeds, n_chain_seeds);
    return true;
}

// The fields of a reg the post-filter scans, 32 B instead of the 112-B mem_alnreg_t (the scan is O(regs x seeds)).
struct PfBox { int64_t rb, re; int32_t qb, qe, seedlen0, w; };

BM2_HD PfBox pf_box_d(const bm2_alnreg_t &a) {
    PfBox b; b.rb = a.rb; b.re = a.re; b.qb = a.qb; b.qe = a.qe; b.seedlen0 = a.seedlen0; b.w = a.w;
    return b;
}

// The post-filter's test of seed s against the box of one earlier reg (src/bwamem.cpp:2964-2977): 0 = the reg is purged (not
// counted), 1 = counted (v++), 2 = s lies on the reg's diagonal band (the scan stops).
BM2_HD int pf_box_kind_d(const ExtParams &p, const bm2_seed &s, const PfBox &q, int l_query) {
    if (q.qb == -1 && q.qe == -1) return 0;
    if (s.rbeg < q.rb || s.rbeg + s.len > q.re || s.qbeg < q.qb || s.qbeg + s.len > q.qe) return 1;
    if (s.len - q.seedlen0 > .1 * l_query) return 1;
    int64_t rd; int qd, w, max_gap;
    qd = s.qbeg - q.qb; rd = s.rbeg - q.rb;
    max_gap = cal_max_gap_d(p, qd < rd ? qd : (int) rd);
    w = max_gap < q.w ? max_gap : q.w;
    if (qd - rd < w && rd - qd < w) return 2;
    qd = q.qe - (s.qbeg + s.len); rd = q.re - (s.rbeg + s.len);
    max_gap = cal_max_gap_d(p, qd < rd ? qd : (int) rd);
    w = max_gap < q.w ? max_gap : q.w;
    if (qd - rd < w && rd - qd < w) return 2;
    return 1;
}

// One step of 32 boxes of the scan in pf_seed_purged_d, resolved from the step's counted (kind 1) and hit (kind 2) masks, bit j = box j of
// the step: advances v exactly as the sequential loop `for (i = 0; i < n_reg && v < lim; ++i)` does over those boxes and returns true
// when that loop ends inside the step (a hit while v < lim, or v reaching lim).  Needs v < lim on entry.  The warp scans resolve their
// ballots with it.
BM2_HD bool pf_scan_step_d(uint32_t counted, uint32_t hit, int &v, int lim) {
    if (hit) {
        const int at = v + BM2_POPC32(counted & ((hit & (0u - hit)) - 1u));    // counted boxes before the first hit
        if (at < lim) { v = at; return true; }
    }
    v += BM2_POPC32(counted);
    if (v >= lim) { v = lim; return true; }
    return false;
}

// The second half of the decision (src/bwamem.cpp:2978-2986), for a seed that lies inside an earlier reg: it is kept only when a
// long seed of the same chain visited before it (srt2[k+1..n), purged ones -1) overlaps it on another diagonal.
BM2_HD bool pf_chain_overlap_d(const bm2_seed *cs, int n, const int32_t *srt2, int k, const bm2_seed &s) {
    for (int vv = k + 1; vv < n; ++vv) {
        if (srt2[vv] < 0) continue;
        const bm2_seed &t = cs[srt2[vv]];
        if (t.len < s.len * .95) continue;
        if (s.qbeg <= t.qbeg && s.qbeg + s.len - t.qbeg >= s.len >> 2 && t.qbeg - s.qbeg != t.rbeg - s.rbeg) return true;
        if (t.qbeg <= s.qbeg && t.qbeg + t.len - s.qbeg >= s.len >> 2 && s.qbeg - t.qbeg != s.rbeg - t.rbeg) return true;
    }
    return false;
}

// Post-filter decision of seed srt2[k] of chain cs[0..n) (src/bwamem.cpp:2957-2986): true = purged.  box[0..): the boxes of the read's
// regs in creation order, purged ones with qb = qe = -1; lim: the number of regs kept so far.  The scan stops after lim counted boxes,
// so it reads only the boxes of regs created before this seed's own.
BM2_HD bool pf_seed_purged_d(const ExtParams &p, const bm2_seed *cs, int n, const int32_t *srt2, int k, int l_query, const PfBox *box,
                             int n_reg, int lim)
{
    const bm2_seed s = cs[srt2[k]];
    int v = 0;
    for (int i = 0; i < n_reg && v < lim; ++i) {
        const int kind = pf_box_kind_d(p, s, box[i], l_query);
        if (kind == 2) break;
        v += kind;
    }
    return v < lim && !pf_chain_overlap_d(cs, n, srt2, k, s);
}

// Post-filter of one read (src/bwamem.cpp:2895-2989).  regs[0..n_reg) in creation order;
// reg_seed[i] = seed index (within its chain) of reg i; srt2: int scratch of >= max chain length;
// box: scratch of n_reg entries.
BM2_HD void ext_postfilter_read_d(const ExtParams &p, const bm2_chain *chains, int n_chain, const bm2_seed *seeds, int l_query,
                                  bm2_alnreg_t *regs, int n_reg, const int32_t *reg_seed, int32_t *srt2, PfBox *box)
{
    for (int i = 0; i < n_reg; ++i) box[i] = pf_box_d(regs[i]);
    int lim = 0, base = 0;
    for (int ci = 0; ci < n_chain; ++ci) {
        const bm2_chain &c = chains[ci];
        const bm2_seed *cs = seeds + c.seed_off;
        const int n = c.n_seeds;
        if (n == 0) continue;
        for (int k = n - 1; k >= 0; --k) srt2[k] = reg_seed[base + (n - 1 - k)];
        for (int k = n - 1; k >= 0; --k) {
            if (pf_seed_purged_d(p, cs, n, srt2, k, l_query, box, n_reg, lim)) {
                const int ai = base + (n - 1 - k);
                regs[ai].qb = regs[ai].qe = -1;
                box[ai].qb = box[ai].qe = -1;
                srt2[k] = -1;
                continue;
            }
            lim++;
        }
        base += n;
    }
}

// ---- lazy extension: extend only the seeds the post-filter keeps ----------------------------------------------------------------
// Whether the post-filter purges a seed depends on the seeds and on the boxes of the EARLIER KEPT regs only (pf_seed_purged_d), so
// a walk in the post-filter's order can decide every seed up to the first kept one whose reg has not been extended yet, and the
// purged seeds before it need no extension at all.  The post-filter of the tail stays the decision that counts: it purges the
// same seeds again, and every reg it keeps has been extended.

// Where the walk of one read stands: chain ci, seed k of its post-filter order (-1: the chain's srt2 is not set up yet), the number
// of kept regs before it, and the reg index of the chain's first reg.  ci == n_chain: the read is decided.
struct PfCursor { int32_t ci, k, lim, base; };

// Resumes the post-filter walk of one read at `cur` (start: {0, -1, 0, 0}).  Purged seeds are marked in srt2 (and, when not extended,
// EXT_SKIP); the box of every decided reg is written for the later decisions.  Stops at the first kept seed whose reg is not extended,
// marks it EXT_NEED and returns false; returns true when every seed of the read is decided.  regs / state / srt2 / box: the read's
// stripes; srt2 and box must be kept between calls.
BM2_HD bool ext_walk_read_d(const ExtParams &p, const bm2_chain *chains, int n_chain, const bm2_seed *seeds, int l_query,
                            const bm2_alnreg_t *regs, int n_reg, const int32_t *reg_seed, uint8_t *state, int32_t *srt2, PfBox *box,
                            PfCursor &cur)
{
    int ci = cur.ci, k = cur.k, lim = cur.lim, base = cur.base;
    for (; ci < n_chain; ++ci, k = -1) {
        const bm2_chain &c = chains[ci];
        const bm2_seed *cs = seeds + c.seed_off;
        const int n = c.n_seeds;
        if (n == 0) continue;
        if (k < 0) {
            for (int kk = n - 1; kk >= 0; --kk) srt2[kk] = reg_seed[base + (n - 1 - kk)];
            k = n - 1;
        }
        for (; k >= 0; --k) {
            const int ai = base + (n - 1 - k);
            if (pf_seed_purged_d(p, cs, n, srt2, k, l_query, box, n_reg, lim)) {
                box[ai].qb = box[ai].qe = -1;
                srt2[k] = -1;
                if (state[ai] != EXT_DONE) state[ai] = EXT_SKIP;
                continue;
            }
            if (state[ai] != EXT_DONE) {
                state[ai] = EXT_NEED;
                cur.ci = ci; cur.k = k; cur.lim = lim; cur.base = base;
                return false;
            }
            box[ai] = pf_box_d(regs[ai]);
            lim++;
        }
        base += n;
    }
    cur.ci = ci; cur.k = -1; cur.lim = lim; cur.base = base;
    return true;
}

// score-only ksw_global2 (src/ksw.cpp:558-668) of query[0..qlen) vs target[0..tlen); sequences are
// read through base + k*stride so that the reverse-strand case needs no copies; he: 2*(qlen+1) ints.
BM2_HD int global_score_d(int qlen, const uint8_t *qp, int qstride, int tlen, const uint8_t *tp, int tstride, const int8_t *mat,
                          int o_del, int e_del, int o_ins, int e_ins, int w, int32_t *he)
{
    const int MINUS_INF = -0x40000000;
    const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
#if defined(BM2_TRACE_GLOBAL_SCORE) && !defined(__CUDA_ARCH__)
    BM2_TRACE_GLOBAL_SCORE(qlen, tlen, w);
#endif
    int32_t *H = he, *E = he + (qlen + 1);
    H[0] = 0; E[0] = MINUS_INF;
    int j;
    for (j = 1; j <= qlen && j <= w; ++j) { H[j] = -(o_ins + e_ins * j); E[j] = MINUS_INF; }
    for (; j <= qlen; ++j) H[j] = E[j] = MINUS_INF;
    for (int i = 0; i < tlen; ++i) {
        int32_t f = MINUS_INF, h1;
        const int beg = i > w ? i - w : 0;
        const int end = i + w + 1 < qlen ? i + w + 1 : qlen;
        const int tb = tp[(long long) i * tstride];
        h1 = beg == 0 ? -(o_del + e_del * (i + 1)) : MINUS_INF;
        auto cell = [&](int32_t m, int32_t e, const int qb, int32_t &hs, int32_t &es) {
            hs = h1;
            m += mat[tb * 5 + qb];
            int32_t h = m >= e ? m : e;
            h = h >= f ? h : f;
            h1 = h;
            int32_t t = m - oe_del;
            e -= e_del; e = e > t ? e : t;
            es = e;
            t = m - oe_ins;
            f -= e_ins; f = f > t ? f : t;
        };
        // four cells per trip, their loads first (the rows live in per-thread global memory: see global_align_d in cigar_device.cuh)
        for (j = beg; j + 4 <= end; j += 4) {
            const int32_t m0 = H[j], m1 = H[j + 1], m2 = H[j + 2], m3 = H[j + 3], e0 = E[j], e1 = E[j + 1], e2 = E[j + 2], e3 = E[j + 3];
            const int q0 = qp[(long long) j * qstride], q1 = qp[(long long) (j + 1) * qstride], q2 = qp[(long long) (j + 2) * qstride],
                      q3 = qp[(long long) (j + 3) * qstride];
            int32_t hs0, hs1, hs2, hs3, es0, es1, es2, es3;
            cell(m0, e0, q0, hs0, es0); cell(m1, e1, q1, hs1, es1); cell(m2, e2, q2, hs2, es2); cell(m3, e3, q3, hs3, es3);
            H[j] = hs0; H[j + 1] = hs1; H[j + 2] = hs2; H[j + 3] = hs3;
            E[j] = es0; E[j + 1] = es1; E[j + 2] = es2; E[j + 3] = es3;
        }
        for (; j < end; ++j) {
            int32_t hs, es;
            cell(H[j], E[j], qp[(long long) j * qstride], hs, es);
            H[j] = hs; E[j] = es;
        }
        H[end] = h1; E[end] = MINUS_INF;
    }
    return H[qlen];
}

// bwa_gen_cigar2 with n_cigar == NM == NULL (src/bwa.cpp:260-347)
BM2_HD bool gen_score_d(const ContigView &cv, const ExtParams &p, const uint8_t *ref, int w_, int l_query, const uint8_t *query,
                        int64_t rb, int64_t re, int32_t *he, int *score)
{
    const int64_t l_pac = cv.l_pac;
    if (l_query <= 0 || rb >= re || (rb < l_pac && re > l_pac)) return false;
    if (re > (l_pac << 1) || rb < 0) return false;
    const int64_t rlen = re - rb;
    const bool rev = rb >= l_pac;
    const uint8_t *qp = rev ? query + (l_query - 1) : query; const int qs = rev ? -1 : 1;
    const uint8_t *tp = rev ? ref + (re - 1) : ref + rb;      const int ts = rev ? -1 : 1;
    if (l_query == rlen && w_ == 0) {
        int sc = 0;
        for (int i = 0; i < l_query; ++i) sc += p.mat[tp[(long long) i * ts] * 5 + qp[(long long) i * qs]];
        *score = sc;
    } else {
        int max_ins = (int) ((double) (((l_query + 1) >> 1) * p.mat[0] - p.o_ins) / p.e_ins + 1.);
        int max_del = (int) ((double) (((l_query + 1) >> 1) * p.mat[0] - p.o_del) / p.e_del + 1.);
        int max_gap = max_ins > max_del ? max_ins : max_del;
        max_gap = max_gap > 1 ? max_gap : 1;
        int diff = (int) (rlen - l_query); if (diff < 0) diff = -diff;
        int w = (max_gap + diff + 1) >> 1;
        w = w < w_ ? w : w_;
        const int min_w = diff + 3;
        w = w > min_w ? w : min_w;
        *score = global_score_d(l_query, qp, qs, (int) rlen, tp, ts, p.mat, p.o_del, p.e_del, p.o_ins, p.e_ins, w, he);
    }
    return true;
}

// mem_patch_reg (src/bwamem.cpp:175-234)
BM2_HD int patch_reg_d(const ContigView &cv, const ExtParams &p, const uint8_t *ref, const uint8_t *query, const bm2_alnreg_t *a,
                       const bm2_alnreg_t *b, int32_t *he, int *_w)
{
    int w, score = 0, q_s, r_s;
    double r;
    if (query == 0) return 0;                                   // mem_patch_reg without a query (mate rescue's dedup, src/bwamem.cpp:179)
    if (a->rb < cv.l_pac && b->rb >= cv.l_pac) return 0;
    if (a->qb >= b->qb || a->qe >= b->qe || a->re >= b->re) return 0;
    w = (int) ((a->re - b->rb) - (a->qe - b->qb));
    w = w > 0 ? w : -w;
    r = (double) (a->re - b->rb) / (b->re - a->rb) - (double) (a->qe - b->qb) / (b->qe - a->qb);
    r = r > 0. ? r : -r;
    if (a->re < b->rb || a->qe < b->qb) {
        if (w > p.w << 1 || r >= 0.05f) return 0;
    } else if (w > p.w << 2 || r >= 0.05f * 2) return 0;
    w += a->w + b->w;
    w = w < p.w << 2 ? w : p.w << 2;
    if (!gen_score_d(cv, p, ref, w, b->qe - a->qb, query + a->qb, a->rb, b->re, he, &score)) score = 0;
    q_s = (int) ((double) (b->qe - a->qb) / ((b->qe - b->qb) + (a->qe - a->qb)) * (b->score + a->score) + .499);
    r_s = (int) ((double) (b->re - a->rb) / ((b->re - b->rb) + (a->re - a->rb)) * (b->score + a->score) + .499);
    if ((double) score / (q_s > r_s ? q_s : r_s) < 0.90f) return 0;
    *_w = w;
    return score;
}

// a[i] <- a[idx[i]] in place (cycle following: every 112-byte record moves once); idx is destroyed
BM2_HD void permute_regs_d(bm2_alnreg_t *a, int32_t *idx, int n) {
    for (int i = 0; i < n; ++i) {
        if (idx[i] < 0 || idx[i] == i) { continue; }
        alignas(16) bm2_alnreg_t tmp;
        reg_copy(&tmp, &a[i]);
        int j = i;
        for (;;) {
            const int src = idx[j];
            idx[j] = -1;
            if (src == i) { reg_copy(&a[j], &tmp); break; }
            reg_copy(&a[j], &a[src]);
            j = src;
        }
    }
}

// the dedup / patch scan of mem_sort_dedup_patch (src/bwamem.cpp:302-333) over the regs sorted by `re` (n_comp already 1)
BM2_HD void sort_dedup_scan_d(const ContigView &cv, const ExtParams &p, const uint8_t *ref, const uint8_t *query, int n, bm2_alnreg_t *a, int32_t *he)
{
    int i, j;
    for (i = 1; i < n; ++i) {
        bm2_alnreg_t *pp = &a[i];
        if (pp->rid != a[i - 1].rid || pp->rb >= a[i - 1].re + p.max_chain_gap) continue;
        for (j = i - 1; j >= 0 && pp->rid == a[j].rid && pp->rb < a[j].re + p.max_chain_gap; --j) {
            bm2_alnreg_t *q = &a[j];
            int64_t or_, oq, mr, mq;
            int score, w;
            if (q->qe == q->qb) continue;
            or_ = q->re - pp->rb;
            oq = q->qb < pp->qb ? q->qe - pp->qb : pp->qe - q->qb;
            mr = q->re - q->rb < pp->re - pp->rb ? q->re - q->rb : pp->re - pp->rb;
            mq = q->qe - q->qb < pp->qe - pp->qb ? q->qe - q->qb : pp->qe - pp->qb;
            if (or_ > p.mask_level_redun * mr && oq > p.mask_level_redun * mq) {
                if (pp->score < q->score) { pp->qe = pp->qb; break; }
                else q->qe = q->qb;
            } else if (q->rb < pp->rb && (score = patch_reg_d(cv, p, ref, query, q, pp, he, &w)) > 0) {
                reg_set_n_comp_d(*pp, reg_n_comp_d(*pp) + reg_n_comp_d(*q) + 1);
                pp->seedcov = pp->seedcov > q->seedcov ? pp->seedcov : q->seedcov;
                pp->sub = pp->sub > q->sub ? pp->sub : q->sub;
                pp->csub = pp->csub > q->csub ? pp->csub : q->csub;
                pp->qb = q->qb; pp->rb = q->rb;
                pp->truesc = pp->score = score;
                pp->w = w;
                q->qb = q->qe;
            }
        }
    }
}

// mem_sort_dedup_patch (src/bwamem.cpp:292-353) on the regs of one read; he: 2*(l_query+1) ints; idx: n ints.
// The two ks_introsort calls run on an index array (same comparisons, same swaps => same permutation as sorting
// the records) and the records are permuted once.
// keys: n entries of 16 bytes; the comparators read these compact copies of the sort fields instead of the 112-byte records.
struct TailSortKey { int64_t r; int32_t score, qb; };
BM2_HD int sort_dedup_patch_d(const ContigView &cv, const ExtParams &p, const uint8_t *ref, const uint8_t *query, int n,
                              bm2_alnreg_t *a, int32_t *he, int32_t *idx, TailSortKey *keys)
{
    int m, i, j;
    if (n <= 1) return n;
    for (i = 0; i < n; ++i) { idx[i] = i; keys[i].r = a[i].re; }
    {
        const TailSortKey *rk = keys;
        ks_introsort_d(idx, (long) n, [rk](int x, int y) { return rk[x].r < rk[y].r; });
    }
    permute_regs_d(a, idx, n);
    for (i = 0; i < n; ++i) reg_set_n_comp_d(a[i], 1);
    sort_dedup_scan_d(cv, p, ref, query, n, a, he);
    for (i = 0, m = 0; i < n; ++i)
        if (a[i].qe > a[i].qb) { if (m != i) reg_copy(&a[m++], &a[i]); else ++m; }
    n = m;
    for (i = 0; i < n; ++i) { idx[i] = i; keys[i].r = a[i].rb; keys[i].score = a[i].score; keys[i].qb = a[i].qb; }
    {
        const TailSortKey *rk = keys;
        ks_introsort_d(idx, (long) n, [rk](int xi, int yi) {
            const TailSortKey x = rk[xi], y = rk[yi];
            return x.score > y.score || (x.score == y.score && (x.r < y.r || (x.r == y.r && x.qb < y.qb)));
        });
    }
    permute_regs_d(a, idx, n);
    for (i = 1; i < n; ++i)
        if (a[i].score == a[i - 1].score && a[i].rb == a[i - 1].rb && a[i].qb == a[i - 1].qb) a[i].qe = a[i].qb;
    for (i = 1, m = 1; i < n; ++i)
        if (a[i].qe > a[i].qb) { if (m != i) reg_copy(&a[m++], &a[i]); else ++m; }
    return m;
}

// Tail of mem_kernel2_core for one read (src/bwamem.cpp:1141-1169): drop purged regs, sort/dedup/
// patch, ALT marking.  Returns the final reg count (regs compacted in place).
BM2_HD int ext_tail_read_d(const ContigView &cv, const ExtParams &p, const uint8_t *ref, const uint8_t *query, bm2_alnreg_t *regs,
                           int n_reg, int32_t *he, int32_t *idx, TailSortKey *keys)
{
    int m = 0;
    for (int i = 0; i < n_reg; ++i)
        if (regs[i].qe > regs[i].qb) { if (m != i) reg_copy(&regs[m++], &regs[i]); else ++m; }
    m = sort_dedup_patch_d(cv, p, ref, query, m, regs, he, idx, keys);
    for (int i = 0; i < m; ++i)
        if (regs[i].rid >= 0 && cv.ann_alt && cv.ann_alt[regs[i].rid]) reg_set_is_alt_d(regs[i], 1);
    return m;
}

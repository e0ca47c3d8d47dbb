// fm_device.cuh — FM-index search over the 2bit.64 Occ table (device logic, one read per thread).
//
// Replaces FMI_search::backwardExt (reference src/FMI_search.cpp:1025-1052), the three SMEM passes
// getSMEMsAllPosOneThread / getSMEMsOnePosOneThread / bwtSeedStrategyAllPosOneThread
// (src/FMI_search.cpp:496-812) as orchestrated by mem_collect_smem (src/bwamem.cpp:626-804), and
// the compressed-SA walk call_one_step (src/FMI_search.cpp:1202-1255).
//
// GPU shape: the search of one read is a chain of ~600 dependent interval extensions, each touching
// two random 64-byte checkpoints of a multi-GB table, so it is HBM-latency/sector bound.  One read
// per thread; the whole three-pass search is ONE state machine with a SINGLE extension call site, so
// the 32 lanes of a warp stay converged at the two checkpoint loads no matter which pass / direction
// each lane is in (a straight port of the nested loops would serialise the lanes).
#pragma once
#include "hd.h"
#include "bm2_b200.h"

// layout 0: the checkpoints as the index file holds them, {cp_count[4]; one_hot_bwt_str[4]} (CP_OCC, src/FMI_search.h:54-58).
// layout 1 (device only, made in place at upload by occ_relayout_kernel, pipeline.cu): the same eight words ordered
// {cnt0, cnt1, bits0, bits1 | cnt2, cnt3, bits2, bits3}: an interval extension by base a needs base a and ONE partner base, and the partner
// is always in a's half ({0,1} or {2,3}, see fm_backward_ext), so one checkpoint costs ONE 32-byte sector (two 128-bit loads, fm_ld256)
// instead of both sectors of the 64-byte line through four 8-byte loads.
struct FmIndexView {
    const bm2_cp_occ *cp_occ;
    const int8_t *sa_ms;
    const uint32_t *sa_ls;
    int64_t count[5];
    int64_t sentinel;
    int layout = 0;
    // Reference text (2 * l_pac codes, forward || reverse complement) for the unique-interval shortcut of fm_forward; null = off (exact `l`
    // values: the staged bm2_collect_smems entry and the host builds)
    const uint8_t *text = nullptr;
    int64_t text_len = 0;
};

#if defined(__CUDA_ARCH__)
// 32 bytes (one aligned sector) by two 128-bit loads on the read-only path: sm_90 has no 256-bit load.  Both halves are issued before
// either is used and lie in the same sector, so the second can be served by the first one's L1 fill (not measured on its own; the
// gather probe of bench.py, shapes 1 and 2, reports the request rate of this access).
BM2_D void fm_ld256(const void *p, uint64_t &a, uint64_t &b, uint64_t &c, uint64_t &d) {
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%4];\n\t"
                 "ld.global.nc.v2.u64 {%2,%3}, [%4+16];" : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p));
}
#endif

struct FmIv { int64_t k, l, s; };

// count[] lives in kernel-parameter space: select instead of indexing dynamically (no local-memory copy)
BM2_HD int64_t fm_count(const FmIndexView &fm, int a) {
    return a == 0 ? fm.count[0] : a == 1 ? fm.count[1] : a == 2 ? fm.count[2] : a == 3 ? fm.count[3] : fm.count[4];
}

struct FmOcc4 { int64_t c[4]; };

// Occ(b, pp) for the four bases from one 64-byte checkpoint (GET_OCC, src/FMI_search.h:66-73).
BM2_HD FmOcc4 fm_occ4(const FmIndexView &fm, int64_t pp) {
    const bm2_cp_occ *e = fm.cp_occ + (pp >> 6);
    FmOcc4 r;
#if defined(__CUDA_ARCH__)
    const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(e);
    ulonglong2 c01 = __ldg(p), c23 = __ldg(p + 1), b01 = __ldg(p + 2), b23 = __ldg(p + 3);
    if (fm.layout) { const ulonglong2 t = c23; c23 = b01; b01 = t; }          // {c01, b01, c23, b23} in memory
    uint64_t cnt[4] = {c01.x, c01.y, c23.x, c23.y}, bits[4] = {b01.x, b01.y, b23.x, b23.y};
#else
    uint64_t cnt[4], bits[4];
    for (int b = 0; b < 4; ++b) { cnt[b] = (uint64_t) e->cp_count[b]; bits[b] = e->one_hot_bwt_str[b]; }
#endif
    const int y = (int) (pp & 63);
    const uint64_t mask = y ? ~0ULL << (64 - y) : 0ULL;      // top y bits (src/FMI_search.cpp:386-394)
#pragma unroll
    for (int b = 0; b < 4; ++b) r.c[b] = (int64_t) cnt[b] + BM2_POPC64(bits[b] & mask);
    return r;
}

// backwardExt (src/FMI_search.cpp:1025-1052): 2 checkpoints = 128 algorithmic bytes.
// Only base `a` and ONE other base are counted: the four per-base interval sizes and the sentinel sum
// to s (every BWT row of [k, k+s) holds one of the four bases or the sentinel), so
//   l_0 = l + s - s_0,  l_1 = l + s - s_0 - s_1,  l_2 = l + [sentinel] + s_3,  l_3 = l + [sentinel]
// are the reference's l[a] exactly, with half the popcounts and 8-byte instead of 16-byte loads.
BM2_HD FmIv fm_backward_ext(const FmIndexView &fm, const FmIv &in, int a) {
    const int64_t p1 = in.k, p2 = in.k + in.s;
#if defined(BM2_TRACE_EXT) && !defined(__CUDA_ARCH__)
    BM2_TRACE_EXT(p1, p2, in.s);                                  // access-locality studies (scripts/study_smem_locality.py)
#endif
    const bm2_cp_occ *e1 = fm.cp_occ + (p1 >> 6), *e2 = fm.cp_occ + (p2 >> 6);
    const int b2 = a == 1 ? 0 : (a == 2 ? 3 : a);                  // the one other base that is needed
    const int y1 = (int) (p1 & 63), y2 = (int) (p2 & 63);
    const uint64_t m1 = y1 ? ~0ULL << (64 - y1) : 0ULL, m2 = y2 ? ~0ULL << (64 - y2) : 0ULL;
#if defined(__CUDA_ARCH__)
    if (fm.layout) {
        // device layout: the half {2h, 2h+1} of a checkpoint is one 32-byte sector {cnt, cnt, bits, bits}; both ends of a small
        // interval usually lie in the same checkpoint, then the second load is skipped
        const int h = a >> 1, odd = a & 1;
        const char *q1 = reinterpret_cast<const char *>(e1) + h * 32, *q2 = reinterpret_cast<const char *>(e2) + h * 32;
        uint64_t c10, c11, b10, b11, c20, c21, b20, b21;
        fm_ld256(q1, c10, c11, b10, b11);
        if (q2 != q1) fm_ld256(q2, c20, c21, b20, b21);
        else { c20 = c10; c21 = c11; b20 = b10; b21 = b11; }
        const int64_t o10 = (int64_t) c10 + __popcll(b10 & m1), o11 = (int64_t) c11 + __popcll(b11 & m1);
        const int64_t o20 = (int64_t) c20 + __popcll(b20 & m2), o21 = (int64_t) c21 + __popcll(b21 & m2);
        const int64_t s0 = o20 - o10, s1 = o21 - o11;
        const int64_t sa = odd ? s1 : s0, sb = odd ? s0 : s1;          // partner of base 1 is base 0, of base 2 is base 3
        const int64_t sent = (in.k <= fm.sentinel && in.k + in.s > fm.sentinel) ? 1 : 0;
        FmIv r;
        r.k = fm_count(fm, a) + (odd ? o11 : o10);
        r.s = sa;
        r.l = a == 0 ? in.l + in.s - sa : a == 1 ? in.l + in.s - sb - sa : a == 2 ? in.l + sent + sb : in.l + sent;
        return r;
    }
#endif
    const int64_t o1a = (int64_t) BM2_LDG64(&e1->cp_count[a]) + BM2_POPC64(BM2_LDG64(&e1->one_hot_bwt_str[a]) & m1);
    const int64_t o2a = (int64_t) BM2_LDG64(&e2->cp_count[a]) + BM2_POPC64(BM2_LDG64(&e2->one_hot_bwt_str[a]) & m2);
    const int64_t o1b = (int64_t) BM2_LDG64(&e1->cp_count[b2]) + BM2_POPC64(BM2_LDG64(&e1->one_hot_bwt_str[b2]) & m1);
    const int64_t o2b = (int64_t) BM2_LDG64(&e2->cp_count[b2]) + BM2_POPC64(BM2_LDG64(&e2->one_hot_bwt_str[b2]) & m2);
    const int64_t sa = o2a - o1a, sb = o2b - o1b;
    const int64_t sent = (in.k <= fm.sentinel && in.k + in.s > fm.sentinel) ? 1 : 0;
    FmIv r;
    r.k = fm_count(fm, a) + o1a;
    r.s = sa;
    r.l = a == 0 ? in.l + in.s - sa : a == 1 ? in.l + in.s - sb - sa : a == 2 ? in.l + sent + sb : in.l + sent;
    return r;
}

// SA of one BWT row: LF-walk to a sampled row (call_one_step; returns 0 on the sentinel, :1230-1233)
BM2_HD int64_t fm_sa_of_row(const FmIndexView &fm, int64_t r, int *lf_steps, int64_t at_sentinel = 0) {
    int64_t steps = 0;
    while (r & 7) {
        const bm2_cp_occ *e = fm.cp_occ + (r >> 6);
        const int y = 63 - (int) (r & 63);
#if defined(__CUDA_ARCH__)
        const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(e);
        ulonglong2 c01 = __ldg(p), c23 = __ldg(p + 1), b01 = __ldg(p + 2), b23 = __ldg(p + 3);
        if (fm.layout) { const ulonglong2 t = c23; c23 = b01; b01 = t; }      // {c01, b01, c23, b23} in memory
        uint64_t cnt[4] = {c01.x, c01.y, c23.x, c23.y}, bits[4] = {b01.x, b01.y, b23.x, b23.y};
#else
        uint64_t cnt[4], bits[4];
        for (int b = 0; b < 4; ++b) { cnt[b] = (uint64_t) e->cp_count[b]; bits[b] = e->one_hot_bwt_str[b]; }
#endif
        int b = ((bits[0] >> y) & 1) ? 0 : ((bits[1] >> y) & 1) ? 1 : ((bits[2] >> y) & 1) ? 2 : ((bits[3] >> y) & 1) ? 3 : 4;
        if (b == 4) { if (lf_steps) *lf_steps += (int) steps; return at_sentinel; }
        const int yy = (int) (r & 63);
        const uint64_t mask = yy ? ~0ULL << (64 - yy) : 0ULL;
        uint64_t cb = b == 0 ? cnt[0] : b == 1 ? cnt[1] : b == 2 ? cnt[2] : cnt[3];
        uint64_t bb = b == 0 ? bits[0] : b == 1 ? bits[1] : b == 2 ? bits[2] : bits[3];
        r = fm_count(fm, b) + (int64_t) cb + BM2_POPC64(bb & mask);
        ++steps;
    }
    if (lf_steps) *lf_steps += (int) steps;
#if defined(__CUDA_ARCH__)
    int64_t sa = ((int64_t) __ldg(fm.sa_ms + (r >> 3)) << 32) + (int64_t) __ldg(fm.sa_ls + (r >> 3));
#else
    int64_t sa = ((int64_t) fm.sa_ms[r >> 3] << 32) + (int64_t) fm.sa_ls[r >> 3];
#endif
    return sa + steps;
}

// Text position of BWT row r (the true suffix-array value), or -1 when the LF walk meets the sentinel (fm_sa_of_row mirrors the
// reference's quirk there and returns 0, which is not a position)
BM2_HD int64_t fm_text_pos_of_row(const FmIndexView &fm, int64_t r) { return fm_sa_of_row(fm, r, nullptr, -1); }

// One entry of the per-read interval list of the SMEM search (prevArray, src/FMI_search.cpp:510).
struct FmPrev { int64_t k, l, s; int32_t m, n; };

struct SmemParams {
    int min_seed_len;        // opt->min_seed_len
    int split_len;           // (int)(min_seed_len * split_factor + .499)   (src/bwamem.cpp:640)
    int split_width;         // opt->split_width
    int max_mem_intv;        // opt->max_mem_intv (0 disables pass 3)
};

struct QPlain {                    // read codes straight from memory
    const uint8_t *p;
    BM2_HD int operator()(int j) const { return p[j]; }
};

// Pass 3 alone (bwtSeedStrategyAllPosOneThread, src/FMI_search.cpp:726-812): forward-only, no interval list, so it
// runs as its own lean kernel (few registers, one hot loop) next to the pass-1/2 automaton.
template <class Emit, class Q>
BM2_HD void fm_smem_pass3(const FmIndexView &fm, const Q &q, int len, const SmemParams &sp, Emit &emit, unsigned &n_ext)
{
    if (len <= 0 || sp.max_mem_intv <= 0) return;
    int x = 0, j = 0, next_x = 0;
    bool searching = false;
    FmIv cur; cur.k = cur.l = cur.s = 0;
    for (;;) {
        // control: find the next extension to do
        bool need = false;
        int base = 0;
        while (!need) {
            if (!searching) {
                if (x >= len) return;
                next_x = x + 1;
                const int a = q(x);
                if (a > 3) { x = next_x; continue; }
                cur.k = fm_count(fm, a); cur.l = fm_count(fm, 3 - a); cur.s = fm_count(fm, a + 1) - cur.k;
                j = x + 1; searching = true;
            }
            if (j >= len) { x = next_x; searching = false; continue; }
            next_x = j + 1;
            const int a = q(j);
            if (a > 3) { x = next_x; searching = false; continue; }
            base = 3 - a; need = true;
        }
        BM2_SYNCWARP();
        FmIv req; req.k = cur.l; req.l = cur.k; req.s = cur.s;
        FmIv r = fm_backward_ext(fm, req, base);
        ++n_ext;
        cur.k = r.l; cur.l = r.k; cur.s = r.s;
        if (cur.s < sp.max_mem_intv && j - x + 1 >= sp.min_seed_len + 1) {
            if (cur.s > 0) emit(x, j, cur.k, cur.l, cur.s);
            x = next_x; searching = false;
        } else ++j;
    }
}

// ---- passes 1 and 2, split into HOMOGENEOUS phases ---------------------------------------------------------------
// getSMEMsOnePosOneThread (src/FMI_search.cpp:496-670) is a forward phase (extend right from x, remember the
// interval whenever its size changes) followed by a backward phase (extend all remembered intervals to the left,
// longest first, emitting SMEMs).  The start of the NEXT search of pass 1 depends on the forward phase only
// (next_x), so all forward phases of a read form one chain and every backward phase is an independent task.
// Running them as separate kernels keeps the lanes of a warp in the same loop (the forward-only pass-3 kernel does
// several times more extensions per second than the mixed automaton did).

// Forward phase(s).  single == false: pass 1, all searches of the read from x = 0 with min_intv 1
// (getSMEMsAllPosOneThread, src/FMI_search.cpp:672-724); single == true: one search from (x0, min_intv), pass 2
// (src/bwamem.cpp:695-753).  scratch: >= len+1 entries, filled from the top down so that the list handed to
// sink(x, min_intv, list, n) is already longest-first (no reversal, :587-592).
template <class Q, class Sink>
BM2_HD void fm_forward(const FmIndexView &fm, const Q &q, int len, int x0, int min_intv, bool single, FmPrev *scratch, Sink &sink,
                       unsigned &n_ext)
{
    if (len <= 0) return;
    const int cap = len + 1;
    int x = x0, j = 0, next_x = 0, top = cap;
    bool searching = false;
    FmPrev cur; cur.k = cur.l = cur.s = 0; cur.m = cur.n = 0;
    // Unique-interval shortcut (fm.text != null): once the interval of read[x..j) has ONE row, the next extensions only ask whether the text
    // goes on like the read: s' = [T[SA[k] + (j - x)] == read[j]], k unchanged (no suffix of the interval sorts before the match), so the
    // search reads the reference text (one sector per 32 bases) instead of one random Occ sector per base.  The interval of the reverse
    // complement (l) is not maintained in that mode: nothing after SMEM collection reads it (src/bwamem.cpp uses k, s, m, n), but the staged
    // entry bm2_collect_smems, whose callers see l, runs without the shortcut.  tpos: text position of read[x], -1 unknown, -2 do not try.
    int64_t tpos = -1;
    for (;;) {
        bool need = false;
        int base = 0;
        while (!need) {
            if (!searching) {
                if (x >= len) return;
                next_x = x + 1;
                const int a = q(x);
                if (a > 3) { if (single) return; x = next_x; continue; }
                cur.m = x; cur.n = x; cur.k = fm_count(fm, a); cur.l = fm_count(fm, 3 - a); cur.s = fm_count(fm, a + 1) - cur.k;
                top = cap; j = x + 1; searching = true; tpos = -1;
            }
            bool stop = j >= len;
            if (!stop) { next_x = j + 1; const int a = q(j); if (a > 3) stop = true; else { base = 3 - a; need = true; } }
            if (stop) {
                if (cur.s >= min_intv) scratch[--top] = cur;
                sink(x, min_intv, scratch + top, cap - top);
                if (single) return;
                x = next_x; searching = false;
            }
        }
        BM2_SYNCWARP();
        FmIv r;
        if (fm.text && cur.s == 1 && tpos == -1) tpos = len - j >= 16 ? fm_text_pos_of_row(fm, cur.k) : -2;      // (-1 from the walk = sentinel met: try no more)
        if (fm.text && cur.s == 1 && tpos >= 0) {
            const int64_t tp = tpos + (j - x);
            r.s = (tp < fm.text_len && (int) fm.text[tp] == 3 - base) ? 1 : 0;
            r.l = cur.k; r.k = cur.l;
        } else {
            if (tpos == -1 && fm.text && cur.s == 1) tpos = -2;
            FmIv req; req.k = cur.l; req.l = cur.k; req.s = cur.s;
            r = fm_backward_ext(fm, req, base);
        }
        ++n_ext;
        if (r.s != cur.s) scratch[--top] = cur;
        if (r.s < min_intv) {
            next_x = j;
            if (cur.s >= min_intv) scratch[--top] = cur;
            sink(x, min_intv, scratch + top, cap - top);
            if (single) return;
            x = next_x; searching = false;
        } else { cur.k = r.l; cur.l = r.k; cur.s = r.s; cur.n = j; ++j; }
    }
}

// Backward phase of one search (src/FMI_search.cpp:594-667): pv[0..num_prev) longest first, compacted in place.
template <class Q, class Emit>
BM2_HD void fm_backward(const FmIndexView &fm, const Q &q, int x, int min_intv, int min_seed_len, FmPrev *pv, int num_prev, Emit &emit,
                        unsigned &n_ext)
{
    int j = x - 1, p = 0, num_curr = 0, curr_s = -1;
    bool first_phase = true;
    for (;;) {
        // next (row, item) that needs an extension
        bool done = false;
        for (;;) {
            if (num_prev == 0 || j < 0) { done = true; break; }
            if (p == 0 && num_curr == 0 && first_phase && q(j) > 3) { done = true; break; }    // row start: stop at an ambiguous base
            if (p < num_prev) break;
            num_prev = num_curr;                                        // row finished
            if (num_curr == 0) { done = true; break; }
            --j; p = 0; num_curr = 0; curr_s = -1; first_phase = true;
        }
        if (done) break;
        BM2_SYNCWARP();
        const FmPrev old = pv[p];
        FmIv req; req.k = old.k; req.l = old.l; req.s = old.s;
        const FmIv r = fm_backward_ext(fm, req, q(j));
        ++n_ext;
        if (first_phase && r.s < min_intv && old.n - old.m + 1 >= min_seed_len) {
            emit(old.m, old.n, old.k, old.l, old.s);
            first_phase = false;
        } else if (r.s >= min_intv && r.s != curr_s) {
            curr_s = (int) r.s;
            FmPrev t; t.k = r.k; t.l = r.l; t.s = r.s; t.m = j; t.n = old.n;
            pv[num_curr++] = t;
            first_phase = false;
        }
        ++p;
    }
    if (num_prev != 0) {
        const FmPrev &s0 = pv[0];
        if (s0.n - s0.m + 1 >= min_seed_len) emit(s0.m, s0.n, s0.k, s0.l, s0.s);
    }
}

// Row-wise form of the backward phase: all intervals of the list are extended by the same base q[j]
// INDEPENDENTLY (one DRAM round trip per row when the lanes of a lane group take one entry each), then the
// sequential keep/emit rule of src/FMI_search.cpp:607-649 is applied to the extended sizes.  Because entry p+1 is
// a proper prefix of entry p (same start j+1, shorter end), the extended sizes ext_s[p] are non-decreasing in p
// and the lengths strictly decreasing, so the rule collapses to:
//   b = first p with ext_s[p] >= min_intv;  if b > 0 and entry 0 is long enough: emit entry 0 (un-extended);
//   keep p >= b iff p == b or ext_s[p] != ext_s[p-1].
// fm_backward_rows applies the rule with plain loops (host model and fallback); the kernel in pipeline.cu applies
// it with ballots.  Returns through emit exactly what fm_backward emits.
template <class Q, class Emit>
BM2_HD void fm_backward_rows(const FmIndexView &fm, const Q &q, int x, int min_intv, int min_seed_len, FmPrev *pv, int num_prev,
                             Emit &emit, unsigned &n_ext)
{
    for (int j = x - 1; j >= 0 && num_prev > 0; --j) {
        const int a = q(j);
        if (a > 3) break;
        // phase 1: independent extensions (results overwrite k,l,s in place; m,n of the old entry are still needed)
#ifdef BM2_TRACE_BWD_ROW
        BM2_TRACE_BWD_ROW(num_prev);
#endif
        int b = num_prev;
        const FmPrev first = pv[0];
        for (int p = 0; p < num_prev; ++p) {
            FmIv req; req.k = pv[p].k; req.l = pv[p].l; req.s = pv[p].s;
            const FmIv r = fm_backward_ext(fm, req, a);
            ++n_ext;
            pv[p].k = r.k; pv[p].l = r.l; pv[p].s = r.s;
            if (r.s >= min_intv && b == num_prev) b = p;
        }
        // phase 2: the keep/emit rule
        if (b > 0 && first.n - first.m + 1 >= min_seed_len) emit(first.m, first.n, first.k, first.l, first.s);
        int num_curr = 0;
        int64_t last_s = -1;
        for (int p = b; p < num_prev; ++p) {
            if (pv[p].s != last_s) { last_s = pv[p].s; FmPrev t = pv[p]; t.m = j; pv[num_curr++] = t; }
        }
        num_prev = num_curr;
    }
    if (num_prev != 0) {
        const FmPrev &s0 = pv[0];
        if (s0.n - s0.m + 1 >= min_seed_len) emit(s0.m, s0.n, s0.k, s0.l, s0.s);
    }
}

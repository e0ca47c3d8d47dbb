// cigar_device.cuh — CIGAR / NM / MD of one alignment whose end points are known (device logic, one alignment per thread).
//
// Replaces bwa_gen_cigar2 (reference src/bwa.cpp:260-347) with its banded global alignment + backtrack ksw_global2
// (src/ksw.cpp:558-668, push_cigar :545-556) as mem_reg2aln calls them (src/bwamem.cpp:1732-1805): SURVEY §8(f) item 2,
// the first widening step after the seed-chain-extend path.  Same band arithmetic (double), same direction bytes
// (f << 4 | e << 2 | h), same tie rules, reverse-strand hits aligned on the reversed sequences so that indels are placed
// leftmost.  Sequences are read through base + k * stride (no reversed copies).
//
// Written as BM2_HD: tests/host_emul/cigar_emul.cpp runs the same code on the CPU against the oracle.
#pragma once
#include "hd.h"
#include "chain_device.cuh"       // ContigView

struct CigarParams {
    int8_t mat[25];
    int o_del, e_del, o_ins, e_ins;
};

// Backtrack matrix of one thread: cell c lives at base[c * stride] (stride = threads of the launch: the lanes of a warp
// touch neighbouring bytes when they are at the same cell index; stride 1 on the host).
struct CigarZ {
    uint8_t *base; long long stride;
    BM2_HD void put(long long c, uint8_t v) const { base[c * stride] = v; }
    BM2_HD uint8_t get(long long c) const { return base[c * stride]; }
};

// push_cigar (src/ksw.cpp:545-556) into a caller-provided array
BM2_HD void cigar_push_d(uint32_t *cigar, int &n, int op, int len) {
    if (n == 0 || op != (int) (cigar[n - 1] & 0xf)) cigar[n++] = (uint32_t) len << 4 | (uint32_t) op;
    else cigar[n - 1] += (uint32_t) len << 4;
}

// Forward pass of ksw_global2 with the band in REGISTERS (round 2).  The band of a global alignment is static (|i - j| <= w), so in the
// coordinate k = j - (i - W) a column moves down by one index per row: cell k reads its column's {H, E} from slot k and writes the next
// row's values into slot k - 1 - an in-place shift for free when the sweep runs over k ascending and every index is a compile-time constant
// (the loops over k are fully unrolled, so the slots are registers; W = capacity, the run-time band w <= W is a predicate on k).  The query
// bases of the window slide the same way, 4 bits per base in a few registers (one funnel shift per word and row, the new base enters at the
// fixed slot 2W).  Same arithmetic and the same backtrack bytes at the same indices as the loop over memory rows below, which it replaces when
// the band fits: no loads on the dependent path at all (the memory version spent 91 cycles per issued instruction waiting for its rows).
// Requires w <= W and qlen <= tlen + w (then the last row reaches column qlen and H[qlen] is its h1).
// slower inside sam_kernel and cigar_kernel in an A/B (168 registers per thread, 2 x 34 slots of unrolled code per row, against the memory
// rows with hoisted loads below), so it is compiled out unless BM2_CIGAR_REG_BAND=1 is defined.
#ifndef BM2_CIGAR_REG_BAND
#define BM2_CIGAR_REG_BAND 0
#endif
template <int W>
BM2_HD int global_forward_reg_d(int qlen, const uint8_t *qp, int qstride, int tlen, const uint8_t *tp, int tstride, const int8_t *mat,
                                int o_del, int e_del, int o_ins, int e_ins, int w, const CigarZ &z)
{
    const int MINUS_INF = -0x40000000;
    const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
    const int n_col = qlen < 2 * w + 1 ? qlen : 2 * w + 1;
    constexpr int NS = 2 * W + 2;                        // slots 0 .. 2W + 1
    constexpr int NQ = (2 * W + 1 + 7) / 8;              // query window words (8 bases each)
    int32_t Hb[NS], Eb[NS];
    uint32_t qw[NQ];
    // row-0 view: slot k <-> column j = k - W
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        const int j = k - W;
        int32_t h = MINUS_INF;
        if (j == 0) h = 0; else if (j >= 1 && j <= qlen && j <= w) h = -(o_ins + e_ins * j);
        Hb[k] = h; Eb[k] = MINUS_INF;
    }
#pragma unroll
    for (int t = 0; t < NQ; ++t) qw[t] = 0;
#pragma unroll
    for (int k = 0; k <= 2 * W; ++k) {
        const int j = k - W;
        if (j >= 0 && j < qlen) qw[k >> 3] |= (uint32_t) (qp[(long long) j * qstride] > 4 ? 4 : qp[(long long) j * qstride]) << ((k & 7) * 4);
    }
    int32_t h1 = MINUS_INF;
    for (int i = 0; i < tlen; ++i) {
        int32_t f = MINUS_INF;
        const int beg = i > w ? i - w : 0;
        const int end = i + w + 1 < qlen ? i + w + 1 : qlen;
        const int tb = tp[(long long) i * tstride];
        h1 = beg == 0 ? -(o_del + e_del * (i + 1)) : MINUS_INF;
        const long long zrow = (long long) i * n_col - beg;          // z index of column j: zrow + j
        const int ke = end - i + W;                                   // slot of column `end` in this row's view
        // the five scores of this row's target base against query bases 0 .. 4
        const int tb5 = (tb > 4 ? 4 : tb) * 5;
        const int s0 = mat[tb5], s1 = mat[tb5 + 1], s2 = mat[tb5 + 2], s3 = mat[tb5 + 3], s4 = mat[tb5 + 4];
#pragma unroll
        for (int k = 0; k <= 2 * W; ++k) {
            const int j = i - W + k;
            if (j >= beg && j < end) {
                int32_t m = Hb[k], e = Eb[k];
                const int32_t hs = h1;
                const uint32_t qb = (qw[k >> 3] >> ((k & 7) * 4)) & 15u;
                m += qb == 0 ? s0 : qb == 1 ? s1 : qb == 2 ? s2 : qb == 3 ? s3 : s4;
                uint8_t d = m >= e ? 0 : 1;
                int32_t h = m >= e ? m : e;
                d = h >= f ? d : 2;
                h = h >= f ? h : f;
                h1 = h;
                int32_t t = m - oe_del;
                e -= e_del;
                d |= e > t ? 1 << 2 : 0;
                e = e > t ? e : t;
                t = m - oe_ins;
                f -= e_ins;
                d |= f > t ? 2 << 4 : 0;
                f = f > t ? f : t;
                z.put(zrow + j, d);
                if (k > 0) { Hb[k - 1] = hs; Eb[k - 1] = e; }
            }
        }
        // H[end] = h1; E[end] = MINUS_INF: column `end` sits in slot ke - 1 of the next row's view
#pragma unroll
        for (int k = 1; k < NS; ++k)
            if (k == ke) { Hb[k - 1] = h1; Eb[k - 1] = MINUS_INF; }
        // the query window slides by one base; column i + 1 + W enters at slot 2W
#pragma unroll
        for (int t = 0; t < NQ; ++t) qw[t] = (qw[t] >> 4) | (t + 1 < NQ ? qw[t + 1] << 28 : 0u);
        {
            const int jn = i + 1 + W;
            if (jn < qlen) {
                const uint32_t c = qp[(long long) jn * qstride];
                qw[(2 * W) >> 3] |= (c > 4 ? 4u : c) << (((2 * W) & 7) * 4);
            }
        }
    }
    return h1;                                            // = H[qlen]: the last row's band ends at column qlen
}

// ksw_global2 with backtrack (src/ksw.cpp:558-668).  he: 2*(qlen+1) ints; z: n_col*tlen cells, n_col = min(qlen, 2w+1);
// cigar: room for qlen + tlen + 2 operations.  Returns the score; *n_cigar operations in cigar[].
BM2_HD int global_align_d(int qlen, const uint8_t *qp, int qstride, int tlen, const uint8_t *tp, int tstride, const int8_t *mat,
                          int o_del, int e_del, int o_ins, int e_ins, int w, int32_t *he, const CigarZ &z, uint32_t *cigar, int *n_cigar)
{
    const int MINUS_INF = -0x40000000;
    const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
    const int n_col = qlen < 2 * w + 1 ? qlen : 2 * w + 1;
    int score_reg = 0;
    const bool in_regs = BM2_CIGAR_REG_BAND && w <= 16 && tlen > 0 && qlen <= tlen + w;
    if (in_regs) score_reg = global_forward_reg_d<16>(qlen, qp, qstride, tlen, tp, tstride, mat, o_del, e_del, o_ins, e_ins, w, z);
    int32_t *H = he, *E = he + (qlen + 1);
    int j;
    if (!in_regs) {
    H[0] = 0; E[0] = MINUS_INF;
    for (j = 1; j <= qlen && j <= w; ++j) { H[j] = -(o_ins + e_ins * j); E[j] = MINUS_INF; }
    for (; j <= qlen; ++j) H[j] = E[j] = MINUS_INF;
    for (int i = 0; i < tlen; ++i) {
        int32_t f = MINUS_INF, h1;
        const int beg = i > w ? i - w : 0;
        const int end = i + w + 1 < qlen ? i + w + 1 : qlen;
        const int tb = tp[(long long) i * tstride];
        h1 = beg == 0 ? -(o_del + e_del * (i + 1)) : MINUS_INF;
        const long long zi = (long long) i * n_col;
        // One cell: the recurrence of ksw_global2 on values already in registers.  hs = the value H[j] takes (the previous cell's h).
        auto cell = [&](int32_t m, int32_t e, const int qb, int32_t &hs, int32_t &es) -> uint8_t {
            hs = h1;
            m += mat[tb * 5 + qb];
            uint8_t d = m >= e ? 0 : 1;
            int32_t h = m >= e ? m : e;
            d = h >= f ? d : 2;
            h = h >= f ? h : f;
            h1 = h;
            int32_t t = m - oe_del;
            e -= e_del;
            d |= e > t ? 1 << 2 : 0;
            e = e > t ? e : t;
            es = e;
            t = m - oe_ins;
            f -= e_ins;
            d |= f > t ? 2 << 4 : 0;
            f = f > t ? f : t;
            return d;
        };
        // Four cells per trip with all their loads (H, E, query bases) issued before the first cell is computed: the loads of neighbouring
        // cells do not depend on each other (only h1 and f run along the row, in registers), so a thread keeps 12 loads in flight instead of
        // waiting for each in turn - the rows live in per-thread global memory and this loop was bound by their latency (round 2 profile of the
        // SAM stage).  Same arithmetic, same order.
        for (j = beg; j + 4 <= end; j += 4) {
            const int32_t m0 = H[j], m1 = H[j + 1], m2 = H[j + 2], m3 = H[j + 3];
            const int32_t e0 = E[j], e1 = E[j + 1], e2 = E[j + 2], e3 = E[j + 3];
            const int q0 = qp[(long long) j * qstride], q1 = qp[(long long) (j + 1) * qstride], q2 = qp[(long long) (j + 2) * qstride],
                      q3 = qp[(long long) (j + 3) * qstride];
            int32_t hs0, hs1, hs2, hs3, es0, es1, es2, es3;
            const uint8_t d0 = cell(m0, e0, q0, hs0, es0), d1 = cell(m1, e1, q1, hs1, es1), d2 = cell(m2, e2, q2, hs2, es2), d3 = cell(m3, e3, q3, hs3, es3);
            H[j] = hs0; H[j + 1] = hs1; H[j + 2] = hs2; H[j + 3] = hs3;
            E[j] = es0; E[j + 1] = es1; E[j + 2] = es2; E[j + 3] = es3;
            const long long zc = zi + (j - beg);
            z.put(zc, d0); z.put(zc + 1, d1); z.put(zc + 2, d2); z.put(zc + 3, d3);
        }
        for (; j < end; ++j) {
            int32_t hs, es;
            const uint8_t d = cell(H[j], E[j], qp[(long long) j * qstride], hs, es);
            H[j] = hs; E[j] = es;
            z.put(zi + (j - beg), d);
        }
        H[end] = h1; E[end] = MINUS_INF;
    }
    }
    const int score = in_regs ? score_reg : H[qlen];
    // backtrack
    int n = 0, which = 0;
    int i = tlen - 1, k = (i + w + 1 < qlen ? i + w + 1 : qlen) - 1;
    while (i >= 0 && k >= 0) {
        which = z.get((long long) i * n_col + (k - (i > w ? i - w : 0))) >> (which << 1) & 3;
        if (which == 0) { cigar_push_d(cigar, n, 0, 1); --i; --k; }
        else if (which == 1) { cigar_push_d(cigar, n, 2, 1); --i; }
        else { cigar_push_d(cigar, n, 1, 1); --k; }
    }
    if (i >= 0) cigar_push_d(cigar, n, 2, i + 1);
    if (k >= 0) cigar_push_d(cigar, n, 1, k + 1);
    for (i = 0; i < n >> 1; ++i) { const uint32_t tmp = cigar[i]; cigar[i] = cigar[n - 1 - i]; cigar[n - 1 - i] = tmp; }
    *n_cigar = n;
    return score;
}

// band of the global alignment (src/bwa.cpp:292-300; double arithmetic as the reference)
BM2_HD int cigar_band_d(const CigarParams &p, int w_, int l_query, long long rlen) {
    int max_ins = (int) ((double) (((l_query + 1) >> 1) * p.mat[0] - p.o_ins) / p.e_ins + 1.);
    int max_del = (int) ((double) (((l_query + 1) >> 1) * p.mat[0] - p.o_del) / p.e_del + 1.);
    int max_gap = max_ins > max_del ? max_ins : max_del;
    max_gap = max_gap > 1 ? max_gap : 1;
    int diff = (int) (rlen - l_query); if (diff < 0) diff = -diff;
    int w = (max_gap + diff + 1) >> 1;
    w = w < w_ ? w : w_;
    const int min_w = diff + 3;
    return w > min_w ? w : min_w;
}

// cells of the backtrack matrix a request needs (0: no DP)
BM2_HD long long cigar_z_cells_d(const CigarParams &p, int64_t l_pac, int w_, int l_query, int64_t rb, int64_t re) {
    if (l_query <= 0 || rb >= re || (rb < l_pac && re > l_pac) || re > (l_pac << 1) || rb < 0) return 0;
    const long long rlen = re - rb;
    if (l_query == rlen && w_ == 0) return 0;
    const int w = cigar_band_d(p, w_, l_query, rlen);
    const long long n_col = l_query < 2 * w + 1 ? l_query : 2 * w + 1;
    return n_col * rlen;
}

// decimal digits of a non-negative int appended to md (kputw)
BM2_HD void md_putw_d(char *md, int &n, int v) {
    char buf[12]; int l = 0;
    if (v == 0) buf[l++] = '0';
    while (v > 0) { buf[l++] = (char) ('0' + v % 10); v /= 10; }
    while (l > 0) md[n++] = buf[--l];
}

// bwa_gen_cigar2 (src/bwa.cpp:260-347).  query: the read's codes (0-4), l_query of them; ref: 2*l_pac codes (fwd || revcomp).
// Outputs: *score (untouched when the request is rejected, as in the reference), cigar[0..*n_cigar), *nm (-1 when rejected),
// md[0..*n_md) (NUL-terminated, the terminator counted as the reference appends it).  Returns false when rejected.
// Capacities: cigar l_query + rlen + 2 operations, md 2*l_query + 7*rlen + 16 bytes, he 2*(l_query+1) ints.
BM2_HD bool gen_cigar_d(const CigarParams &p, int64_t l_pac, const uint8_t *ref, int w_, int l_query, const uint8_t *query, int64_t rb, int64_t re,
                        int32_t *he, const CigarZ &z, int *score, uint32_t *cigar, int *n_cigar, int *nm, char *md, int *n_md)
{
    *n_cigar = 0; *nm = -1; *n_md = 0;
    if (l_query <= 0 || rb >= re || (rb < l_pac && re > l_pac)) return false;
    if (re > (l_pac << 1) || rb < 0) return false;                       // bns_get_seq clips: rlen != re - rb
    const long long rlen = re - rb;
    const bool rev = rb >= l_pac;
    const uint8_t *qp = rev ? query + (l_query - 1) : query; const int qs = rev ? -1 : 1;
    const uint8_t *tp = rev ? ref + (re - 1) : ref + rb;      const int ts = rev ? -1 : 1;
    int n = 0;
    if (l_query == rlen && w_ == 0) {
        cigar[0] = (uint32_t) l_query << 4 | 0; n = 1;
        int sc = 0;
        for (int i = 0; i < l_query; ++i) sc += p.mat[tp[(long long) i * ts] * 5 + qp[(long long) i * qs]];
        *score = sc;
    } else {
        const int w = cigar_band_d(p, w_, l_query, rlen);
        *score = global_align_d(l_query, qp, qs, (int) rlen, tp, ts, p.mat, p.o_del, p.e_del, p.o_ins, p.e_ins, w, he, z, cigar, &n);
    }
    *n_cigar = n;
    // NM and MD (src/bwa.cpp:305-337)
    {
        int x = 0, y = 0, u = 0, n_mm = 0, n_gap = 0, m = 0;
        for (int k = 0; k < n; ++k) {
            const int op = (int) (cigar[k] & 0xf), len = (int) (cigar[k] >> 4);
            if (op == 0) {
                for (int i = 0; i < len; ++i) {
                    const int qb = qp[(long long) (x + i) * qs], tb = tp[(long long) (y + i) * ts];
                    if (qb != tb) {
                        md_putw_d(md, m, u);
                        md[m++] = rev ? "TGCAN"[tb] : "ACGTN"[tb];
                        ++n_mm; u = 0;
                    } else ++u;
                }
                x += len; y += len;
            } else if (op == 2) {
                if (k > 0 && k < n - 1) {
                    md_putw_d(md, m, u); md[m++] = '^';
                    for (int i = 0; i < len; ++i) { const int tb = tp[(long long) (y + i) * ts]; md[m++] = rev ? "TGCAN"[tb] : "ACGTN"[tb]; }
                    u = 0; n_gap += len;
                }
                y += len;
            } else if (op == 1) { x += len; n_gap += len; }
        }
        md_putw_d(md, m, u); md[m++] = 0;
        *nm = n_mm + n_gap;
        *n_md = m;
    }
    return true;
}

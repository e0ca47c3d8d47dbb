// bqsr_device.cuh — the per-record rule of bm2_mem --recal-file: GATK 4 BaseRecalibrator's substitution covariates at its defaults
// (mismatch context 2, low-quality tail 2, qualities below 6 preserved, maximum cycle 500, no BAQ), one BAM record at a time.  bqsr.cu's kernel
// runs it with one warp per record; tests/host_emul/bqsr_emul.cpp compiles it for the host, and tests/bqsr_util.py restates it in Python.
//
//   counted   a record without 0x4, 0x100, 0x800, 0x400 or 0x200, with MAPQ neither 0 nor 255, a CIGAR and bases
//   clipping  (1-based: start = pos + 1, end = pos + reference length, mate_start = mpos + 1, T = TLEN) adaptor clipping when T != 0, 0x1,
//             neither read nor mate unmapped, the strands differ, and (reverse) end > mate_start or (forward) start <= mate_start + T: the
//             boundary b is mate_start - 1 (reverse) or start + |T| (forward); when start <= b <= end a reverse read loses every base up to
//             and including the last one aligned at a position <= b, a forward read every base from the first one aligned at >= b.  Then
//             soft clips go.  The bases left, [lo, hi) of the read, are the clipped read; an empty one is not counted
//   errors    a read without qualities (0xff), a clipped read of more than 500 bases, a quality above 93: the record is not counted and
//             the call reports it
//   read group  (bm2_baserecalibrator; bm2_mem has one read group and no lookup) a record that passes the filters must have an RG:Z tag whose
//             value is an @RG ID of the headers (bqsr_rg_lookup), checked before the errors above: a record without the tag, or with a value
//             that is no ID, is an error; the record counts into the tables of that ID's covariate.  A filtered record's tag is not read.
//   a base    of the clipped read: aligned (M = X) at reference g, or inserted between g and g + 1.  Skipped when its base is N, its quality
//             is below 6, or it is a known-site base (aligned: `covered` bit g; inserted: `junction` bit g).  An error when aligned and its
//             base differs from the reference's (N inside an .amb hole)
//   covariates  quality; cycle (i + 1) * f forward, (L - i) * f reverse (i its index in the clipped read, L its length, f = -1 for the
//             second of a pair); context: the clipped read's bases with the low-quality tails (quality <= 2 at either end) written as N, in
//             sequencing order (reverse-complemented for a reverse read), the two letters ending at the base, none for the first base or an N
#pragma once
#include "hd.h"
#include <stdint.h>

#define BQSR_NQ 94                  // qualities 0..93
#define BQSR_NCTX 16                // contexts: 4 * first + second letter, A C G T = 0 1 2 3
#define BQSR_MAX_CYCLE 500
#define BQSR_NCYC 1001              // cycles -500..500, at cycle + 500
#define BQSR_MIN_Q 6
#define BQSR_TAIL_Q 2

// the counters of one covariate (bqsr.cu's kernel, bm2_bqsr_tables, bm2_recal_tables): (quality, context) observations and errors, (quality,
// cycle) observations and errors, reads, bases
constexpr int kBqsrCxTab = 2 * BQSR_NQ * BQSR_NCTX;
constexpr int64_t kBqsrCxObs = 0, kBqsrCxErr = BQSR_NQ * BQSR_NCTX, kBqsrCyObs = kBqsrCxTab, kBqsrCyErr = kBqsrCyObs + BQSR_NQ * BQSR_NCYC,
                  kBqsrReads = kBqsrCyErr + BQSR_NQ * BQSR_NCYC, kBqsrBases = kBqsrReads + 1, kBqsrCounts = kBqsrBases + 1;
// Up to this many covariates the kernel keeps their (quality, context) tables (23.5 KB each) per CTA in shared memory; above it, in global
// memory.  Two tables and a full read-group map (kBqsrMapMax) take 79 KB, two CTAs of 8 warps per SM; two tables and a small map keep four.
constexpr int kBqsrSharedCovMax = 2;
constexpr int64_t kBqsrMapMax = 32768;      // bytes of a read-group map: 16 per ID and the IDs' bytes

enum { BQSR_COUNT = 0, BQSR_FILTERED = 1, BQSR_EMPTY = 2, BQSR_ERR_NOQUAL = 3, BQSR_ERR_CYCLES = 4, BQSR_ERR_QUAL = 5, BQSR_ERR_NORG = 6,
       BQSR_ERR_BADRG = 7 };

// the reference and the known sites, all over the forward strand's concatenated contigs [0, l_pac)
struct BqsrView {
    const uint8_t *ref;                 // codes 0..3, one byte per base; nullptr: pac holds the reference
    const int64_t *ann_off;             // each contig's offset
    int32_t n_seqs;
    int64_t l_pac;
    const uint64_t *covered, *junction; // 1 bit per base
    const int64_t *holes;               // .amb holes as [beg, end) pairs, sorted
    int64_t n_holes;
    const uint8_t *pac;                 // 2 bits per base, base g at pac[g >> 2] >> ((~g & 3) << 1) & 3 (the .pac layout), when ref is nullptr
};

struct BqsrRec {
    int status;                         // BQSR_*
    int rev, f;                         // reverse strand, cycle sign
    int32_t lo, hi;                     // the clipped read: read bases [lo, hi)
    int32_t tl, tr;                     // the bases outside [tl, tr) are the low-quality tails (set by the caller: bqsr_tails)
    int64_t g0;                         // the global coordinate of pos
    int64_t hole;                       // the first hole that ends after g0, when one starts before the alignment ends; else -1
    const uint32_t *cig; int n_cigar;
    const uint8_t *seq, *qual; int32_t l_seq;
};

BM2_HD int32_t bqsr_le32(const uint8_t *p) { return (int32_t) ((uint32_t) p[0] | (uint32_t) p[1] << 8 | (uint32_t) p[2] << 16 | (uint32_t) p[3] << 24); }
BM2_HD uint32_t bqsr_cig(const uint32_t *c, int k) { return (uint32_t) bqsr_le32((const uint8_t *) (c + k)); }
BM2_HD bool bqsr_bit(const uint64_t *b, int64_t g) { return (b[g >> 6] >> (g & 63)) & 1; }

// a BAM base (4-bit code) as 0..3, anything but A C G T as 4
BM2_HD int bqsr_base_code(const uint8_t *seq, int32_t k) {
    const int c = (seq[k >> 1] >> ((k & 1) ? 0 : 4)) & 15;
    return c == 1 ? 0 : c == 2 ? 1 : c == 4 ? 2 : c == 8 ? 3 : 4;
}

// the fixed fields, filters and clipping of one record (rec: its block_size field)
BM2_HD void bqsr_prep(const uint8_t *rec, const BqsrView &v, BqsrRec &r) {
    const int32_t rid = bqsr_le32(rec + 4), pos = bqsr_le32(rec + 8);
    const int l_name = rec[12], mapq = rec[13];
    const int n_cigar = rec[16] | rec[17] << 8, flag = rec[18] | rec[19] << 8;
    const int32_t l_seq = bqsr_le32(rec + 20), mpos = bqsr_le32(rec + 28), tlen = bqsr_le32(rec + 32);
    r.status = BQSR_FILTERED; r.hole = -1;
    r.cig = (const uint32_t *) (rec + 36 + l_name); r.n_cigar = n_cigar;
    r.seq = rec + 36 + l_name + 4 * n_cigar; r.qual = r.seq + ((l_seq + 1) >> 1); r.l_seq = l_seq;
    r.rev = (flag & 16) != 0; r.f = (flag & 1) && (flag & 0x80) ? -1 : 1;
    if ((flag & (0x4 | 0x100 | 0x800 | 0x400 | 0x200)) || mapq == 0 || mapq == 255 || rid < 0 || rid >= v.n_seqs || n_cigar == 0 || l_seq <= 0) return;
    if (r.qual[0] == 0xff) { r.status = BQSR_ERR_NOQUAL; return; }
    int64_t rlen = 0;
    int32_t sl = 0, sr = 0, k = 0;
    bool seen = false;
    for (int c = 0; c < n_cigar; ++c) {
        const uint32_t o = bqsr_cig(r.cig, c), op = o & 15, n = o >> 4;
        if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += n;
        if (op == 4) { if (seen) sr += (int32_t) n; else sl += (int32_t) n; }
        else if (op != 5) seen = true;
    }
    int32_t lo = sl, hi = l_seq - sr;
    const int64_t start = (int64_t) pos + 1, end = (int64_t) pos + rlen, mstart = (int64_t) mpos + 1;
    if (tlen != 0 && (flag & 1) && !(flag & 4) && !(flag & 8) && ((flag >> 4) & 1) != ((flag >> 5) & 1) &&
        (r.rev ? end > mstart : start <= mstart + tlen)) {
        const int64_t b = r.rev ? mstart - 1 : start + (tlen < 0 ? -(int64_t) tlen : (int64_t) tlen);
        if (start <= b && b <= end) {
            int64_t g = start;                                                  // 1-based position of the next reference base
            int32_t last_le = -1, first_ge = l_seq;
            for (int c = 0; c < n_cigar; ++c) {
                const uint32_t o = bqsr_cig(r.cig, c), op = o & 15, n = o >> 4;
                if (op == 0 || op == 7 || op == 8) {                            // the op covers [g, g + n)
                    if (n && g <= b) last_le = k + (int32_t) bm2_min<int64_t>((int64_t) n - 1, b - g);
                    if (n && first_ge == l_seq && g + (int64_t) n - 1 >= b) first_ge = k + (int32_t) bm2_max<int64_t>(0, b - g);
                    k += (int32_t) n; g += n;
                } else if (op == 1 || op == 4) k += (int32_t) n;
                else if (op == 2 || op == 3) g += n;
            }
            if (r.rev) lo = bm2_max(lo, last_le + 1);
            else hi = bm2_min(hi, first_ge);
        }
    }
    r.lo = lo; r.hi = hi;
    if (hi <= lo) { r.status = BQSR_EMPTY; return; }
    if (hi - lo > BQSR_MAX_CYCLE) { r.status = BQSR_ERR_CYCLES; return; }
    r.g0 = v.ann_off[rid] + pos;
    r.tl = lo; r.tr = hi;
    if (v.n_holes) {                                                         // the first hole that ends after g0
        int64_t a = 0, e = v.n_holes;
        while (a < e) { const int64_t m = (a + e) >> 1; if (v.holes[2 * m + 1] <= r.g0) a = m + 1; else e = m; }
        if (a < v.n_holes && v.holes[2 * a] < r.g0 + rlen) r.hole = a;
    }
    r.status = BQSR_COUNT;
}

// the low-quality tails and the quality check of a prepared record, one base at a time (the kernel does the same with ballots)
BM2_HD void bqsr_tails(BqsrRec &r) {
    int32_t tl = r.hi, tr = r.lo;
    for (int32_t k = r.lo; k < r.hi; ++k) {
        const int q = r.qual[k];
        if (q > BQSR_NQ - 1) { r.status = BQSR_ERR_QUAL; return; }
        if (q > BQSR_TAIL_Q) { if (tl == r.hi) tl = k; tr = k + 1; }
    }
    if (tl == r.hi) tr = r.hi;
    r.tl = tl; r.tr = tr;
}

// the context letter of read base k: N (4) inside a low-quality tail
BM2_HD int bqsr_ctx_letter(const BqsrRec &r, int32_t k) { return k < r.tl || k >= r.tr ? 4 : bqsr_base_code(r.seq, k); }

// the reference base at g: N (4) inside an .amb hole
BM2_HD int bqsr_ref_base(const BqsrRec &r, const BqsrView &v, int64_t g) {
    if (r.hole >= 0)
        for (int64_t h = r.hole; h < v.n_holes && v.holes[2 * h] <= g; ++h)
            if (g < v.holes[2 * h + 1]) return 4;
    return v.ref ? v.ref[g] : (v.pac[g >> 2] >> ((~g & 3) << 1)) & 3;
}

// the context (-1: none) and cycle of read base k of [lo, hi), the tails set: what both the counting and the apply side key a base by
BM2_HD void bqsr_covariates(const BqsrRec &r, int32_t k, int &cx, int &cyc) {
    const int32_t i = k - r.lo, L = r.hi - r.lo;
    cyc = (r.rev ? L - i : i + 1) * r.f;
    cx = -1;
    int c0, c1;
    if (!r.rev) {
        if (k == r.lo) return;
        c0 = bqsr_ctx_letter(r, k - 1); c1 = bqsr_ctx_letter(r, k);
    } else {
        if (k == r.hi - 1) return;
        c0 = bqsr_ctx_letter(r, k + 1); c1 = bqsr_ctx_letter(r, k);
        c0 = c0 == 4 ? 4 : 3 - c0; c1 = c1 == 4 ? 4 : 3 - c1;
    }
    if (c0 != 4 && c1 != 4) cx = c0 * 4 + c1;
}

// read base k of a counted record, aligned at g (ins false) or inserted between g and g + 1 (ins true): false when skipped, else its
// quality, context (-1: none), cycle and whether it is an error
BM2_HD bool bqsr_base(const BqsrRec &r, const BqsrView &v, int32_t k, bool ins, int64_t g, int &q, int &cx, int &cyc, int &err) {
    const int b = bqsr_base_code(r.seq, k);
    q = r.qual[k];
    if (b == 4 || q < BQSR_MIN_Q) return false;
    if (ins ? (g >= 0 && g + 1 < v.l_pac && bqsr_bit(v.junction, g)) : bqsr_bit(v.covered, g)) return false;
    err = !ins && bqsr_ref_base(r, v, g) != b;
    bqsr_covariates(r, k, cx, cyc);
    return true;
}

// the walk of a counted record's CIGAR: fn(k, ins, g) for every read base k of [lo, hi) that is aligned or inserted
template <class Fn> BM2_HD void bqsr_walk(const BqsrRec &r, Fn fn) {
    int32_t k = 0; int64_t g = r.g0;
    for (int c = 0; c < r.n_cigar; ++c) {
        const uint32_t o = bqsr_cig(r.cig, c), op = o & 15, n = o >> 4;
        if (op == 0 || op == 7 || op == 8) {
            for (uint32_t j = 0; j < n; ++j) if (k + (int32_t) j >= r.lo && k + (int32_t) j < r.hi) fn(k + (int32_t) j, false, g + j);
            k += (int32_t) n; g += n;
        } else if (op == 1) {
            for (uint32_t j = 0; j < n; ++j) if (k + (int32_t) j >= r.lo && k + (int32_t) j < r.hi) fn(k + (int32_t) j, true, g - 1);
            k += (int32_t) n;
        } else if (op == 4) k += (int32_t) n;
        else if (op == 2 || op == 3) g += n;
    }
}

// ---- the apply side (bm2_applybqsr): GATK 4 ApplyBQSR's BQSRReadTransformer at its defaults (no quantization, qualities below 6 kept,
// no OQ tag, no global prior), one BAM record at a time.  bqsr_apply.cu's kernel runs it with one warp per record;
// tests/host_emul/applybqsr_emul.cpp compiles it for the host, and tests/applybqsr_util.py restates it in Python.
//   read group  the RG:Z tag's value, matched to the input header's @RG IDs (the first line with that ID), that line's covariate (PU, else
//               ID) and its tables (bqsr_report.h).  A record without the tag, with an ID not in the header, or of a read group without a
//               RecalTable0 row is written unchanged; so are l_seq 0 and QUAL '*' (0xff).  Every flag is recalibrated.
//   errors      more than 500 bases, a quality above 93: the record is not rewritten and the call reports it
//   a base      q < 6 stays; else clamp(fastRound(P[q] + ((0.0 + D_ctx[q][ctx]) + D_cyc[q][cyc])), 1, 93), fastRound(d) = (int) (d + 0.5) for
//               d > 0, else (int) (d - 0.5).  ctx and cyc are bqsr_covariates over the whole stored read (lo = 0, hi = l_seq: no adaptor
//               clipping, soft clips kept), the tails being the qualities <= 2 at either end; no context: D_ctx = 0
enum { BQSR_APPLY = 0, BQSR_KEEP = 1 };   // and BQSR_ERR_CYCLES, BQSR_ERR_QUAL

// one read group's dense tables: P [94], D_ctx [94 * 16], D_cyc [94 * 1001] (cycle + 500)
struct BqsrApplyView { const double *P, *ctx, *cyc; };

// where a record's RG:Z value starts (offset from rec, its block_size field) and its length without the NUL; -1 without one.  The walk
// stops at the first tag it cannot step over.
BM2_HD int32_t bqsr_aux_rg(const uint8_t *rec, int32_t *len) {
    const int32_t end = 4 + bqsr_le32(rec), l_seq = bqsr_le32(rec + 20);
    int32_t p = 36 + rec[12] + 4 * (rec[16] | rec[17] << 8) + ((l_seq + 1) >> 1) + l_seq;
    while (p + 3 <= end) {
        const uint8_t t0 = rec[p], t1 = rec[p + 1], ty = rec[p + 2];
        p += 3;
        if (ty == 'Z' || ty == 'H') {
            int32_t q = p;
            while (q < end && rec[q]) ++q;
            if (q >= end) return -1;
            if (t0 == 'R' && t1 == 'G' && ty == 'Z') { *len = q - p; return p; }
            p = q + 1;
        } else if (ty == 'B') {
            if (p + 5 > end) return -1;
            const uint8_t s = rec[p];
            const int es = s == 'c' || s == 'C' ? 1 : s == 's' || s == 'S' ? 2 : s == 'i' || s == 'I' || s == 'f' ? 4 : 0;
            const int64_t n = (int64_t) (uint32_t) bqsr_le32(rec + p + 1);
            if (!es || p + 5 + n * es > end) return -1;
            p += 5 + (int32_t) (n * es);
        } else {
            const int sz = ty == 'A' || ty == 'c' || ty == 'C' ? 1 : ty == 's' || ty == 'S' ? 2 : ty == 'i' || ty == 'I' || ty == 'f' ? 4 : 0;
            if (!sz) return -1;
            p += sz;
        }
    }
    return -1;
}

// one entry of a read-group map: the map is n_ids entries, then the IDs' bytes; off is an ID's offset from the map's start, val what the
// caller keeps per ID (a table, library or covariate index)
struct BqsrRgEntry { int32_t off, len, val, pad; };

// the index of the first map entry whose ID is the len bytes at rec + at (bqsr_aux_rg's value), -1 when none.  On the device the whole warp
// calls it with the same arguments, and the lanes compare 32 IDs at a time.
BM2_HD int bqsr_rg_lookup(const BqsrRgEntry *map, int n_ids, const uint8_t *rec, int32_t at, int32_t len) {
    const uint8_t *bytes = (const uint8_t *) map;
#if defined(__CUDA_ARCH__)
    const int lane = threadIdx.x & 31;
    for (int j0 = 0; j0 < n_ids; j0 += 32) {
        const int j = j0 + lane;
        bool m = false;
        if (j < n_ids) {
            const BqsrRgEntry e = map[j];
            m = e.len == len;
            for (int k = 0; m && k < len; ++k) m = bytes[e.off + k] == rec[at + k];
        }
        const unsigned b = __ballot_sync(0xFFFFFFFFu, m);
        if (b) return j0 + __ffs(b) - 1;
    }
#else
    for (int j = 0; j < n_ids; ++j) {
        bool m = map[j].len == len;
        for (int k = 0; m && k < len; ++k) m = bytes[map[j].off + k] == rec[at + k];
        if (m) return j;
    }
#endif
    return -1;
}

// the fixed fields of a record to recalibrate: status BQSR_APPLY, BQSR_KEEP or BQSR_ERR_CYCLES; lo = 0, hi = l_seq
BM2_HD void bqsr_apply_prep(const uint8_t *rec, BqsrRec &r) {
    const int l_name = rec[12], n_cigar = rec[16] | rec[17] << 8, flag = rec[18] | rec[19] << 8;
    const int32_t l_seq = bqsr_le32(rec + 20);
    r.seq = rec + 36 + l_name + 4 * n_cigar; r.qual = r.seq + ((l_seq + 1) >> 1); r.l_seq = l_seq;
    r.rev = (flag & 16) != 0; r.f = (flag & 1) && (flag & 0x80) ? -1 : 1;
    r.lo = 0; r.hi = l_seq; r.tl = 0; r.tr = l_seq;
    r.cig = nullptr; r.n_cigar = 0; r.g0 = 0; r.hole = -1;
    r.status = l_seq <= 0 || r.qual[0] == 0xff ? (int) BQSR_KEEP : l_seq > BQSR_MAX_CYCLE ? (int) BQSR_ERR_CYCLES : (int) BQSR_APPLY;
}

// the recalibrated quality of a base of quality q with context cx (-1: none) and cycle cyc
BM2_HD int bqsr_recal_q(const BqsrApplyView &t, int q, int cx, int cyc) {
    if (q < BQSR_MIN_Q) return q;
    const double d = t.P[q] + ((0.0 + (cx >= 0 ? t.ctx[q * BQSR_NCTX + cx] : 0.0)) + t.cyc[q * BQSR_NCYC + cyc + BQSR_MAX_CYCLE]);
    const int v = d > 0 ? (int) (d + 0.5) : (int) (d - 0.5);
    return v < 1 ? 1 : v > BQSR_NQ - 1 ? BQSR_NQ - 1 : v;
}

// wgs_device.cuh — the per-record and per-locus rule of bm2_wgsmetrics (wgs.cu): BM2_HD functions, so that the host emulation
// tests/host_emul/wgsmetrics_emul.cpp compiles the same source.  It restates Picard CollectWgsMetrics at its defaults (MINIMUM_MAPPING_QUALITY
// 20, MINIMUM_BASE_QUALITY 20, COVERAGE_CAP 250, COUNT_UNPAIRED false, no INTERVALS, USE_FAST_ALGORITHM false); byte equality with Picard is
// not claimed.
//
//   locus     g = the contig's offset in the concatenated reference (.ann) + pos + the reference offset inside the alignment.  A locus inside
//             an .amb hole of N, n or . is no-call (Picard's SequenceUtil.isNoCall); holes of other IUPAC letters are ordinary loci.
//   skip      records with 0x4, refID -1 or 0x200 count nowhere (0x200 is our choice; bwa-mem2 never sets it)
//   filters   the first that matches takes the record; its aligned bases (the lengths of its M / = / X operations, no-call loci included, as
//             Picard counts alignment blocks) go to that counter:
//               MAPQ < min_mapq -> EXC_MAPQ;  0x400 -> EXC_DUPE;  without count_unpaired, no 0x1 or with 0x8 -> EXC_UNPAIRED;
//               0x100 -> dropped, counted nowhere (Picard's non-counting SecondaryAlignmentFilter).  0x800 passes like a primary.
//   bases     of a record that passes, each aligned base at locus g: nothing at a no-call locus; quality < min_baseq or read base N (nibble
//             15) -> EXC_BASEQ; otherwise high-quality: EXC_OVERLAP when a record earlier in the file with the same QNAME has a high-quality
//             base at g, else pileup[g] += 1.  So pileup[g] is the number of distinct QNAMEs with a high-quality base at g.
//   loci      every locus that is not no-call: depth = min(pileup, cap), EXC_CAPPED += max(0, pileup - cap), H[depth] += 1
//   errors    a record that is not skipped whose refID is not a contig or whose alignment does not lie inside its contig; a record whose
//             CIGAR moved to CG:B,I runs past the record; a record that passes with l_seq 0, QUAL '*', or a CIGAR whose query length is not l_seq
#pragma once
#include "hd.h"
#include "bam_sort_device.cuh"
#include "markdup_device.cuh"

// tests build the emulation with -DWGS_HASH_MASK=0 so that every name hashes alike and only the byte comparison tells templates apart
#ifndef WGS_HASH_MASK
#define WGS_HASH_MASK 0x7FFFFFFFFFFFFFFFull
#endif

enum { WGS_EXC_MAPQ, WGS_EXC_DUPE, WGS_EXC_UNPAIRED, WGS_EXC_BASEQ, WGS_EXC_OVERLAP, WGS_EXC_CAPPED, WGS_NEXC };
// a record's status; the filter statuses index the exclusion counters
enum { WGS_FILT_MAPQ = WGS_EXC_MAPQ, WGS_FILT_DUPE = WGS_EXC_DUPE, WGS_FILT_UNPAIRED = WGS_EXC_UNPAIRED, WGS_SKIP = 3, WGS_DROP = 4, WGS_PASS = 5,
       WGS_ERR_NOQUAL = 6, WGS_ERR_SPAN = 7, WGS_ERR_CIGAR = 8 };
constexpr uint64_t WGS_NOT_CANDIDATE = 1ull << 63;      // the sort key of a record the overlap pass does not take

// a record's placement, kept on the device (and the host, for the carry) from the check to the overlap pass
struct WgsInfo {
    int64_t g0, g1;      // the loci [g0, g1) its alignment spans
    int32_t rid, status;
    int32_t aligned;     // the lengths of its M / = / X operations
    int32_t _pad;
};

BM2_HD bool wgs_aligned_op(uint32_t op) { const uint32_t t = op & 15; return t == 0 || t == 7 || t == 8; }
BM2_HD bool wgs_query_op(uint32_t op) { const uint32_t t = op & 15; return t == 0 || t == 1 || t == 4 || t == 7 || t == 8; }

// the part lane `lane` of `lanes` adds over the CIGAR: [0] aligned, [1] reference length, [2] query length
BM2_HD void wgs_cigar_part(const DupCigar &c, int lane, int lanes, int64_t s[3]) {
    s[0] = s[1] = s[2] = 0;
    for (int64_t k = lane; k < c.n; k += lanes) {
        const uint32_t op = dup_op(c, k), len = op >> 4;
        if (wgs_aligned_op(op)) s[0] += len;
        if (dup_consumes_ref(op)) s[1] += len;
        if (wgs_query_op(op)) s[2] += len;
    }
}

// CG:B,I operations that lie inside the record (dup_cigar finds the tag but does not bound its array)
BM2_HD bool wgs_cigar_inside(const uint8_t *r, const DupCigar &c) {
    const BamFixed f = bam_fixed(r);
    return c.ops + 4 * c.n <= r + 4 + f.block_size;
}

// the record's status from its fixed fields and its CIGAR sums s (wgs_cigar_part summed over all lanes); sets info (g0 only when not skipped)
BM2_HD int wgs_status(const uint8_t *r, const int64_t s[3], bool cigar_inside, const int64_t *contig_off, const int32_t *contig_len, int32_t n_contigs,
                      const bm2_wgs_params_t &p, WgsInfo &info) {
    const BamFixed f = bam_fixed(r);
    info.rid = f.rid; info.g0 = info.g1 = 0; info.aligned = (int32_t) s[0]; info._pad = 0;
    if ((f.flag & 4) || f.rid == -1 || (f.flag & 0x200)) return info.status = WGS_SKIP;
    if (!cigar_inside) return info.status = WGS_ERR_CIGAR;
    if (f.rid < 0 || f.rid >= n_contigs || f.pos < 0 || (int64_t) f.pos + s[1] > (int64_t) contig_len[f.rid]) return info.status = WGS_ERR_SPAN;
    info.g0 = contig_off[f.rid] + f.pos;
    info.g1 = info.g0 + s[1];
    const int mapq = r[13];
    if (mapq < p.min_mapq) return info.status = WGS_FILT_MAPQ;
    if (f.flag & 0x400) return info.status = WGS_FILT_DUPE;
    if (!p.count_unpaired && (!(f.flag & 1) || (f.flag & 8))) return info.status = WGS_FILT_UNPAIRED;
    if (f.flag & 0x100) return info.status = WGS_DROP;
    const int32_t l_seq = bam_le32(r + 20);
    const uint8_t *q = r + 36 + f.l_read_name + 4 * f.n_cigar + (l_seq + 1) / 2;
    if (l_seq <= 0 || q[0] == 0xFF) return info.status = WGS_ERR_NOQUAL;
    if (s[2] != l_seq) return info.status = WGS_ERR_CIGAR;
    return info.status = WGS_PASS;
}

// where a record's sequence and qualities are
struct WgsSeq { const uint8_t *seq, *qual; };
BM2_HD WgsSeq wgs_seq(const uint8_t *r) {
    const BamFixed f = bam_fixed(r);
    const int32_t l_seq = bam_le32(r + 20);
    const uint8_t *s = r + 36 + f.l_read_name + 4 * f.n_cigar;
    return WgsSeq{s, s + (l_seq + 1) / 2};
}

// read base k is high-quality
BM2_HD bool wgs_hq(const WgsSeq &s, int64_t k, int min_baseq) {
    const int b = (s.seq[k >> 1] >> ((k & 1) ? 0 : 4)) & 15;
    return s.qual[k] >= min_baseq && b != 15;
}

BM2_HD bool wgs_nocall(const uint32_t *bits, int64_t g) { return (bits[g >> 5] >> (g & 31)) & 1; }

// word w of a bitset over n sorted, disjoint [beg, end) ranges (ranges[2h], ranges[2h + 1]): bit k set when locus 32w + k lies in one
BM2_HD uint32_t wgs_range_word(const int64_t *ranges, int64_t n, int64_t w) {
    const int64_t b = w * 32, e = b + 32;
    int64_t lo = 0, hi = n;                                              // the first range ending after b
    while (lo < hi) { const int64_t m = (lo + hi) / 2; if (ranges[2 * m + 1] <= b) lo = m + 1; else hi = m; }
    uint32_t v = 0;
    for (int64_t h = lo; h < n && ranges[2 * h] < e; ++h) {
        const int64_t x = bm2_max(ranges[2 * h], b) - b, y = bm2_min(ranges[2 * h + 1], e) - b;
        for (int64_t k = x; k < y; ++k) v |= 1u << k;
    }
    return v;
}

// whether a passing record has a high-quality base at locus g (a linear walk of its CIGAR; false outside its aligned blocks)
BM2_HD bool wgs_hq_at(const uint8_t *r, const DupCigar &c, int64_t g0, int64_t g, int min_baseq) {
    if (g < g0) return false;
    int64_t k = 0, at = g0;
    for (int64_t i = 0; i < c.n; ++i) {
        const uint32_t op = dup_op(c, i), len = op >> 4;
        if (wgs_aligned_op(op) && g < at + len) return wgs_hq(wgs_seq(r), k + (g - at), min_baseq);
        if (dup_consumes_ref(op)) { at += len; if (g < at) return false; }
        if (wgs_query_op(op)) k += len;
    }
    return false;
}

// the QNAME's 64-bit hash (FNV-1a), masked to 63 bits so that WGS_NOT_CANDIDATE sorts after every candidate
BM2_HD uint64_t wgs_name_hash(const uint8_t *name, int len) {
    uint64_t h = 1469598103934665603ull;
    for (int i = 0; i < len; ++i) { h ^= name[i]; h *= 1099511628211ull; }
    return h & (uint64_t) WGS_HASH_MASK;
}

// the sort key of record i: candidates (carried, or passing) by name hash; the rest after them
BM2_HD uint64_t wgs_key(const uint8_t *r, const WgsInfo &info) {
    return info.status == WGS_PASS ? wgs_name_hash(r + 36, r[12] ? r[12] - 1 : 0) : WGS_NOT_CANDIDATE;
}

// two records' names are equal, byte for byte
BM2_HD bool wgs_same_name(const uint8_t *a, const uint8_t *b) {
    if (a[12] != b[12]) return false;
    for (int i = 0; i < a[12]; ++i) if (a[36 + i] != b[36 + i]) return false;
    return true;
}

// two placed records' reference spans overlap
BM2_HD bool wgs_spans_overlap(const WgsInfo &a, const WgsInfo &b) { return a.g0 < b.g1 && b.g0 < a.g1; }

// after a window whose last record is at (rid, pos): a candidate is carried into the next window when a later record may still overlap it
BM2_HD bool wgs_carried(const WgsInfo &c, int32_t last_rid, int64_t last_g) { return c.status == WGS_PASS && c.rid == last_rid && c.g1 > last_g; }

// markdup_device.cuh — the per-template and per-group logic of bm2_mem --markdup (markdup.cu): BM2_HD functions, so that the host emulation
// tests/host_emul/markdup_emul.cpp compiles the same source.  The rule follows Picard MarkDuplicates's defaults (SUM_OF_BASE_QUALITIES, no
// optical duplicates); equality with Picard or samtools is not claimed.
//
//   primary     a record without 0x100 or 0x800 (bwa-mem2 writes exactly one per read)
//   end         of a mapped primary: (refID, unclipped 5' coordinate, reverse), packed into 64 bits by dup_end_key.  Forward: pos minus the
//               leading S/H lengths; reverse: bam_endpos - 1 plus the trailing S/H lengths.  A CIGAR moved to CG:B,I (more than 65535
//               operations) is read from there.  The coordinate may be negative or past the contig end; it is held exactly.
//   score       of a read: min(sum of base qualities >= 15, 16383); a QUAL of '*' (0xFF) scores 0
//   template    the read, or both reads of a pair; its id is the 0-based input-order index of its first read
//     pair      two primaries, both mapped: a pair entry, key (min(endA, endB), max(endA, endB)), score the sum of both reads' scores; and a
//               pair-end entry per end in the fragment space
//     fragment  one mapped primary (a single-end read, or a pair whose mate is unmapped): a fragment entry, key its end, score its read score
//     none      nothing mapped: no entry
//   groups      entries with the same key, sorted by (key, score descending, template id).  Pair space: the first entry is kept, every other is
//               a duplicate.  Fragment space: a group that holds a pair-end entry makes every fragment entry in it a duplicate; otherwise the
//               first fragment entry is kept and the others are duplicates.  Pair-end entries are never duplicates.
//
// Optical duplicates (--markdup-metrics) are counted, never marked apart: Picard's defaults give them 0x400 like any other duplicate.
//   location    of a template: the QNAME of its first record split on ':'.  Exactly 5 or 7 fields: tile, x, y from the last three, each as
//               Picard's rapidParseInt (dup_parse_int); a field without a digit means no location.  Any other count (more than 7 included):
//               no location.  The lane is not part of it.
//   class       of a pair template: the strand of its primary with 0x40 (its first primary's when neither has 0x40), Picard's
//               orientationForOpticalDuplicates split: an FR / RF group can hold both classes, counted apart; an FF / RR group holds one
//   optical     of a pair group of 2 .. DUP_OPTICAL_MAX_SET members: within one class, two members are linked when both have a location,
//               the same tile, |x1-x2| <= d and |y1-y2| <= d (in 64 bits); the count is the sum over the connected components of size - 1,
//               a member without a location being a component of its own.  This is the count of Picard's graph path and of its small-set
//               path, wherever the keeper sits.  It is at most the group's duplicates (size - 1).  Larger groups and fragment groups: 0.
//   read group  (bm2_markdup) loc's bits 2 and up hold the pair's read-group index (DUP_LOC_RG_SHIFT); dup_optical_linked compares the whole
//               loc, so members of different read groups are never linked.  bm2_mem's entries have 0 there.
//   cells       (the exact pass of groups larger than a warp, markdup.cu) members of one class, tile and read group binned by (floor(x / (d+1)),
//               floor(y / (d+1))): two members of a cell are always linked, so a cell is one component, and only the four neighbouring cells
//               behind a cell need tests - side neighbours by the cells' extreme x or y alone, diagonal ones per member by a binary search
//               in the x-sorted neighbour and its suffix extreme of y (dup_cell_diag_linked).
#pragma once
#include "hd.h"
#include "bam_sort_device.cuh"

enum { DUP_KIND_PAIR = 0, DUP_KIND_FRAG = 1, DUP_KIND_PAIR_END = 2 };

// an end: refID (< 2^30) << 34 | (coord + 2^32) (34 bits, coord in [-2^32, 2^32)) << 1 | reverse; the numeric order is (refID, coord, reverse)
BM2_HD uint64_t dup_end_key(int32_t rid, int64_t coord, int rev) {
    return (uint64_t) (uint32_t) rid << 34 | (uint64_t) (coord + ((int64_t) 1 << 32)) << 1 | (uint64_t) (rev ? 1 : 0);
}

// where a record's CIGAR operations are: inline, or in CG:B,I behind the <l_seq>S<ref_len>N placeholder
struct DupCigar { const uint8_t *ops; int64_t n; };

// the size of a tag's value of type t at p (SAMv1 §4.2.4); -1 when the type is unknown
BM2_HD int64_t dup_tag_value_size(char t, const uint8_t *p) {
    switch (t) {
        case 'A': case 'c': case 'C': return 1;
        case 's': case 'S': return 2;
        case 'i': case 'I': case 'f': return 4;
        case 'Z': case 'H': { int64_t k = 0; while (p[k]) ++k; return k + 1; }
        case 'B': {
            const char s = (char) p[0];
            const int64_t n = (int64_t) (uint32_t) bam_le32(p + 1);
            const int64_t w = (s == 'c' || s == 'C') ? 1 : (s == 's' || s == 'S') ? 2 : 4;
            return 5 + n * w;
        }
        default: return -1;
    }
}

BM2_HD DupCigar dup_cigar(const uint8_t *r) {
    const BamFixed f = bam_fixed(r);
    const uint8_t *c = r + 36 + f.l_read_name;
    DupCigar d{c, f.n_cigar};
    const int32_t l_seq = bam_le32(r + 20);
    if (f.n_cigar == 2 && ((uint32_t) bam_le32(c) & 15) == 4 && ((uint32_t) bam_le32(c) >> 4) == (uint32_t) l_seq &&
        ((uint32_t) bam_le32(c + 4) & 15) == 3) {
        const uint8_t *p = c + 8 + (l_seq + 1) / 2 + l_seq, *e = r + 4 + f.block_size;
        while (p + 3 <= e) {
            if (p[0] == 'C' && p[1] == 'G' && p[2] == 'B' && p[3] == 'I') { d.ops = p + 8; d.n = (int64_t) (uint32_t) bam_le32(p + 4); break; }
            const int64_t s = dup_tag_value_size((char) p[2], p + 3);
            if (s < 0) break;
            p += 3 + s;
        }
    }
    return d;
}

BM2_HD uint32_t dup_op(const DupCigar &c, int64_t k) { return (uint32_t) bam_le32(c.ops + 4 * k); }
BM2_HD bool dup_is_clip(uint32_t op) { return (op & 15) == 4 || (op & 15) == 5; }
BM2_HD bool dup_consumes_ref(uint32_t op) { const uint32_t t = op & 15; return t == 0 || t == 2 || t == 3 || t == 7 || t == 8; }

// the part of a sum that lane `lane` of `lanes` adds: the CIGAR's reference length, and the qualities >= 15
BM2_HD int64_t dup_ref_len_part(const DupCigar &c, int lane, int lanes) {
    int64_t s = 0;
    for (int64_t k = lane; k < c.n; k += lanes) { const uint32_t op = dup_op(c, k); if (dup_consumes_ref(op)) s += op >> 4; }
    return s;
}
BM2_HD uint32_t dup_qual_part(const uint8_t *r, int lane, int lanes) {
    const BamFixed f = bam_fixed(r);
    const int32_t l_seq = bam_le32(r + 20);
    const uint8_t *q = r + 36 + f.l_read_name + 4 * f.n_cigar + (l_seq + 1) / 2;
    if (l_seq <= 0 || q[0] == 0xFF) return 0;
    uint32_t s = 0;
    for (int32_t k = lane; k < l_seq; k += lanes) if (q[k] >= 15) s += q[k];
    return s;
}

// a mapped primary's end from its summed reference length; the leading and trailing clips are read here (at most two operations each)
BM2_HD uint64_t dup_read_end(const uint8_t *r, const DupCigar &c, int64_t ref_len) {
    const BamFixed f = bam_fixed(r);
    const int rev = (f.flag & 16) != 0;
    int64_t clip = 0;
    if (!rev) for (int64_t k = 0; k < c.n && dup_is_clip(dup_op(c, k)); ++k) clip += dup_op(c, k) >> 4;
    else for (int64_t k = c.n - 1; k >= 0 && dup_is_clip(dup_op(c, k)); --k) clip += dup_op(c, k) >> 4;
    const int64_t end = (int64_t) f.pos + (ref_len ? ref_len : 1);                     // bam_endpos
    return dup_end_key(f.rid, rev ? end - 1 + clip : (int64_t) f.pos - clip, rev);
}

BM2_HD int32_t dup_read_score(uint32_t qsum) { return (int32_t) bm2_min<uint32_t>(qsum, 16383u); }

BM2_HD bool dup_is_primary(int32_t flag) { return (flag & 0x900) == 0; }

// a template's entries from its primaries (in record order, at most two; more are an input error and give no entry): mapped[k], end[k] and
// score[k] of each.  Writes *pair (when it returns has_pair) and frag[0..*n_frag).  Returns 1 when the template has a pair or fragment entry.
BM2_HD int dup_template_entries(int n_prim, const int *mapped, const uint64_t *end, const int32_t *score, int64_t tid, bm2_dup_entry *pair,
                                int *has_pair, bm2_dup_entry *frag, int *n_frag) {
    *has_pair = 0; *n_frag = 0;
    if (n_prim == 2 && mapped[0] && mapped[1]) {
        const int lo = end[1] < end[0] ? 1 : 0;
        pair->k1 = end[lo]; pair->k2 = end[1 - lo]; pair->tid = tid; pair->score = score[0] + score[1]; pair->kind = DUP_KIND_PAIR;
        *has_pair = 1;
        for (int k = 0; k < 2; ++k) { frag[k].k1 = end[k]; frag[k].k2 = 0; frag[k].tid = tid; frag[k].score = score[k]; frag[k].kind = DUP_KIND_PAIR_END; }
        *n_frag = 2;
        return 1;
    }
    if (n_prim < 1 || n_prim > 2) return 0;
    for (int k = 0; k < n_prim; ++k)
        if (mapped[k]) { frag[0].k1 = end[k]; frag[0].k2 = 0; frag[0].tid = tid; frag[0].score = score[k]; frag[0].kind = DUP_KIND_FRAG; *n_frag = 1; return 1; }
    return 0;
}

// ---- groups ----
// the sort order: key (k1, k2), score descending, template id
BM2_HD bool dup_same_key(const bm2_dup_entry &a, const bm2_dup_entry &b) { return a.k1 == b.k1 && a.k2 == b.k2; }
BM2_HD bool dup_less(const bm2_dup_entry &a, const bm2_dup_entry &b) {
    if (a.k1 != b.k1) return a.k1 < b.k1;
    if (a.k2 != b.k2) return a.k2 < b.k2;
    if (a.score != b.score) return a.score > b.score;
    return a.tid < b.tid;
}
// entry i of a sorted group: has_pair_end, whether the group holds a pair-end entry; first, the index of its first entry that is not one
BM2_HD bool dup_is_duplicate(int kind, int has_pair_end, int64_t first, int64_t i) {
    return kind != DUP_KIND_PAIR_END && (has_pair_end || first != i);
}
// marking: a record of a duplicate template (bit tid of bits) gets 0x400 unless it is unmapped
BM2_HD uint16_t dup_marked_flag(uint16_t flag, int64_t tid, const uint64_t *bits, int64_t n_bits) {
    if ((flag & 4) || tid < 0 || tid >= n_bits) return flag;
    return ((bits[tid >> 6] >> (tid & 63)) & 1) ? (uint16_t) (flag | 0x400) : flag;
}
// the score key of the radix sort: descending score as an ascending 15-bit key (scores are at most 2 x 16383)
BM2_HD uint64_t dup_score_key(int32_t score) { return (uint64_t) (32767 - score); }

// ---- optical duplicates ----
enum { DUP_LOC_HAS = 1, DUP_LOC_REV = 2 };
constexpr int DUP_LOC_RG_SHIFT = 2;
BM2_HD uint32_t dup_loc_rg(int32_t loc) { return (uint32_t) loc >> DUP_LOC_RG_SHIFT; }
constexpr int64_t DUP_OPTICAL_MAX_SET = 300000;          // Picard's MAX_OPTICAL_DUPLICATE_SET_SIZE

// Picard's rapidParseInt of p[0..len): an optional leading '-', then the decimal digits up to the first non-digit, accumulated as a Java int
// (wrapping); false when there is no digit
BM2_HD bool dup_parse_int(const uint8_t *p, int len, int32_t *v) {
    int i = 0;
    const bool neg = len > 0 && p[0] == '-';
    if (neg) i = 1;
    uint32_t a = 0;
    bool any = false;
    for (; i < len && p[i] >= '0' && p[i] <= '9'; ++i) { a = a * 10u + (uint32_t) (p[i] - '0'); any = true; }
    *v = (int32_t) (neg ? 0u - a : a);
    return any;
}

// the location from the name's length and its colons: nc of them, c1 < c2 < c3 the last three (-1 when fewer).  Returns the loc bits (0 or
// DUP_LOC_HAS) and sets tile / x / y (0 without a location).
BM2_HD int dup_location_from_colons(const uint8_t *name, int len, int nc, int c1, int c2, int c3, int32_t *tile, int32_t *x, int32_t *y) {
    *tile = *x = *y = 0;
    if (nc != 4 && nc != 6) return 0;
    int32_t t, a, b;
    if (!dup_parse_int(name + c1 + 1, c2 - c1 - 1, &t) || !dup_parse_int(name + c2 + 1, c3 - c2 - 1, &a) || !dup_parse_int(name + c3 + 1, len - c3 - 1, &b))
        return 0;
    *tile = t; *x = a; *y = b;
    return DUP_LOC_HAS;
}

// the same from the name alone, one byte at a time (the kernel finds the colons with a ballot)
BM2_HD int dup_name_location(const uint8_t *name, int len, int32_t *tile, int32_t *x, int32_t *y) {
    int nc = 0, c1 = -1, c2 = -1, c3 = -1;
    for (int i = 0; i < len; ++i) if (name[i] == ':') { c1 = c2; c2 = c3; c3 = i; ++nc; }
    return dup_location_from_colons(name, len, nc, c1, c2, c3, tile, x, y);
}

// a pair template's class from its two primaries' flags
BM2_HD int dup_pair_class(int32_t flag0, int32_t flag1) {
    const int32_t f = (flag0 & 0x40) || !(flag1 & 0x40) ? flag0 : flag1;
    return (f & 16) ? DUP_LOC_REV : 0;
}

BM2_HD bool dup_optical_linked(const bm2_dup_loc_entry &a, const bm2_dup_loc_entry &b, int64_t d) {
    if (!(a.loc & DUP_LOC_HAS) || !(b.loc & DUP_LOC_HAS) || a.loc != b.loc || a.tile != b.tile) return false;
    const int64_t dx = (int64_t) a.x - b.x, dy = (int64_t) a.y - b.y;
    return dx <= d && -dx <= d && dy <= d && -dy <= d;
}

// a coordinate's cell: floor(v / (d + 1)), as an order-preserving unsigned 32-bit value (|v| <= 2^31, d + 1 >= 1)
BM2_HD uint32_t dup_cell(int32_t v, int64_t d) {
    const int64_t w = d + 1, c = v >= 0 ? (int64_t) v / w : -((-(int64_t) v + w - 1) / w);
    return (uint32_t) ((int32_t) c) ^ 0x80000000u;
}
// the cell sort's keys: (group, class, tile) and (cx, cy)
BM2_HD uint64_t dup_cell_hi(uint32_t group, const bm2_dup_loc_entry &e) {
    return (uint64_t) group << 33 | (uint64_t) ((e.loc & DUP_LOC_REV) ? 1 : 0) << 32 | (uint64_t) ((uint32_t) e.tile ^ 0x80000000u);
}
BM2_HD uint64_t dup_cell_lo(const bm2_dup_loc_entry &e, int64_t d) { return (uint64_t) dup_cell(e.x, d) << 32 | dup_cell(e.y, d); }

// b against the cell A behind it diagonally (cx - 1, cy - 1 when below, cy + 1 when above): A's members ax[0..n) sorted by x, with
// suf[k] the max (below) or min (above) of their y over [k, n).  Linked when some a has ax >= bx - d and ay within d of by.
BM2_HD bool dup_cell_diag_linked(const int32_t *ax, const int32_t *suf, int64_t n, int32_t bx, int32_t by, int64_t d, bool below) {
    int64_t lo = 0, hi = n;                              // the first a with ax >= bx - d
    while (lo < hi) { const int64_t m = (lo + hi) / 2; if ((int64_t) ax[m] < (int64_t) bx - d) lo = m + 1; else hi = m; }
    if (lo == n) return false;
    return below ? (int64_t) suf[lo] >= (int64_t) by - d : (int64_t) suf[lo] <= (int64_t) by + d;
}

// ---- mate pairing (bm2_markdup) ----
// a QNAME's hash: 64-bit FNV-1a over its bytes
BM2_HD uint64_t dup_name_hash(const uint8_t *name, int len) {
    uint64_t h = 14695981039346656037ull;
    for (int i = 0; i < len; ++i) { h ^= name[i]; h *= 1099511628211ull; }
    return h;
}

// one run [a, b) of the halves sorted by (hash, read group, index): ord[i] the index of the i-th.  Each half is joined to the first earlier
// half of the run that is still unjoined and whose name equals its own byte for byte; partner[] gets both indices (-1: unjoined).  This is
// a table keyed by the whole name, visited in index order, so equal hashes of different names never join.
BM2_HD void dup_pair_run(const bm2_markdup_half *h, const uint32_t *ord, int64_t a, int64_t b, const uint8_t *names, int32_t *partner) {
    for (int64_t i = a; i < b; ++i) partner[ord[i]] = -1;
    for (int64_t i = a + 1; i < b; ++i) {
        const bm2_markdup_half &u = h[ord[i]];
        for (int64_t j = a; j < i; ++j) {
            if (partner[ord[j]] != -1) continue;
            const bm2_markdup_half &v = h[ord[j]];
            bool same = u.name_len == v.name_len;
            for (int32_t k = 0; same && k < u.name_len; ++k) same = names[u.name_off + k] == names[v.name_off + k];
            if (same) { partner[ord[j]] = (int32_t) ord[i]; partner[ord[i]] = (int32_t) ord[j]; break; }
        }
    }
}

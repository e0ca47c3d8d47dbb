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

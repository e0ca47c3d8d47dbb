// bam_sort_device.cuh — the per-record logic of bm2_bam_sort_compress (bam_sort.cu): a BAM record's fixed fields (SAMv1 §4.2), its
// coordinate key and its reference end, the read-name order of bm2_bam_qname_sort_compress, and (host only) where the sorted records fall in
// the BGZF blocks.  BM2_HD functions, so that the host emulations tests/host_emul/bam_sort_emul.cpp and bamsort_emul.cpp compile the same source.
//
//   key   ((uint32) refID << 32) | ((uint32) (pos + 1) << 1) | (flag & 16 ? 1 : 0): samtools' coordinate key.  A placed unmapped mate sorts at
//         its mate's position (its refID and pos are the mate's); refID -1 sorts last.
//   end   bam_endpos: pos + the reference length of the CIGAR, pos + 1 when the record is unmapped or no operation consumes the reference.
//         A record whose CIGAR moved to CG:B,I keeps the placeholder <l_seq>S<ref_len>N, whose N already gives the span.
#pragma once
#include "hd.h"
#include "bgzf_device.cuh"
#include "bm2_b200.h"
#include <vector>

struct BamFixed { int32_t rid, pos, l_read_name, n_cigar, flag, block_size; };

BM2_HD int32_t bam_le32(const uint8_t *p) { return (int32_t) ((uint32_t) p[0] | (uint32_t) p[1] << 8 | (uint32_t) p[2] << 16 | (uint32_t) p[3] << 24); }
BM2_HD uint32_t bam_le16(const uint8_t *p) { return (uint32_t) p[0] | (uint32_t) p[1] << 8; }

// r: a record, its block_size first
BM2_HD BamFixed bam_fixed(const uint8_t *r) {
    BamFixed f;
    f.block_size = bam_le32(r);
    f.rid = bam_le32(r + 4);
    f.pos = bam_le32(r + 8);
    f.l_read_name = r[12];
    f.n_cigar = (int32_t) bam_le16(r + 16);
    f.flag = (int32_t) bam_le16(r + 18);
    return f;
}

BM2_HD uint64_t bam_coord_key(int32_t rid, int32_t pos, int32_t flag) {
    return (uint64_t) (uint32_t) rid << 32 | (uint64_t) (uint32_t) (pos + 1) << 1 | (uint64_t) ((flag & 16) ? 1 : 0);
}

BM2_HD int32_t bam_end_pos(const uint8_t *r, const BamFixed &f) {
    int64_t rlen = 0;
    if (!(f.flag & 4)) {
        const uint8_t *c = r + 36 + f.l_read_name;
        for (int i = 0; i < f.n_cigar; ++i) {
            const uint32_t op = (uint32_t) bam_le32(c + 4 * i);
            const uint32_t t = op & 15;
            if (t == 0 || t == 2 || t == 3 || t == 7 || t == 8) rlen += op >> 4;      // M D N = X consume the reference
        }
    }
    return (int32_t) (f.pos + (rlen ? rlen : 1));
}

// SAMv1 §5.3 reg2bin of [beg, end)
BM2_HD int32_t bam_reg2bin(int64_t beg, int64_t end) {
    --end;
    if (beg >> 14 == end >> 14) return (int32_t) (((1 << 15) - 1) / 7 + (beg >> 14));
    if (beg >> 17 == end >> 17) return (int32_t) (((1 << 12) - 1) / 7 + (beg >> 17));
    if (beg >> 20 == end >> 20) return (int32_t) (((1 << 9) - 1) / 7 + (beg >> 20));
    if (beg >> 23 == end >> 23) return (int32_t) (((1 << 6) - 1) / 7 + (beg >> 23));
    if (beg >> 26 == end >> 26) return (int32_t) (((1 << 3) - 1) / 7 + (beg >> 26));
    return 0;
}

// bm2_sort_rec of one record (the block and offset are the layout's): bin = reg2bin(pos, end), 4680 for refID -1 as bm2_bam_format_ex writes it
BM2_HD bm2_sort_rec bam_sort_rec(const uint8_t *r) {
    const BamFixed f = bam_fixed(r);
    bm2_sort_rec s;
    s.rid = f.rid; s.pos = f.pos;
    s.end = f.rid >= 0 ? bam_end_pos(r, f) : f.pos + 1;
    s.bin = (uint16_t) (f.rid >= 0 && f.pos >= 0 ? bam_reg2bin(f.pos, s.end) : 4680);
    s.flag = (uint16_t) f.flag;
    s.block = 0; s.offset = 0; s._pad = 0;
    return s;
}

// ---- name order (bm2_bam_qname_sort_compress, bm2_sort -n): samtools sort -n ----
// The names are compared by strnum_cmp of samtools' bam_sort.c (the 1.9-era form, recalled, not checked against samtools), bytes unsigned,
// both names NUL-terminated: outside digits, the first differing byte decides; where both sides are on a digit, the zeros and then the equal
// digits are skipped on each side, and then a longer digit run is greater (the first differing digit decides at equal lengths), a side still on
// a digit is greater, and a side that has consumed fewer bytes is greater.  A name that ends first is less.  Digit runs are never parsed into
// integers, so runs of any length compare by their length.  The order is total with the flag bits and the ordinal after the names: the host
// merge (bam_sort.h, without the ordinal), the device sort and the host emulation all call bam_qname_cmp.
BM2_HD bool bam_is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

BM2_HD int bam_strnum_cmp(const uint8_t *a, const uint8_t *b) {
    const uint8_t *pa = a, *pb = b;
    while (*pa && *pb) {
        if (bam_is_digit(*pa) && bam_is_digit(*pb)) {
            while (*pa == '0') ++pa;
            while (*pb == '0') ++pb;
            while (bam_is_digit(*pa) && bam_is_digit(*pb) && *pa == *pb) ++pa, ++pb;
            if (bam_is_digit(*pa) && bam_is_digit(*pb)) {
                int64_t i = 0;
                while (bam_is_digit(pa[i]) && bam_is_digit(pb[i])) ++i;
                return bam_is_digit(pa[i]) ? 1 : bam_is_digit(pb[i]) ? -1 : (int) *pa - (int) *pb;
            }
            if (bam_is_digit(*pa)) return 1;
            if (bam_is_digit(*pb)) return -1;
            if (pa - a != pb - b) return pa - a < pb - b ? 1 : -1;
        } else {
            if (*pa != *pb) return (int) *pa - (int) *pb;
            ++pa; ++pb;
        }
    }
    return *pa ? 1 : *pb ? -1 : 0;
}

// -1, 0 or 1: the names a and b (NUL-terminated), then flag & 0xc0 ascending, then the ordinals
BM2_HD int bam_qname_cmp(const uint8_t *a, uint32_t fa, int64_t oa, const uint8_t *b, uint32_t fb, int64_t ob) {
    const int c = bam_strnum_cmp(a, b);
    if (c) return c < 0 ? -1 : 1;
    fa &= 0xc0; fb &= 0xc0;
    if (fa != fb) return fa < fb ? -1 : 1;
    return oa < ob ? -1 : oa > ob ? 1 : 0;
}

// bam_qname_cmp of two records (block_size first) without the ordinal: the sink's merge order for bm2_sort -n
BM2_HD int bam_qname_rec_cmp(const uint8_t *a, const uint8_t *b) { return bam_qname_cmp(a + 36, bam_le16(a + 18), 0, b + 36, bam_le16(b + 18), 0); }

// the name-order entry of the record at r = buffer + start: the offset of its QNAME in the buffer << 8 | flag & 0xc0
BM2_HD uint64_t bam_qname_entry(const uint8_t *r, int64_t start) { return (uint64_t) (start + 36) << 8 | (bam_le16(r + 18) & 0xc0); }

// ---- host only: the blocks of the stream carry + sorted records, and each record's block and offset ----
// carry_len bytes of the previous call's unfinished block come first (one "record" for the cut rule: only their length matters); then the
// records at carry_len + offs[i].  The stream is cut by bgzf_cut_blocks over all of it.  When !last and the final block is not full, it is
// the new carry: it is not compressed now, and the records in it get block index n_full (block 0 of the next call's numbering is that block,
// so the caller counts blocks across calls without a gap).
struct SortLayout { std::vector<int64_t> starts; int64_t n_blocks = 0, n_full = 0; };

template <class V> inline void bam_sort_layout(int64_t carry_len, const int64_t *offs, int64_t n_recs, int64_t total, bool last, V &cut,
                                               SortLayout &L, bm2_sort_rec *recs) {
    cut.clear();
    for (int64_t i = 0; i < n_recs; ++i) cut.push_back(carry_len + offs[i]);
    L.starts.clear();
    L.n_blocks = bgzf_cut_blocks(carry_len + total, cut.data(), (int64_t) cut.size(), L.starts);
    const bool open = L.n_blocks > 0 && !last && L.starts[(size_t) L.n_blocks] - L.starts[(size_t) L.n_blocks - 1] < BGZF_BLOCK;
    L.n_full = L.n_blocks - (open ? 1 : 0);
    int64_t b = 0;
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t at = carry_len + offs[i];
        while (b + 1 < L.n_blocks && L.starts[(size_t) b + 1] <= at) ++b;
        recs[i].block = b; recs[i].offset = (int32_t) (at - L.starts[(size_t) b]);
    }
}

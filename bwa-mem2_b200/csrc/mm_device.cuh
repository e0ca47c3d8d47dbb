// mm_device.cuh — the per-record rule of bm2_multiplemetrics (mm.cu): BM2_HD functions, so that the host emulation
// tests/host_emul/multiplemetrics_emul.cpp compiles the same source.  It restates Picard CollectAlignmentSummaryMetrics and
// CollectInsertSizeMetrics at their defaults (MAPPING_QUALITY_THRESHOLD 20, BASE_QUALITY_THRESHOLD 20, MAX_INSERT_SIZE 100000, FR pairs
// expected, duplicates left out of the insert sizes, ALL_READS); byte equality with Picard is not claimed.  The formulas are mm_metrics.h's.
//
//   counted    every record without 0x100 or 0x800; category FIRST_OF_PAIR (0x1 and 0x40), SECOND_OF_PAIR (0x1 without 0x40), UNPAIRED
//   every      TOTAL_READS, the read-length histogram (l_seq), the no-calls (read base N) by cycle in sequencing order (reversed for 0x10)
//   PF         no 0x200: PF_READS; XN:i:1 -> PF_NOISE_READS; with 0x4, PCT_ADAPTER when the first 16 stored bases equal the first 16 of a
//              default adapter, or their reverse complement, with at most 1 mismatch (a read N is never one; shorter reads never match)
//   aligned    PF without 0x4: PF_READS_ALIGNED; 0x1 without 0x8 -> in pairs; 0x1 without 0x2 -> improper; no 0x10 -> forward; the S and H
//              bases; the 3' soft clip (the S next to the read's 3' end, past any H: the last operation on the forward strand, the first on
//              the reverse) and whether there is one; the I and D operations; over the M / = / X bases, the aligned bases and the
//              mismatches: the read letter (=ACMGRSVTWYHKDBN[nibble]) differs from the reference letter (an .amb hole's letter, upper
//              case, or ACGT[pac code]).
//   HQ         an aligned record with MAPQ >= 20: its reads, bases, bases of quality >= 20 (none under QUAL '*'), mismatches, one entry of its
//              mismatch count in the per-read histogram, the chimera denominator; chimeric when 0x1 without 0x8 and (the mate on another
//              contig, |TLEN| > 100000 or an orientation other than FR), else when it has an SA tag
//   insert     a counted record with 0x1, without 0x4, 0x8, 0x40 or 0x400, and TLEN != 0: |TLEN| in its orientation's histogram
//              (htsjdk's SamPairUtil.getPairOrientation, mm_orientation)
//   errors     a counted record with l_seq 0 or above MM_MAX_LSEQ; an aligned record whose CG:B,I runs past the record, whose refID is not a
//              contig or whose alignment runs past its contig's end, or whose CIGAR query length is not l_seq (checked in that order)
//
// GC bias (CollectGcBiasMetrics at its defaults: SCAN_WINDOW_SIZE 100, MINIMUM_GENOME_FRACTION 1e-5, ALL_READS, no bisulfite, duplicates
// kept), only when bm2_mm_gc_set turned it on; the formulas and text are mm_gcbias.h's.  Picard's loops are restated from memory:
//   letters    mm_ref_letter's; G and C are GC, N is N, every other letter (IUPAC S included) neither; the denominator is W = 100, Ns included
//   windows    per contig of length L, the starts 1 <= i < L - W (Picard's loop skips window 0 and the last full window); a window with more
//              than 4 Ns is not binned, else its bin is gc * 100 / W; windows never span two contigs
//   records    counted as above (no 0x100 or 0x800); TOTAL_CLUSTERS without 0x1 or with 0x40; placed (MMB_PLACED): without 0x4, whatever
//              0x200 and 0x400 say -> ALIGNED_READS, and the span and CIGAR errors above apply to it as to an aligned record.  Its window is
//              p = pos + 1 forward (Picard's 1-based alignment start used as a 0-based index) or p = pos + ref_len - W reverse; when p is a
//              counted, binned window of the contig the record adds 1 read start, l_seq bases and its errors (the mismatches over M / = / X,
//              plus the I and D lengths) to that bin.  Windows at p = L - W or beyond enter no bin (Picard would read bin 0 or fail there).
#pragma once
#include "hd.h"
#include "bam_sort_device.cuh"
#include "markdup_device.cuh"
#include "wgs_device.cuh"

enum { MM_FIRST, MM_SECOND, MM_UNPAIRED, MM_NCAT };
// the per-category counters
enum { MM_TOTAL, MM_PF, MM_NOISE, MM_ADAPTER, MM_ALIGNED, MM_IN_PAIRS, MM_IMPROPER, MM_FORWARD, MM_SOFTCLIP, MM_HARDCLIP, MM_SC3_SUM,
       MM_SC3_READS, MM_INDELS, MM_ALIGNED_BASES, MM_MISMATCH, MM_HQ_READS, MM_HQ_BASES, MM_HQ_Q20, MM_HQ_MISMATCH, MM_CHIM_DEN, MM_CHIM,
       MM_NCOUNT };
static_assert(MM_NCOUNT == BM2_MM_NCOUNT && MM_NCAT == BM2_MM_NCAT, "bm2_mm_result_t's counters");
enum { MM_FR, MM_RF, MM_TANDEM, MM_NORIENT };
// a record's bits
enum { MMB_COUNTED = 1, MMB_PF = 2, MMB_NOISE = 4, MMB_ADAPTER = 8, MMB_ALIGNED = 16, MMB_IN_PAIRS = 32, MMB_IMPROPER = 64, MMB_FORWARD = 128,
       MMB_HQ = 256, MMB_CHIM = 512, MMB_INSERT = 1024, MMB_REV = 2048, MMB_NOQUAL = 4096, MMB_PLACED = 8192 };
enum { MM_ERR_LSEQ = 1, MM_ERR_SPAN = 2, MM_ERR_CIGAR = 3 };

constexpr int MM_MIN_MAPQ = 20, MM_MIN_BASEQ = 20;
constexpr int64_t MM_CHIMERA_INSERT = 100000;          // MAX_INSERT_SIZE
constexpr int32_t MM_MAX_LSEQ = 1 << 20;               // a chosen bound: the per-cycle and per-length arrays stay dense
constexpr int64_t MM_DENSE_INSERT = 1 << 20;           // insert sizes below this go to dense bins, larger ones to a list
constexpr int MM_ADAPTER_LEN = 16, MM_N_ADAPTER_KMERS = 12;
constexpr int MM_GC_W = 100, MM_GC_BINS = 101, MM_GC_MAX_N = 4;  // SCAN_WINDOW_SIZE, the bins 0..100, the most Ns of a binned window

// a record's classification, from the check kernel to the count kernel
struct MmInfo {
    int64_t g0;              // the locus of its first aligned base (aligned records)
    int64_t insert;          // |TLEN| (MMB_INSERT)
    int32_t bits, err, cat, l_seq;
    int32_t aligned, softclip, hardclip, sc3, indels, orient;
};

BM2_HD int mm_category(int32_t flag) { return !(flag & 1) ? MM_UNPAIRED : (flag & 0x40) ? MM_FIRST : MM_SECOND; }

// htsjdk's getPairOrientation for a read with both ends mapped: 1-based starts, the read's alignment end start + ref_len - 1
BM2_HD int mm_orientation(int32_t flag, int32_t pos, int32_t mpos, int32_t tlen, int64_t ref_len) {
    const bool rev = flag & 0x10, mrev = flag & 0x20;
    if (rev == mrev) return MM_TANDEM;
    const int64_t pos5 = rev ? (int64_t) mpos + 1 : (int64_t) pos + 1;
    const int64_t neg5 = rev ? (int64_t) pos + ref_len : (int64_t) pos + 1 + tlen;
    return pos5 < neg5 ? MM_FR : MM_RF;
}

// the type byte of tag (a, b) whose value lies inside the record, or null
BM2_HD const uint8_t *mm_tag(const uint8_t *r, char a, char b) {
    const BamFixed f = bam_fixed(r);
    const int32_t l_seq = bam_le32(r + 20);
    const uint8_t *p = r + 36 + f.l_read_name + 4 * (int64_t) f.n_cigar + (l_seq + 1) / 2 + l_seq, *e = r + 4 + f.block_size;
    while (p + 3 <= e) {
        const char t = (char) p[2];
        int64_t s;
        if (t == 'Z' || t == 'H') { const uint8_t *q = p + 3; while (q < e && *q) ++q; s = q - (p + 3) + 1; }
        else if (t == 'B' && p + 8 > e) return nullptr;
        else s = dup_tag_value_size(t, p + 3);
        if (s < 0 || p + 3 + s > e) return nullptr;
        if (p[0] == a && p[1] == b) return p + 2;
        p += 3 + s;
    }
    return nullptr;
}

// an integer tag's value is 1
BM2_HD bool mm_int_tag_is_one(const uint8_t *t) {
    if (!t) return false;
    switch ((char) t[0]) {
        case 'c': return (int8_t) t[1] == 1;
        case 'C': return t[1] == 1;
        case 's': case 'S': return bam_le16(t + 1) == 1;
        case 'i': case 'I': return bam_le32(t + 1) == 1;
        default: return false;
    }
}

BM2_HD char mm_read_letter(int nibble) { return "=ACMGRSVTWYHKDBN"[nibble & 15]; }
BM2_HD int mm_nibble(const uint8_t *seq, int64_t k) { return (seq[k >> 1] >> ((k & 1) ? 0 : 4)) & 15; }

// the first 16 stored bases match one of the kmers (the adapters' first 16 bases and their reverse complements) with at most one mismatch
BM2_HD bool mm_is_adapter(const uint8_t *seq, int32_t l_seq, const char (*kmers)[MM_ADAPTER_LEN]) {
    if (l_seq < MM_ADAPTER_LEN) return false;
    for (int a = 0; a < MM_N_ADAPTER_KMERS; ++a) {
        int mm = 0;
        for (int k = 0; k < MM_ADAPTER_LEN && mm <= 1; ++k) {
            const int nb = mm_nibble(seq, k);
            mm += nb != 15 && mm_read_letter(nb) != kmers[a][k];
        }
        if (mm <= 1) return true;
    }
    return false;
}

// the part lane `lane` of `lanes` adds over the CIGAR: [0] soft-clipped bases, [1] hard-clipped bases, [2] I and D operations
BM2_HD void mm_clip_part(const DupCigar &c, int lane, int lanes, int64_t s[3]) {
    s[0] = s[1] = s[2] = 0;
    for (int64_t k = lane; k < c.n; k += lanes) {
        const uint32_t op = dup_op(c, k), t = op & 15;
        if (t == 4) s[0] += op >> 4;
        if (t == 5) s[1] += op >> 4;
        if (t == 1 || t == 2) s[2] += 1;
    }
}

// the 3' soft clip: the S operation next to the read's 3' end, past any H
BM2_HD int32_t mm_sc3(const DupCigar &c, bool rev) {
    int64_t k = rev ? 0 : c.n - 1;
    const int64_t d = rev ? 1 : -1;
    while (k >= 0 && k < c.n && (dup_op(c, k) & 15) == 5) k += d;
    return k >= 0 && k < c.n && (dup_op(c, k) & 15) == 4 ? (int32_t) (dup_op(c, k) >> 4) : 0;
}

// the record's classification from its fixed fields, the CIGAR sums s (wgs_cigar_part: aligned, reference, query) and t (mm_clip_part),
// both summed over all lanes, and whether a CG:B,I CIGAR lies inside the record.  gc (GC bias on): the checks of an aligned record apply to
// every placed one, which gets MMB_PLACED and g0.
BM2_HD void mm_classify(const uint8_t *r, const int64_t s[3], const int64_t t[3], bool cigar_inside, const int64_t *contig_off,
                        const int32_t *contig_len, int32_t n_contigs, const char (*kmers)[MM_ADAPTER_LEN], MmInfo &in, bool gc = false) {
    const BamFixed f = bam_fixed(r);
    in.g0 = 0; in.insert = 0; in.bits = 0; in.err = 0; in.cat = 0; in.aligned = in.softclip = in.hardclip = in.sc3 = in.indels = in.orient = 0;
    in.l_seq = bam_le32(r + 20);
    if (f.flag & 0x900) return;
    in.cat = mm_category(f.flag);
    int32_t b = MMB_COUNTED;
    if (in.l_seq <= 0 || in.l_seq > MM_MAX_LSEQ) { in.err = MM_ERR_LSEQ; return; }
    const uint8_t *seq = r + 36 + f.l_read_name + 4 * (int64_t) f.n_cigar;
    if (seq[(in.l_seq + 1) / 2] == 0xFF) b |= MMB_NOQUAL;
    if (f.flag & 0x10) b |= MMB_REV;
    const bool pf = !(f.flag & 0x200), aligned = pf && !(f.flag & 4), placed = gc ? !(f.flag & 4) : aligned;
    if (placed) {
        if (!cigar_inside) { in.err = MM_ERR_CIGAR; return; }
        if (f.rid < 0 || f.rid >= n_contigs || f.pos < 0 || (int64_t) f.pos + s[1] > (int64_t) contig_len[f.rid]) { in.err = MM_ERR_SPAN; return; }
        if (s[2] != in.l_seq) { in.err = MM_ERR_CIGAR; return; }
    }
    const int32_t mrid = bam_le32(r + 24), mpos = bam_le32(r + 28), tlen = bam_le32(r + 32);
    const int64_t ref_len = cigar_inside ? s[1] : 0;
    if (gc && placed) { b |= MMB_PLACED; in.g0 = contig_off[f.rid] + f.pos; }
    if (pf) {
        b |= MMB_PF;
        if (mm_int_tag_is_one(mm_tag(r, 'X', 'N'))) b |= MMB_NOISE;
        if ((f.flag & 4) && mm_is_adapter(seq, in.l_seq, kmers)) b |= MMB_ADAPTER;
    }
    if (aligned) {
        b |= MMB_ALIGNED;
        in.g0 = contig_off[f.rid] + f.pos;
        const bool mated = (f.flag & 1) && !(f.flag & 8);
        if (mated) b |= MMB_IN_PAIRS;
        if ((f.flag & 1) && !(f.flag & 2)) b |= MMB_IMPROPER;
        if (!(f.flag & 0x10)) b |= MMB_FORWARD;
        in.aligned = (int32_t) s[0]; in.softclip = (int32_t) t[0]; in.hardclip = (int32_t) t[1]; in.indels = (int32_t) t[2];
        in.sc3 = mm_sc3(dup_cigar(r), f.flag & 0x10);
        if (r[13] >= MM_MIN_MAPQ) {
            b |= MMB_HQ;
            const bool chim = mated ? (mrid != f.rid || (tlen < 0 ? -(int64_t) tlen : (int64_t) tlen) > MM_CHIMERA_INSERT ||
                                       mm_orientation(f.flag, f.pos, mpos, tlen, ref_len) != MM_FR)
                                    : mm_tag(r, 'S', 'A') != nullptr;
            if (chim) b |= MMB_CHIM;
        }
    }
    if ((f.flag & 1) && !(f.flag & (4 | 8 | 0x40 | 0x400)) && tlen != 0) {
        b |= MMB_INSERT;
        in.insert = tlen < 0 ? -(int64_t) tlen : (int64_t) tlen;
        in.orient = mm_orientation(f.flag, f.pos, mpos, tlen, ref_len);
    }
    in.bits = b;
}

// a counted record's counters (v[MM_NCOUNT], added to its category) from its classification and its per-base sums: the mismatches and the
// bases of quality >= 20 over its aligned bases
BM2_HD void mm_record_counts(const MmInfo &in, int64_t mism, int64_t q20, int64_t v[MM_NCOUNT]) {
    for (int k = 0; k < MM_NCOUNT; ++k) v[k] = 0;
    const int32_t b = in.bits;
    v[MM_TOTAL] = 1;
    v[MM_PF] = (b & MMB_PF) != 0; v[MM_NOISE] = (b & MMB_NOISE) != 0; v[MM_ADAPTER] = (b & MMB_ADAPTER) != 0;
    if (!(b & MMB_ALIGNED)) return;
    v[MM_ALIGNED] = 1; v[MM_IN_PAIRS] = (b & MMB_IN_PAIRS) != 0; v[MM_IMPROPER] = (b & MMB_IMPROPER) != 0; v[MM_FORWARD] = (b & MMB_FORWARD) != 0;
    v[MM_SOFTCLIP] = in.softclip; v[MM_HARDCLIP] = in.hardclip; v[MM_SC3_SUM] = in.sc3; v[MM_SC3_READS] = in.sc3 > 0; v[MM_INDELS] = in.indels;
    v[MM_ALIGNED_BASES] = in.aligned; v[MM_MISMATCH] = mism;
    if (!(b & MMB_HQ)) return;
    v[MM_HQ_READS] = 1; v[MM_HQ_BASES] = in.aligned; v[MM_HQ_Q20] = q20; v[MM_HQ_MISMATCH] = mism;
    v[MM_CHIM_DEN] = 1; v[MM_CHIM] = (b & MMB_CHIM) != 0;
}

// the reference letter at locus g: an .amb hole's letter in upper case (holes: n sorted, disjoint [beg, end) pairs), else ACGT[pac code]
BM2_HD char mm_ref_letter(const uint8_t *pac, const uint32_t *hole_bits, const int64_t *holes, const char *hole_char, int64_t n, int64_t g) {
    if (wgs_nocall(hole_bits, g)) {
        int64_t lo = 0, hi = n;                                          // the last hole beginning at or before g
        while (hi - lo > 1) { const int64_t m = (lo + hi) / 2; if (holes[2 * m] <= g) lo = m; else hi = m; }
        const char c = hole_char[lo];
        return c >= 'a' && c <= 'z' ? (char) (c - 32) : c;
    }
    return "ACGT"[(pac[g >> 2] >> ((~g & 3) << 1)) & 3];
}

// an aligned base: read base k at locus g; adds to the mismatches and the bases of quality >= 20
BM2_HD void mm_base(const WgsSeq &sq, bool noqual, int64_t k, int64_t g, const uint8_t *pac, const uint32_t *hole_bits, const int64_t *holes,
                    const char *hole_char, int64_t n_holes, uint32_t &mism, uint32_t &q20) {
    mism += mm_read_letter(mm_nibble(sq.seq, k)) != mm_ref_letter(pac, hole_bits, holes, hole_char, n_holes, g);
    q20 += !noqual && sq.qual[k] >= MM_MIN_BASEQ;
}

// ---- GC bias ----

// a record's GC bias placement, from the check kernel to the count kernel (GC bias on only)
struct MmGc {
    int64_t gw;              // the first locus of the record's window when it is a counted window of the contig (1 <= p < L - W), else -1
    int64_t idlen;           // the summed I and D lengths
};

// the summed I and D lengths lane `lane` of `lanes` adds over the CIGAR
BM2_HD int64_t mm_gc_idlen_part(const DupCigar &c, int lane, int lanes) {
    int64_t s = 0;
    for (int64_t k = lane; k < c.n; k += lanes) {
        const uint32_t op = dup_op(c, k), t = op & 15;
        if (t == 1 || t == 2) s += op >> 4;
    }
    return s;
}

// the first locus of a placed record's window (ref_len: its CIGAR's reference length), or -1 when the window is not one the reference scan
// counts; whether the window has more than 4 Ns is left to the caller
BM2_HD int64_t mm_gc_window(const uint8_t *r, int64_t ref_len, const int64_t *contig_off, const int32_t *contig_len) {
    const BamFixed f = bam_fixed(r);
    const int64_t p = (f.flag & 0x10) ? (int64_t) f.pos + ref_len - MM_GC_W : (int64_t) f.pos + 1;
    return p >= 1 && p < (int64_t) contig_len[f.rid] - MM_GC_W ? contig_off[f.rid] + p : -1;
}

// a reference letter's class: 1 GC, 2 N, 0 neither
BM2_HD int mm_gc_class(char c) { return c == 'G' || c == 'C' ? 1 : c == 'N' ? 2 : 0; }

// the bin of a window with gc GC letters and n Ns, or -1 when it is not binned
BM2_HD int mm_gc_bin(int gc, int n) { return n > MM_GC_MAX_N ? -1 : gc * 100 / MM_GC_W; }

// the GC and N bitsets of locus word w (loci 32w .. 32w + 31, bit k for locus 32w + k; no bit at or past l_pac): ACGT[pac code] outside the
// holes, the hole's letter (upper case) inside, found by a binary search of the holes as wgs_range_word does
BM2_HD void mm_gc_word(const uint8_t *pac, const uint32_t *hole_bits, const int64_t *holes, const char *hole_char, int64_t n_holes, int64_t l_pac,
                       int64_t w, uint32_t &gcm, uint32_t &nm) {
    gcm = nm = 0;
    const int64_t b = w * 32;
    if (b >= l_pac) return;
    const int64_t pb = (l_pac + 3) / 4;
    uint64_t v = 0;
    if (8 * w + 8 <= pb) v = *(const uint64_t *) (pac + 8 * w);
    else for (int64_t j = 8 * w; j < pb; ++j) v |= (uint64_t) pac[j] << (8 * (j - 8 * w));
    for (int k = 0; k < 32; ++k) {
        const uint32_t code = (uint32_t) (v >> (8 * (k >> 2) + 2 * (3 - (k & 3)))) & 3;
        gcm |= ((code ^ (code >> 1)) & 1) << k;                         // C (1) and G (2)
    }
    const uint32_t hb = hole_bits[w];
    if (hb) {
        gcm &= ~hb;
        int64_t lo = 0, hi = n_holes;                                    // the first hole ending after b
        while (lo < hi) { const int64_t m = (lo + hi) / 2; if (holes[2 * m + 1] <= b) lo = m + 1; else hi = m; }
        for (int64_t h = lo; h < n_holes && holes[2 * h] < b + 32; ++h) {
            const int64_t x = bm2_max(holes[2 * h], b) - b, y = bm2_min(holes[2 * h + 1], b + 32) - b;
            const uint32_t m = (y - x >= 32 ? ~0u : ((1u << (y - x)) - 1)) << x;
            char c = hole_char[h];
            c = c >= 'a' && c <= 'z' ? (char) (c - 32) : c;
            const int cls = mm_gc_class(c);
            if (cls == 1) gcm |= m;
            if (cls == 2) nm |= m;
        }
    }
    if (b + 32 > l_pac) { const uint32_t keep = (1u << (l_pac - b)) - 1; gcm &= keep; nm &= keep; }
}

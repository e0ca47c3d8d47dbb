// bam2fq_device.cuh — the per-record rule of bm2_bam2fq (bam2fq.cu): BM2_HD functions, so that the host emulation
// tests/host_emul/bam2fq_emul.cpp compiles the same source.  Where it follows `samtools fastq` at its defaults it says so; byte equality
// with samtools is not claimed.
//
//   kept      a record without 0x100 and 0x800 (samtools fastq's default -F 0x900); QC-fail and duplicate records are kept
//   kind      of a kept record: READ1 (0x40 without 0x80), READ2 (0x80 without 0x40), other (both or neither, whatever 0x1 says)
//   text      '@' QNAME [/1 | /2], SEQ, '+', QUAL + 33, one line each; the suffix only on a READ1 or READ2, and only when suffixes are on.
//             A record with 0x10 is written reverse-complemented with its qualities reversed; the complement of a 4-bit code is its bit
//             reversal (htslib's seq_comp_table).  A record whose QUAL is '*' (0xFF) is a FASTA record: '>' QNAME [/1 | /2] and SEQ (our
//             choice: samtools fills in a default quality)
//   errors    a kept record with l_seq 0, or with a quality above 93 (it would not be printable)
#pragma once
#include "hd.h"
#include "bam_sort_device.cuh"

enum { B2F_SKIP = 0, B2F_READ1 = 1, B2F_READ2 = 2, B2F_OTHER = 3 };
enum { B2F_ERR_NONE = 0, B2F_ERR_EMPTY = 1, B2F_ERR_QUAL = 2 };

BM2_HD int b2f_kind(uint32_t flag) {
    if (flag & 0x900) return B2F_SKIP;
    const uint32_t e = flag & 0xC0;
    return e == 0x40 ? B2F_READ1 : e == 0x80 ? B2F_READ2 : B2F_OTHER;
}

// the complement of a 4-bit base code: its bit reversal (=, A<->T, C<->G, M<->K, R<->Y, S, W, H<->D, V<->B, N)
BM2_HD uint32_t b2f_comp(uint32_t c) { return (c & 1) << 3 | (c & 2) << 1 | (c & 4) >> 1 | (c & 8) >> 3; }
BM2_HD uint8_t b2f_letter(uint32_t c) { return (uint8_t) "=ACMGRSVTWYHKDBN"[c & 15]; }

struct B2fView {
    const uint8_t *name, *seq, *qual;
    int32_t name_len, l_seq;
    uint32_t flag;
    int suffix;                  // 0, or the digit '1' / '2' after a '/'
    bool fasta;
};

BM2_HD B2fView b2f_view(const uint8_t *r, int suffixes) {
    const BamFixed f = bam_fixed(r);
    B2fView v;
    v.flag = (uint32_t) f.flag;
    v.l_seq = bam_le32(r + 20);
    v.name = r + 36;
    v.name_len = bm2_max<int32_t>(f.l_read_name - 1, 0);
    v.seq = r + 36 + f.l_read_name + 4 * (int64_t) f.n_cigar;
    v.qual = v.seq + (v.l_seq + 1) / 2;
    const int k = b2f_kind(v.flag);
    v.suffix = suffixes && (k == B2F_READ1 || k == B2F_READ2) ? (k == B2F_READ1 ? '1' : '2') : 0;
    v.fasta = v.l_seq > 0 && v.qual[0] == 0xFF;
    return v;
}

BM2_HD int64_t b2f_head_len(const B2fView &v) { return 1 + (int64_t) v.name_len + (v.suffix ? 2 : 0) + 1; }
BM2_HD int64_t b2f_text_len(const B2fView &v) {
    return b2f_head_len(v) + (int64_t) v.l_seq + 1 + (v.fasta ? 0 : 2 + (int64_t) v.l_seq + 1);
}

// the j-th base and quality character as written (reverse-complemented / reversed with 0x10)
BM2_HD uint8_t b2f_base_at(const B2fView &v, int64_t j) {
    const bool rev = (v.flag & 16) != 0;
    const int64_t i = rev ? v.l_seq - 1 - j : j;
    const uint32_t c = (v.seq[i >> 1] >> ((~i & 1) << 2)) & 15;
    return b2f_letter(rev ? b2f_comp(c) : c);
}
BM2_HD uint8_t b2f_qual_at(const B2fView &v, int64_t j) {
    return (uint8_t) (v.qual[(v.flag & 16) ? v.l_seq - 1 - j : j] + 33);
}

// the part of a kept record's check that lane `lane` of `lanes` does: B2F_ERR_QUAL when one of its qualities is above 93
BM2_HD int b2f_check_part(const B2fView &v, int lane, int lanes) {
    if (v.fasta) return B2F_ERR_NONE;
    for (int64_t j = lane; j < v.l_seq; j += lanes) if (v.qual[j] > 93) return B2F_ERR_QUAL;
    return B2F_ERR_NONE;
}

// the text bytes of a record that lane `lane` of `lanes` writes at out: byte k of each line goes to lane k mod lanes, so a warp writes
// 32 consecutive bytes of a line at a time
BM2_HD void b2f_write_part(const B2fView &v, uint8_t *out, int lane, int lanes) {
    if (lane == 0) out[0] = v.fasta ? '>' : '@';
    for (int64_t k = lane; k < v.name_len; k += lanes) out[1 + k] = v.name[k];
    int64_t at = 1 + v.name_len;
    if (v.suffix && lane == 0) { out[at] = '/'; out[at + 1] = (uint8_t) v.suffix; }
    at += v.suffix ? 2 : 0;
    if (lane == 0) out[at] = '\n';
    ++at;
    for (int64_t j = lane; j < v.l_seq; j += lanes) out[at + j] = b2f_base_at(v, j);
    at += v.l_seq;
    if (lane == 0) out[at] = '\n';
    ++at;
    if (v.fasta) return;
    if (lane == 0) { out[at] = '+'; out[at + 1] = '\n'; }
    at += 2;
    for (int64_t j = lane; j < v.l_seq; j += lanes) out[at + j] = b2f_qual_at(v, j);
    at += v.l_seq;
    if (lane == 0) out[at] = '\n';
}

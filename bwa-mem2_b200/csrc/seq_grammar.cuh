// seq_grammar.cuh — one kseq_read call (reference src/kseq.h:185-227) restated over line ends instead of bytes, as a BM2_HD function:
// bm2_seq_encode (fastq.cu) runs it on the GPU from every candidate record start and again, one warp per record, to gather the bytes;
// bm2_mem's chunker runs it on the host; tests/host_emul/seq_emul.cpp compiles it with g++.
//
// The grammar, as kseq reads a stream (last_char = 0 at the start and after a FASTQ record, else the header character already read):
//   header     after a FASTQ record or at the start: the first '>' or '@' byte anywhere (junk before it, even mid-line, is skipped);
//              after a FASTA record: the first byte of the line that ended its sequence.  A header character that is the last byte of
//              the input is no record (ks_getuntil returns -1).
//   name       up to the first isspace byte (' ' '\t' '\n' '\v' '\f' '\r'); unless that byte is '\n', the rest of the line is the comment;
//              then trim_readno (src/bwa.cpp:62-66) drops a final "/<digit>" from a name longer than two bytes.
//   sequence   lines until one that starts with '>', '@' or '+' (or the end of input); an empty line is skipped.  Each line is its first
//              byte (ks_getc) plus the rest of the line (ks_getuntil2 with append).
//   '+'        FASTQ: the rest of the '+' line is skipped; no line end after it is a malformed record.
//   quality    whole lines appended (an empty one too) while l_qual < l_seq, at least one line; l_qual != l_seq is a malformed record.
//   '\r' rule  after each ks_getuntil2 call that found any byte left (src/kseq.h:148): the last byte of the string built so far is dropped
//              when it is '\r' and the string is longer than one byte.  It can reach back into an earlier line: an empty quality line after
//              "A\r\r" turns "A\r" into "A".  The state kept for it is the length L and the count R of '\r' bytes that end the string.
// Bytes are emitted through a sink as (buffer position, count, offset in the string): every popped byte is the last one written, so
// writing each line's kept bytes at the current length and shortening the length on a pop leaves exactly the string kseq builds.
#pragma once
#include "hd.h"
#include <stdint.h>

struct SeqRec {
    int64_t next;                 // header character of the next record, or n (end of input)
    int64_t end;                  // first byte after the record's last line
    int64_t name_beg, cmt_beg;    // name (after the header character) and comment positions
    int32_t name_len, cmt_len;    // name length after trim_readno; comment length after the '\r' rule (0: none)
    int64_t seq_first, seq_last;  // starts of the first and the last sequence line (-1: none)
    int64_t plus, qual_last;      // position of the '+' and start of the last quality line (-1: FASTA)
    int32_t l_seq, l_qual;
    int32_t lines;                // lines from the header line to the last line read
    int32_t name_full_len;        // name length as kseq_read returns it, before trim_readno (bm2_fasta_pack keeps it)
    int8_t status;                // SEQ_OK, SEQ_NONE (no record: end of input), SEQ_BAD (kseq_read would return -2)
    int8_t simple;                // four-line FASTQ that fastq_spans_kernel parses to the same record (see seq_record)
};
enum { SEQ_OK = 0, SEQ_NONE = 1, SEQ_BAD = 2 };

BM2_HD bool seq_isspace(unsigned char c) { return c == ' ' || (c >= '\t' && c <= '\r'); }

struct SeqNullSink {
    BM2_HD void seq(int64_t, int64_t, int64_t) const {}
    BM2_HD void qual(int64_t, int64_t, int64_t) const {}
};

// one string (sequence or qualities) under construction: length, trailing '\r' count
struct SeqAcc {
    int64_t L = 0, R = 0;
    // a line [b, e) appended; rule: whether the ks_getuntil2 call found bytes left.  Returns the number of the line's bytes that stay
    template <class Src> BM2_HD int64_t push(const Src &s, int64_t b, int64_t e, bool rule) {
        const int64_t len = e - b;
        int64_t t = 0;
        while (t < len && s.raw[e - 1 - t] == '\r') ++t;
        R = t == len ? R + len : t;
        L += len;
        if (rule && L > 1 && R > 0) { --L; --R; return len - 1; }
        return len;
    }
};

// one kseq_read from the header character at h.  Src: raw, n, eol(p) (first '\n' at or after p, else n), hdr(p) (first '>' or '@' at or
// after p, else n).  simple: a FASTQ record of exactly four lines, '@' header, the name ended by ' ', '\t', the line end or an '\r' that
// ends the line, no sequence or quality line that is a lone '\r', and a sequence that is not empty - on such a record fastq_spans_kernel's
// rules give kseq's name, comment, sequence and qualities (its '\r' strip differs from kseq's only on one-byte lines; an empty sequence has
// no qualities for kseq, so SAM prints '*', which only bm2_seq_encode's qual_present carries).
template <class Src, class Sink> BM2_HD SeqRec seq_record(const Src &s, int64_t h, const Sink &sink) {
    const char *raw = s.raw; const int64_t n = s.n;
    SeqRec r;
    r.next = n; r.end = n; r.name_beg = h + 1; r.cmt_beg = 0; r.name_len = 0; r.cmt_len = 0;
    r.seq_first = r.seq_last = r.plus = r.qual_last = -1; r.l_seq = r.l_qual = 0; r.lines = 1; r.name_full_len = 0; r.status = SEQ_NONE; r.simple = 0;
    if (h + 1 >= n) return r;
    // name: up to the first isspace byte (ks_getuntil, KS_SEP_SPACE)
    int64_t i = h + 1;
    while (i < n && !seq_isspace((unsigned char) raw[i])) ++i;
    int32_t nl = (int32_t) (i - (h + 1));
    r.name_full_len = nl;
    if (nl > 2 && raw[h + nl - 1] == '/' && raw[h + nl] >= '0' && raw[h + nl] <= '9') nl -= 2;
    r.name_len = nl;
    const unsigned char c0 = i < n ? (unsigned char) raw[i] : 0;
    int64_t p = i < n ? i + 1 : n;
    bool name_ok = c0 == ' ' || c0 == '\t' || c0 == '\n' || (c0 == '\r' && (i + 1 == n || raw[i + 1] == '\n'));
    if (c0 != '\n' && p < n) {                          // comment: the rest of the line (ks_getuntil, KS_SEP_LINE)
        const int64_t e = s.eol(p);
        int64_t len = e - p;
        if (len > 1 && raw[e - 1] == '\r') --len;
        r.cmt_beg = p; r.cmt_len = (int32_t) len;
        p = e < n ? e + 1 : n;
    }
    // sequence lines
    SeqAcc sq; bool lone_cr = false;
    int c = -1;
    while (p < n) {
        c = (unsigned char) raw[p];
        if (c == '>' || c == '@' || c == '+') break;
        ++r.lines;
        if (c == '\n') { ++p; c = -1; continue; }
        const bool rule = p + 1 < n;
        const int64_t e = rule ? s.eol(p + 1) : n;
        if (e - p == 1 && c == '\r') lone_cr = true;
        if (r.seq_first < 0) r.seq_first = p;
        r.seq_last = p;
        const int64_t at = sq.L;
        const int64_t k = sq.push(s, p, e, rule);
        sink.seq(p, k, at);
        p = e < n ? e + 1 : n;
        c = -1;
    }
    r.l_seq = (int32_t) sq.L;
    if (c != '+') {                                     // FASTA: the next header is the byte that ended the sequence
        r.status = SEQ_OK; r.end = p; r.next = p;
        return r;
    }
    ++r.lines;
    r.plus = p;
    const int64_t pe = p + 1 < n ? s.eol(p + 1) : n;
    if (pe >= n) { r.status = SEQ_BAD; r.end = n; return r; }
    p = pe + 1;
    SeqAcc qa;
    do {
        if (p >= n) break;                              // ks_getuntil2 returns -1: nothing appended, no rule
        const int64_t e = s.eol(p);
        ++r.lines;
        if (e - p == 1 && raw[p] == '\r') lone_cr = true;
        r.qual_last = p;
        const int64_t at = qa.L;
        const int64_t k = qa.push(s, p, e, true);
        sink.qual(p, k, at);
        p = e < n ? e + 1 : n;
    } while (qa.L < sq.L);
    r.l_qual = (int32_t) qa.L;
    r.end = p;
    if (qa.L != sq.L) { r.status = SEQ_BAD; return r; }
    r.status = SEQ_OK;
    r.next = s.hdr(p);
    r.simple = r.lines == 4 && raw[h] == '@' && name_ok && !lone_cr && r.l_qual > 0;
    return r;
}

// the device source (bm2_seq_encode): line ends and header characters by binary search in their position tables, with the index of the
// last line end found as a hint (a walk asks for the next line end almost always)
struct SeqTableSrc {
    const char *raw; int64_t n;
    const int32_t *nl; int n_nl; const int32_t *hp; int n_hp;
    mutable int k;
    BM2_HD int64_t eol(int64_t p) const {
        if (k < n_nl && nl[k] >= p && (k == 0 || nl[k - 1] < p)) return nl[k];
        if (k + 1 < n_nl && nl[k + 1] >= p && nl[k] < p) return nl[++k];
        int lo = 0, hi = n_nl;
        while (lo < hi) { const int m = (lo + hi) >> 1; if (nl[m] < p) lo = m + 1; else hi = m; }
        k = lo;
        return lo < n_nl ? nl[lo] : n;
    }
    BM2_HD int64_t hdr(int64_t p) const {
        int lo = 0, hi = n_hp;
        while (lo < hi) { const int m = (lo + hi) >> 1; if (hp[m] < p) lo = m + 1; else hi = m; }
        return lo < n_hp ? hp[lo] : n;
    }
};

// the host source: memchr over a buffer in memory
struct SeqHostSrc {
    const char *raw; int64_t n;
    int64_t eol(int64_t p) const;
    int64_t hdr(int64_t p) const;
};
#if !defined(__CUDA_ARCH__)
#include <cstring>
inline int64_t SeqHostSrc::eol(int64_t p) const {
    const void *q = p < n ? memchr(raw + p, '\n', (size_t) (n - p)) : nullptr;
    return q ? (int64_t) ((const char *) q - raw) : n;
}
inline int64_t SeqHostSrc::hdr(int64_t p) const {
    for (; p < n; ++p) if (raw[p] == '>' || raw[p] == '@') return p;
    return n;
}
#endif

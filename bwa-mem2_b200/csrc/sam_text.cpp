// sam_text.cpp — SAM text or BAM records of a chunk from the records of seam 4 (host code, a pool of threads over read ranges).
//
// Replaces the formatting half of mem_aln2sam (reference src/bwamem.cpp:1592-1730) as worker_sam calls it through mem_reg2sam / mem_sam_pe:
// the arithmetic half (FLAG, POS, MAPQ, CIGAR, NM, MD, AS, XS, mate columns, XA entries) is done on the GPU by bm2_sam_pe / bm2_sam_se and
// arrives as bm2_sam_rec / bm2_sam_xa; what is left is text - QNAME, the tab-separated columns, SEQ / QUAL trimmed by the record's hard
// clips and reverse-complemented on the reverse strand (:1655-1680), the tag syntax NM MD MC AS XS SA pa XA in the reference's order
// (:1683-1727), and with bm2_sam_format_ex the -R / -C / -V additions (RG, the FASTQ comment, XR: :1693, :1720-1728).
// The reference formats inside worker_sam on all host threads (about 125 k reads/s per thread); this formatter is the same kind of code,
// one pass per record with no allocation per line, so that the host keeps up with the GPU stages in front of it.
//
// Which records and tags a read gets, and in what order, is decided once, by format_read_range; an emitter turns each piece into bytes:
// TextEmit into SAM lines, BamEmit into BAM records (SAMv1 §4.2) with the typed tags `samtools view -b` makes of the same text.
#include "bm2_b200.h"
#include <cctype>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

void bm2_set_error(struct bm2_ctx *ctx, const std::string &msg);

namespace {

struct Out {            // append-only byte buffer: raw pointer writes, doubling growth (one std::string::push_back per character was the
    char *p = nullptr;  // formatter's whole cost in the first version: 0.5 GB/s on 16 threads)
    size_t n = 0, cap = 0;
    ~Out() { free(p); }
    void need(size_t k) {
        if (n + k <= cap) return;
        size_t c = cap ? cap : (size_t) 1 << 16;
        while (c < n + k) c <<= 1;
        p = (char *) realloc(p, c); cap = c;
    }
    void num(long long v) {
        need(24);
        char b[24]; int m = 0;
        unsigned long long u = v < 0 ? (unsigned long long) (-(v + 1)) + 1ULL : (unsigned long long) v;
        do { b[m++] = (char) ('0' + u % 10); u /= 10; } while (u);
        if (v < 0) p[n++] = '-';
        while (m) p[n++] = b[--m];
    }
    void bytes(const void *q, size_t k) { need(k); memcpy(p + n, q, k); n += k; }
    void str(const char *q) { bytes(q, strlen(q)); }
    void ch(char c) { need(1); p[n++] = c; }
    void ops(const uint32_t *o, int k, const char *alphabet) {
        need((size_t) k * 12 + 1);
        for (int i = 0; i < k; ++i) { num((long long) (o[i] >> 4)); p[n++] = alphabet[o[i] & 15]; }
    }
    template <class T> void le(T v) { need(sizeof v); memcpy(p + n, &v, sizeof v); n += sizeof v; }      // x86-64: little-endian as BAM
};

inline bool is_secondary(const bm2_sam_rec &r) { return (r.flag & 0x100) && r.sub < 0; }      // a true secondary (-a), not a -M supplementary

// SEQ / QUAL of one record: the read's bases [qb, qe), reversed and complemented when rev; qual NULL: none
struct SeqSpan { const uint8_t *seq; const char *qual; int64_t qb, qe; bool rev; };

// SAM text, byte for byte mem_aln2sam's
struct TextEmit {
    Out &o;
    bool begin(const char *qn, size_t qlen, const bm2_sam_rec &r, const uint32_t *ops, const SeqSpan *, const char *const *cn) {
        o.bytes(qn, qlen);
        o.ch('\t'); o.num(r.flag); o.ch('\t');
        if (r.rid >= 0) {
            o.str(cn[r.rid]); o.ch('\t'); o.num(r.pos); o.ch('\t'); o.num(r.mapq); o.ch('\t');
            if (r.n_cigar) o.ops(ops, r.n_cigar, "MIDSH"); else o.ch('*');
        } else o.str("*\t0\t0\t*");
        o.ch('\t');
        if (r.rnext >= 0) {
            if (r.rnext == r.rid) o.ch('='); else o.str(cn[r.rnext]);
            o.ch('\t'); o.num(r.pnext); o.ch('\t'); o.num(r.tlen);
        } else o.str("*\t0\t0");
        o.ch('\t');
        return true;
    }
    void seq(const SeqSpan *s) {
        static const char comp[6] = { 'T', 'G', 'C', 'A', 'N', 'N' };
        static const char fwd[6] = { 'A', 'C', 'G', 'T', 'N', 'N' };
        if (!s) { o.str("*\t*"); return; }
        const size_t L = (size_t) (s->qe > s->qb ? s->qe - s->qb : 0);
        o.need(2 * L + 4);
        char *w = o.p + o.n;
        if (!s->rev) {
            for (int64_t i = s->qb; i < s->qe; ++i) *w++ = fwd[s->seq[i] > 5 ? 4 : s->seq[i]];
            *w++ = '\t';
            if (s->qual) { memcpy(w, s->qual + s->qb, L); w += L; } else *w++ = '*';
        } else {
            for (int64_t i = s->qe - 1; i >= s->qb; --i) *w++ = comp[s->seq[i] > 5 ? 4 : s->seq[i]];
            *w++ = '\t';
            if (s->qual) { for (int64_t i = s->qe - 1; i >= s->qb; --i) *w++ = s->qual[i]; } else *w++ = '*';
        }
        o.n = (size_t) (w - o.p);
    }
    void tag_i(const char *t, long long v) { o.ch('\t'); o.bytes(t, 2); o.str(":i:"); o.num(v); }
    void z_begin(const char *t) { o.ch('\t'); o.bytes(t, 2); o.str(":Z:"); }
    void z_end() {}
    void tag_pa(const char *txt) { o.str("\tpa:f:"); o.str(txt); }
    bool comment(const char *c, size_t k, const char *, size_t) { o.ch('\t'); o.bytes(c, k); return true; }
    void end() { o.ch('\n'); }
    std::string err;
};

// BAM records (SAMv1 §4.2)
inline int bam_reg2bin(int64_t beg, int64_t end) {      // SAMv1 §5.3, arithmetic shifts: an unplaced record (-1, 0) gets 4680
    --end;
    if (beg >> 14 == end >> 14) return (int) (((1 << 15) - 1) / 7 + (beg >> 14));
    if (beg >> 17 == end >> 17) return (int) (((1 << 12) - 1) / 7 + (beg >> 17));
    if (beg >> 20 == end >> 20) return (int) (((1 << 9) - 1) / 7 + (beg >> 20));
    if (beg >> 23 == end >> 23) return (int) (((1 << 6) - 1) / 7 + (beg >> 23));
    if (beg >> 26 == end >> 26) return (int) (((1 << 3) - 1) / 7 + (beg >> 26));
    return 0;
}

struct BamEmit {
    Out &o;
    size_t at = 0;                         // this record's block_size field
    const uint32_t *long_ops = nullptr;    // > 65535 operations: the real CIGAR, written as CG:B,I after the tags
    int n_long = 0;
    std::string err;
    static uint32_t op(uint32_t x) { static const uint8_t code[5] = { 0, 1, 2, 4, 5 }; return (x >> 4) << 4 | code[(x & 15) < 5 ? (x & 15) : 0]; }
    bool begin(const char *qn, size_t qlen, const bm2_sam_rec &r, const uint32_t *ops, const SeqSpan *s, const char *const *cn) {
        if (qlen > 254) { err = "read " + std::string(qn, qlen) + ": a QNAME longer than 254 bytes cannot be stored in BAM"; return false; }
        const bool placed = r.rid >= 0;
        const int n_cigar = placed ? r.n_cigar : 0;
        int64_t rlen = 0;
        for (int i = 0; i < n_cigar; ++i) if ((ops[i] & 15) == 0 || (ops[i] & 15) == 2) rlen += ops[i] >> 4;
        const int64_t pos = (placed ? r.pos : 0) - 1;
        const int32_t l_seq = s ? (int32_t) (s->qe > s->qb ? s->qe - s->qb : 0) : 0;
        long_ops = n_cigar > 65535 ? ops : nullptr; n_long = n_cigar;
        at = o.n;
        o.le<int32_t>(0);
        o.le<int32_t>(placed ? r.rid : -1);
        o.le<int32_t>((int32_t) pos);
        o.le<uint8_t>((uint8_t) (qlen + 1));
        o.le<uint8_t>((uint8_t) (placed ? r.mapq : 0));
        o.le<uint16_t>((uint16_t) bam_reg2bin(pos, pos + (rlen ? rlen : 1)));
        o.le<uint16_t>((uint16_t) (long_ops ? 2 : n_cigar));
        o.le<uint16_t>((uint16_t) r.flag);
        o.le<int32_t>(l_seq);
        o.le<int32_t>(r.rnext >= 0 ? r.rnext : -1);
        o.le<int32_t>((int32_t) (r.rnext >= 0 ? r.pnext - 1 : -1));
        o.le<int32_t>((int32_t) (r.rnext >= 0 ? r.tlen : 0));
        o.bytes(qn, qlen); o.ch(0);
        if (long_ops) { o.le<uint32_t>((uint32_t) l_seq << 4 | 4); o.le<uint32_t>((uint32_t) rlen << 4 | 3); }      // kSmN, SAMv1 §4.2.2
        else for (int i = 0; i < n_cigar; ++i) o.le<uint32_t>(op(ops[i]));
        return true;
    }
    void seq(const SeqSpan *s) {
        if (!s) return;
        static const uint8_t fwd[6] = { 1, 2, 4, 8, 15, 15 }, comp[6] = { 8, 4, 2, 1, 15, 15 };
        const int64_t L = s->qe > s->qb ? s->qe - s->qb : 0;
        o.need((size_t) (L + 1) / 2 + (size_t) L);
        uint8_t *w = (uint8_t *) o.p + o.n;
        for (int64_t k = 0; k < L; k += 2) {
            uint8_t b[2] = { 0, 0 };
            for (int h = 0; h < 2 && k + h < L; ++h) {
                const uint8_t c = s->rev ? s->seq[s->qe - 1 - k - h] : s->seq[s->qb + k + h];
                b[h] = (s->rev ? comp : fwd)[c > 5 ? 4 : c];
            }
            *w++ = (uint8_t) (b[0] << 4 | b[1]);
        }
        if (!s->qual) { memset(w, 0xff, (size_t) L); w += L; }
        else if (!s->rev) for (int64_t i = s->qb; i < s->qe; ++i) *w++ = (uint8_t) (s->qual[i] - 33);
        else for (int64_t i = s->qe - 1; i >= s->qb; --i) *w++ = (uint8_t) (s->qual[i] - 33);
        o.n = (size_t) (w - (uint8_t *) o.p);
    }
    void int_val(const char *t, long long v) {     // sam_parse1's rule: the smallest type that holds the value, signed only when negative
        o.bytes(t, 2);
        if (v < 0) {
            if (v >= INT8_MIN) { o.ch('c'); o.le<int8_t>((int8_t) v); }
            else if (v >= INT16_MIN) { o.ch('s'); o.le<int16_t>((int16_t) v); }
            else { o.ch('i'); o.le<int32_t>((int32_t) v); }
        } else if (v <= UINT8_MAX) { o.ch('C'); o.le<uint8_t>((uint8_t) v); }
        else if (v <= UINT16_MAX) { o.ch('S'); o.le<uint16_t>((uint16_t) v); }
        else { o.ch('I'); o.le<uint32_t>((uint32_t) v); }
    }
    void tag_i(const char *t, long long v) { int_val(t, v); }
    void z_begin(const char *t) { o.bytes(t, 2); o.ch('Z'); }
    void z_end() { o.ch(0); }
    void tag_pa(const char *txt) { o.bytes("paf", 3); o.le<float>(strtof(txt, nullptr)); }
    bool comment(const char *c, size_t k, const char *qn, size_t qlen);
    void end() {
        if (long_ops) {
            o.bytes("CGBI", 4); o.le<int32_t>(n_long);
            for (int i = 0; i < n_long; ++i) o.le<uint32_t>(op(long_ops[i]));
        }
        const int32_t bs = (int32_t) (o.n - at - 4);
        memcpy(o.p + at, &bs, 4);
    }
};

// -C in BAM: the comment is tab-separated SAM tags TG:T:VALUE, parsed as sam_parse1 parses the optional fields of a SAM line
bool BamEmit::comment(const char *c, size_t k, const char *qn, size_t qlen) {
    const char *p = c, *e = c + k;
    auto fail = [&](const char *why) { err = "read " + std::string(qn, qlen) + ": its comment is not SAM tags (" + why + "): " + std::string(c, k); return false; };
    while (p < e) {
        const char *f = (const char *) memchr(p, '\t', (size_t) (e - p));
        if (!f) f = e;
        const size_t n = (size_t) (f - p);
        if (n < 5 || p[2] != ':' || p[4] != ':' || !isalpha((unsigned char) p[0]) || !isalnum((unsigned char) p[1])) return fail("TG:T:VALUE expected");
        const char type = p[3];
        const std::string v(p + 5, n - 5);
        char *q = nullptr;
        if (type == 'A') {
            if (v.size() != 1) return fail("A takes one character");
            o.bytes(p, 2); o.ch('A'); o.ch(v[0]);
        } else if (strchr("cCsSiI", type)) {
            errno = 0;
            const long long x = strtoll(v.c_str(), &q, 10);
            if (v.empty() || *q || errno || x < INT32_MIN || x > (long long) UINT32_MAX) return fail("bad integer");
            int_val(p, x);
        } else if (type == 'f') {
            const float x = strtof(v.c_str(), &q);
            if (v.empty() || *q) return fail("bad float");
            o.bytes(p, 2); o.ch('f'); o.le<float>(x);
        } else if (type == 'Z' || type == 'H') {
            if (type == 'H' && (v.size() % 2 || v.find_first_not_of("0123456789ABCDEFabcdef") != std::string::npos)) return fail("bad hex");
            o.bytes(p, 2); o.ch(type); o.bytes(v.data(), v.size()); o.ch(0);
        } else if (type == 'B') {
            if (v.empty() || !strchr("cCsSiIf", v[0]) || (v.size() > 1 && v[1] != ',')) return fail("bad array");
            const char sub = v[0];
            std::vector<std::string> items;
            for (size_t a = 2; v.size() > 1 && a <= v.size();) {
                size_t b = v.find(',', a); if (b == std::string::npos) b = v.size();
                items.push_back(v.substr(a, b - a)); a = b + 1;
            }
            o.bytes(p, 2); o.ch('B'); o.ch(sub); o.le<int32_t>((int32_t) items.size());
            for (const std::string &it : items) {
                if (sub == 'f') { const float x = strtof(it.c_str(), &q); if (it.empty() || *q) return fail("bad array"); o.le<float>(x); continue; }
                errno = 0;
                const long long x = strtoll(it.c_str(), &q, 10);
                if (it.empty() || *q || errno) return fail("bad array");
                if (sub == 'c') o.le<int8_t>((int8_t) x); else if (sub == 'C') o.le<uint8_t>((uint8_t) x);
                else if (sub == 's') o.le<int16_t>((int16_t) x); else if (sub == 'S') o.le<uint16_t>((uint16_t) x);
                else if (sub == 'i') o.le<int32_t>((int32_t) x); else o.le<uint32_t>((uint32_t) x);
            }
        } else return fail("unknown type");
        p = f + 1;
    }
    return true;
}

struct Job {
    const bm2_sam_text_in *in;
    const bm2_sam_text_extra *x;           // may be NULL
    const int64_t *first_rec_of_read;      // n_reads + 1
    const int64_t *first_xa_of_read;       // n_reads + 1
    int64_t r0, r1;                        // read range
    Out out;
    std::vector<int64_t> read_at;          // BAM: where each read's records start in out
    std::string err;
};

// the records of reads [r0, r1): which fields, tags and additions each gets, in mem_aln2sam's order
template <class E> void format_read_range(Job &j) {
    const bm2_sam_text_in &in = *j.in;
    const bm2_sam_result &res = *in.res;
    const bm2_read_batch &rb = *in.reads;
    const char *const *cn = in.contig_names;
    E e{j.out};
    j.out.need((size_t) (j.r1 - j.r0) * 440 + 1024);
    j.read_at.reserve((size_t) (j.r1 - j.r0));
    char rname[24];
    for (int64_t rd = j.r0; rd < j.r1; ++rd) {
        j.read_at.push_back((int64_t) j.out.n);
        const int64_t k0 = j.first_rec_of_read[rd], k1 = j.first_rec_of_read[rd + 1];
        const int64_t so = rb.offsets[rd], l_seq = rb.offsets[rd + 1] - so;
        const uint8_t *seq = rb.codes + so;
        const char *qual = in.quals && !(j.x && j.x->qual_present && !j.x->qual_present[rd]) ? in.quals + so : nullptr;
        // QNAME
        const char *qn; size_t qlen;
        if (in.names) { qn = in.names[rd]; qlen = strlen(qn); }
        else if (in.name_beg && in.name_len && in.name_buf[0]) {      // QNAME as a span of the caller's FASTQ buffer (bm2_fastq_batch)
            const char *nb = (in.name_buf[1] && (rd & 1)) ? in.name_buf[1] : in.name_buf[0];
            qn = nb + in.name_beg[rd]; qlen = (size_t) in.name_len[rd];
        } else { qlen = (size_t) snprintf(rname, sizeof rname, "r%lld", (long long) rd); qn = rname; }
        for (int64_t k = k0; k < k1; ++k) {
            const bm2_sam_rec &r = res.recs[k];
            const uint32_t *ops = res.cigar + r.cigar_off;
            // SEQ QUAL (src/bwamem.cpp:1650-1682): none for a true secondary, else trimmed by the hard clips
            const bool sec = is_secondary(r);
            SeqSpan ss = { seq, qual, 0, l_seq, (r.flag & 0x10) != 0 };
            if (r.n_cigar && (ops[0] & 15) == 4) { if (ss.rev) ss.qe -= ops[0] >> 4; else ss.qb += ops[0] >> 4; }
            if (r.n_cigar && (ops[r.n_cigar - 1] & 15) == 4) { if (ss.rev) ss.qb += ops[r.n_cigar - 1] >> 4; else ss.qe -= ops[r.n_cigar - 1] >> 4; }
            // QNAME FLAG RNAME POS MAPQ CIGAR RNEXT PNEXT TLEN
            if (!e.begin(qn, qlen, r, ops, sec ? nullptr : &ss, cn)) { j.err = e.err; return; }
            e.seq(sec ? nullptr : &ss);
            // tags: NM MD MC AS XS RG SA pa XA
            if (r.n_cigar) {
                e.tag_i("NM", r.nm);
                e.z_begin("MD"); j.out.bytes(res.md + r.md_off, (size_t) (r.n_md > 0 ? r.n_md - 1 : 0)); e.z_end();
            }
            if (r.n_mc > 0) { e.z_begin("MC"); j.out.ops(ops + r.n_cigar, r.n_mc, "MIDSH"); e.z_end(); }
            if (r.score >= 0) e.tag_i("AS", r.score);
            if (r.sub >= 0) e.tag_i("XS", r.sub);
            if (j.x && j.x->rg_id && j.x->rg_id[0]) { e.z_begin("RG"); j.out.str(j.x->rg_id); e.z_end(); }
            if (!sec) {
                Out &o = j.out;
                bool any = false;
                for (int64_t q = k0; q < k1; ++q) {
                    if (q == k || is_secondary(res.recs[q])) continue;
                    const bm2_sam_rec &t = res.recs[q];
                    if (!any) { e.z_begin("SA"); any = true; }
                    o.str(cn[t.rid]); o.ch(','); o.num(t.pos); o.ch(','); o.ch((t.flag & 0x10) ? '-' : '+'); o.ch(',');
                    o.ops(res.cigar + t.cigar_off, t.n_cigar, "MIDSS");
                    o.ch(','); o.num(t.mapq); o.ch(','); o.num(t.nm); o.ch(';');
                }
                if (any) e.z_end();
                if (r.alt_sc > 0) { char b[48]; snprintf(b, sizeof b, "%.3f", (double) r.score / r.alt_sc); e.tag_pa(b); }
            }
            if (r.reg >= 0) {
                Out &o = j.out;
                bool any = false;
                for (int64_t x = j.first_xa_of_read[rd]; x < j.first_xa_of_read[rd + 1]; ++x) {
                    const bm2_sam_xa &xe = res.xa[x];
                    if (xe.reg != r.reg) continue;
                    if (!any) { e.z_begin("XA"); any = true; }
                    o.str(cn[xe.rid]); o.ch(','); o.ch(xe.is_rev ? '-' : '+'); o.num(xe.pos + 1); o.ch(',');
                    o.ops(res.cigar + xe.cigar_off, xe.n_cigar, "MIDSHN");
                    o.ch(','); o.num(xe.nm); o.ch(';');
                }
                if (any) e.z_end();
            }
            if (j.x && j.x->comment_beg && j.x->comment_len && j.x->comment_len[rd] > 0 && in.name_buf[0]) {
                const char *cb = (in.name_buf[1] && (rd & 1)) ? in.name_buf[1] : in.name_buf[0];
                if (!e.comment(cb + j.x->comment_beg[rd], (size_t) j.x->comment_len[rd], qn, qlen)) { j.err = e.err; return; }
            }
            if (j.x && j.x->ref_hdr && j.x->contig_anno && r.rid >= 0 && j.x->contig_anno[r.rid] && j.x->contig_anno[r.rid][0]) {
                e.z_begin("XR");
                const size_t at = j.out.n;
                j.out.str(j.x->contig_anno[r.rid]);
                for (size_t i = at; i < j.out.n; ++i) if (j.out.p[i] == '\t') j.out.p[i] = ' ';
                e.z_end();
            }
            e.end();
        }
    }
}

// the records of a batch on n_threads threads, one read range each, the pieces joined in read order; read_off: NULL, or n_reads + 1 offsets
template <class E> int format_batch(const char *what, const bm2_sam_text_in *in, const bm2_sam_text_extra *x, int n_threads, char **text,
                                    int64_t *len, int64_t **read_off) {
    if (!in || !in->res || !in->reads || !in->contig_names || !text || !len) return 1;
    const bm2_sam_result &res = *in->res;
    const int64_t n_reads = in->reads->n_reads;
    // records and XA entries are grouped by read, reads ascending (bm2_sam_pe / bm2_sam_se emit pair by pair): index them per read
    std::vector<int64_t> first_rec((size_t) n_reads + 1, 0), first_xa((size_t) n_reads + 1, 0);
    {
        int64_t prev = -1;
        for (int64_t k = 0; k < res.n_recs; ++k) {
            const int64_t rd = res.recs[k].read;
            if (rd < prev || rd >= n_reads) return 2;                   // not grouped / out of range
            ++first_rec[(size_t) rd + 1]; prev = rd;
        }
        prev = -1;
        for (int64_t k = 0; k < res.n_xa; ++k) {
            const int64_t rd = res.xa[k].read;
            if (rd < prev || rd >= n_reads) return 2;
            ++first_xa[(size_t) rd + 1]; prev = rd;
        }
        for (int64_t r = 0; r < n_reads; ++r) { first_rec[(size_t) r + 1] += first_rec[(size_t) r]; first_xa[(size_t) r + 1] += first_xa[(size_t) r]; }
    }
    if (n_threads < 1) n_threads = 1;
    if ((int64_t) n_threads > n_reads) n_threads = n_reads > 0 ? (int) n_reads : 1;
    std::vector<Job> jobs((size_t) n_threads);
    for (int t = 0; t < n_threads; ++t) {
        jobs[t].in = in; jobs[t].x = x; jobs[t].first_rec_of_read = first_rec.data(); jobs[t].first_xa_of_read = first_xa.data();
        jobs[t].r0 = n_reads * t / n_threads; jobs[t].r1 = n_reads * (t + 1) / n_threads;
    }
    {
        std::vector<std::thread> th;
        for (int t = 1; t < n_threads; ++t) th.emplace_back(format_read_range<E>, std::ref(jobs[t]));
        format_read_range<E>(jobs[0]);
        for (auto &t : th) t.join();
    }
    for (auto &j : jobs) if (!j.err.empty()) { bm2_set_error(nullptr, std::string(what) + ": " + j.err); return 4; }
    size_t total = 0;
    for (auto &j : jobs) total += j.out.n;
    char *buf = (char *) malloc(total + 1);
    int64_t *ro = read_off ? (int64_t *) malloc(((size_t) n_reads + 1) * sizeof(int64_t)) : nullptr;
    if (!buf || (read_off && !ro)) { free(buf); free(ro); return 3; }
    {   // the pieces into one buffer, one thread per piece
        std::vector<size_t> at((size_t) n_threads, 0);
        for (int t = 1; t < n_threads; ++t) at[t] = at[t - 1] + jobs[t - 1].out.n;
        std::vector<std::thread> th;
        auto cp = [&](int t) {
            if (jobs[t].out.n) memcpy(buf + at[t], jobs[t].out.p, jobs[t].out.n);
            if (ro) for (int64_t r = jobs[t].r0; r < jobs[t].r1; ++r) ro[r] = (int64_t) at[t] + jobs[t].read_at[(size_t) (r - jobs[t].r0)];
        };
        for (int t = 1; t < n_threads; ++t) th.emplace_back(cp, t);
        cp(0);
        for (auto &t : th) t.join();
    }
    buf[total] = 0;
    if (ro) { ro[n_reads] = (int64_t) total; *read_off = ro; }
    *text = buf; *len = (int64_t) total;
    return 0;
}

}  // namespace

extern "C" int bm2_sam_format_ex(const bm2_sam_text_in *in, const bm2_sam_text_extra *x, int n_threads, char **text, int64_t *len) {
    return format_batch<TextEmit>("bm2_sam_format", in, x, n_threads, text, len, nullptr);
}

extern "C" int bm2_sam_format(const bm2_sam_text_in *in, int n_threads, char **text, int64_t *len) { return bm2_sam_format_ex(in, nullptr, n_threads, text, len); }

extern "C" int bm2_bam_format_ex(const bm2_sam_text_in *in, const bm2_sam_text_extra *x, int n_threads, char **bam, int64_t *len, int64_t **read_off) {
    if (!read_off) return 1;
    return format_batch<BamEmit>("bm2_bam_format", in, x, n_threads, bam, len, read_off);
}

extern "C" void bm2_free(void *p) { free(p); }

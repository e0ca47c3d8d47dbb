// sam_text.cpp — SAM text of a chunk from the records of seam 4 (host code, a pool of threads over read ranges).
//
// Replaces the formatting half of mem_aln2sam (reference src/bwamem.cpp:1592-1730) as worker_sam calls it through mem_reg2sam / mem_sam_pe:
// the arithmetic half (FLAG, POS, MAPQ, CIGAR, NM, MD, AS, XS, mate columns, XA entries) is done on the GPU by bm2_sam_pe / bm2_sam_se and
// arrives as bm2_sam_rec / bm2_sam_xa; what is left is text - QNAME, the tab-separated columns, SEQ / QUAL trimmed by the record's hard
// clips and reverse-complemented on the reverse strand (:1655-1680), the tag syntax NM MD MC AS XS SA pa XA in the reference's order
// (:1683-1727), and with bm2_sam_format_ex the -R / -C / -V additions (RG, the FASTQ comment, XR: :1693, :1720-1728).
// The reference formats inside worker_sam on all host threads (about 125 k reads/s per thread); this formatter is the same kind of code,
// one pass per record with no allocation per line, so that the host keeps up with the GPU stages in front of it.
#include "bm2_b200.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

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
    void bytes(const char *q, size_t k) { need(k); memcpy(p + n, q, k); n += k; }
    void str(const char *q) { bytes(q, strlen(q)); }
    void ch(char c) { need(1); p[n++] = c; }
    void ops(const uint32_t *o, int k, const char *alphabet) {
        need((size_t) k * 12 + 1);
        for (int i = 0; i < k; ++i) { num((long long) (o[i] >> 4)); p[n++] = alphabet[o[i] & 15]; }
    }
};

inline bool is_secondary(const bm2_sam_rec &r) { return (r.flag & 0x100) && r.sub < 0; }      // a true secondary (-a), not a -M supplementary

struct Job {
    const bm2_sam_text_in *in;
    const bm2_sam_text_extra *x;           // may be NULL
    const int64_t *first_rec_of_read;      // n_reads + 1
    const int64_t *first_xa_of_read;       // n_reads + 1
    int64_t r0, r1;                        // read range
    Out out;
};

void format_read_range(Job &j) {
    const bm2_sam_text_in &in = *j.in;
    const bm2_sam_result &res = *in.res;
    const bm2_read_batch &rb = *in.reads;
    static const char comp[6] = { 'T', 'G', 'C', 'A', 'N', 'N' };
    static const char fwd[6] = { 'A', 'C', 'G', 'T', 'N', 'N' };
    j.out.need((size_t) (j.r1 - j.r0) * 440 + 1024);
    for (int64_t rd = j.r0; rd < j.r1; ++rd) {
        const int64_t k0 = j.first_rec_of_read[rd], k1 = j.first_rec_of_read[rd + 1];
        const int64_t so = rb.offsets[rd], l_seq = rb.offsets[rd + 1] - so;
        const uint8_t *seq = rb.codes + so;
        const char *qual = in.quals && !(j.x && j.x->qual_present && !j.x->qual_present[rd]) ? in.quals + so : nullptr;
        for (int64_t k = k0; k < k1; ++k) {
            const bm2_sam_rec &r = res.recs[k];
            Out &o = j.out;
            const uint32_t *ops = res.cigar + r.cigar_off;
            // QNAME FLAG RNAME POS MAPQ CIGAR
            if (in.names) o.str(in.names[rd]);
            else if (in.name_beg && in.name_len && in.name_buf[0]) {      // QNAME as a span of the caller's FASTQ buffer (bm2_fastq_batch)
                const char *nb = (in.name_buf[1] && (rd & 1)) ? in.name_buf[1] : in.name_buf[0];
                o.bytes(nb + in.name_beg[rd], (size_t) in.name_len[rd]);
            } else { o.ch('r'); o.num(rd); }
            o.ch('\t'); o.num(r.flag); o.ch('\t');
            if (r.rid >= 0) {
                o.str(in.contig_names[r.rid]); o.ch('\t'); o.num(r.pos); o.ch('\t'); o.num(r.mapq); o.ch('\t');
                if (r.n_cigar) o.ops(ops, r.n_cigar, "MIDSH"); else o.ch('*');
            } else o.str("*\t0\t0\t*");
            o.ch('\t');
            // RNEXT PNEXT TLEN
            if (r.rnext >= 0) {
                if (r.rnext == r.rid) o.ch('='); else o.str(in.contig_names[r.rnext]);
                o.ch('\t'); o.num(r.pnext); o.ch('\t'); o.num(r.tlen);
            } else o.str("*\t0\t0");
            o.ch('\t');
            // SEQ QUAL (src/bwamem.cpp:1650-1682)
            const bool sec = is_secondary(r);
            if (sec) o.str("*\t*");
            else {
                int64_t qb = 0, qe = l_seq;
                const bool rev = (r.flag & 0x10) != 0;
                if (r.n_cigar && (ops[0] & 15) == 4) { if (rev) qe -= ops[0] >> 4; else qb += ops[0] >> 4; }
                if (r.n_cigar && (ops[r.n_cigar - 1] & 15) == 4) { if (rev) qb += ops[r.n_cigar - 1] >> 4; else qe -= ops[r.n_cigar - 1] >> 4; }
                const size_t L = (size_t) (qe > qb ? qe - qb : 0);
                o.need(2 * L + 4);
                char *w = o.p + o.n;
                if (!rev) {
                    for (int64_t i = qb; i < qe; ++i) *w++ = fwd[seq[i] > 5 ? 4 : seq[i]];
                    *w++ = '\t';
                    if (qual) { memcpy(w, qual + qb, L); w += L; } else *w++ = '*';
                } else {
                    for (int64_t i = qe - 1; i >= qb; --i) *w++ = comp[seq[i] > 5 ? 4 : seq[i]];
                    *w++ = '\t';
                    if (qual) { for (int64_t i = qe - 1; i >= qb; --i) *w++ = qual[i]; } else *w++ = '*';
                }
                o.n = (size_t) (w - o.p);
            }
            // tags: NM MD MC AS XS SA pa XA
            if (r.n_cigar) {
                o.str("\tNM:i:"); o.num(r.nm);
                o.str("\tMD:Z:"); o.bytes(res.md + r.md_off, (size_t) (r.n_md > 0 ? r.n_md - 1 : 0));
            }
            if (r.n_mc > 0) { o.str("\tMC:Z:"); o.ops(ops + r.n_cigar, r.n_mc, "MIDSH"); }
            if (r.score >= 0) { o.str("\tAS:i:"); o.num(r.score); }
            if (r.sub >= 0) { o.str("\tXS:i:"); o.num(r.sub); }
            if (j.x && j.x->rg_id && j.x->rg_id[0]) { o.str("\tRG:Z:"); o.str(j.x->rg_id); }
            if (!sec) {
                bool any = false;
                for (int64_t q = k0; q < k1; ++q) {
                    if (q == k || is_secondary(res.recs[q])) continue;
                    const bm2_sam_rec &t = res.recs[q];
                    if (!any) { o.str("\tSA:Z:"); any = true; }
                    o.str(in.contig_names[t.rid]); o.ch(','); o.num(t.pos); o.ch(','); o.ch((t.flag & 0x10) ? '-' : '+'); o.ch(',');
                    o.ops(res.cigar + t.cigar_off, t.n_cigar, "MIDSS");
                    o.ch(','); o.num(t.mapq); o.ch(','); o.num(t.nm); o.ch(';');
                }
                if (r.alt_sc > 0) { char b[48]; snprintf(b, sizeof b, "\tpa:f:%.3f", (double) r.score / r.alt_sc); o.str(b); }
            }
            if (r.reg >= 0) {
                bool any = false;
                for (int64_t x = j.first_xa_of_read[rd]; x < j.first_xa_of_read[rd + 1]; ++x) {
                    const bm2_sam_xa &e = res.xa[x];
                    if (e.reg != r.reg) continue;
                    if (!any) { o.str("\tXA:Z:"); any = true; }
                    o.str(in.contig_names[e.rid]); o.ch(','); o.ch(e.is_rev ? '-' : '+'); o.num(e.pos + 1); o.ch(',');
                    o.ops(res.cigar + e.cigar_off, e.n_cigar, "MIDSHN");
                    o.ch(','); o.num(e.nm); o.ch(';');
                }
            }
            if (j.x && j.x->comment_beg && j.x->comment_len && j.x->comment_len[rd] > 0 && in.name_buf[0]) {
                const char *cb = (in.name_buf[1] && (rd & 1)) ? in.name_buf[1] : in.name_buf[0];
                o.ch('\t'); o.bytes(cb + j.x->comment_beg[rd], (size_t) j.x->comment_len[rd]);
            }
            if (j.x && j.x->ref_hdr && j.x->contig_anno && r.rid >= 0 && j.x->contig_anno[r.rid] && j.x->contig_anno[r.rid][0]) {
                o.str("\tXR:Z:");
                const size_t at = o.n;
                o.str(j.x->contig_anno[r.rid]);
                for (size_t i = at; i < o.n; ++i) if (o.p[i] == '\t') o.p[i] = ' ';
            }
            o.ch('\n');
        }
    }
}

}  // namespace

extern "C" int bm2_sam_format_ex(const bm2_sam_text_in *in, const bm2_sam_text_extra *x, int n_threads, char **text, int64_t *len) {
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
        for (int t = 1; t < n_threads; ++t) th.emplace_back(format_read_range, std::ref(jobs[t]));
        format_read_range(jobs[0]);
        for (auto &x : th) x.join();
    }
    size_t total = 0;
    for (auto &j : jobs) total += j.out.n;
    char *buf = (char *) malloc(total + 1);
    if (!buf) return 3;
    {   // the pieces into one buffer, one thread per piece
        std::vector<size_t> at((size_t) n_threads, 0);
        for (int t = 1; t < n_threads; ++t) at[t] = at[t - 1] + jobs[t - 1].out.n;
        std::vector<std::thread> th;
        auto cp = [&](int t) { if (jobs[t].out.n) memcpy(buf + at[t], jobs[t].out.p, jobs[t].out.n); };
        for (int t = 1; t < n_threads; ++t) th.emplace_back(cp, t);
        cp(0);
        for (auto &x : th) x.join();
    }
    buf[total] = 0;
    *text = buf; *len = (int64_t) total;
    return 0;
}

extern "C" int bm2_sam_format(const bm2_sam_text_in *in, int n_threads, char **text, int64_t *len) { return bm2_sam_format_ex(in, nullptr, n_threads, text, len); }

extern "C" void bm2_free(void *p) { free(p); }

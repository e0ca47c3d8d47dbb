// bm2_mem — FASTQ in, SAM or BAM out, on the GPU path: the host side of `bwa-mem2 mem` for the seams of libbm2b200.so (C++, as the reference's host
// code; only the C ABI of include/bm2_b200.h is used).
//
//   bm2_mem [options] <index prefix> <reads_1.fq> [reads_2.fq]
//
// The options are those of `bwa-mem2 mem` (main_mem, src/fastmap.cpp:616-943: the same getopt string, presets, update_a, -I, -R, -H, -j), with
// the same SAM output, plus two of this program's own: `-p N` (N a positive decimal integer, as a separate argument) is the number of chunks in
// flight (see below), and `--dump-opt` prints the parsed options and the header as JSON and exits before any device call.  Any other -p, alone
// or in a cluster such as -5SP, is the reference's smart pairing.  usage() lists them.
//
// What the reference does in main_mem / process / ktp_worker (src/fastmap.cpp:616-1003, :280-349), with every step of a chunk behind a seam:
//   chunk of the input            bseq_read_orig's rule (src/bwa.cpp:170-216): records until the base count reaches the task size
//                                 (-K, else chunk_size x threads, src/fastmap.cpp:943-949) at an even record count, mates kept together
//   bm2_fastq_encode              parsing + nst_nt4_table encoding on the GPU                         (kseq + src/bwamem.cpp:992-1000)
//     or bm2_seq_encode           the same for any input kseq reads (FASTA, wrapped FASTQ, ...): a chunk goes through bm2_fastq_encode
//                                 when all its records are "simple" four-line FASTQ records that end where the next begins (seq_grammar.cuh)
//   bm2_fastq_smart_pair          -p: bseq_classify on the GPU, then the two calls of mem_process_seqs (src/fastmap.cpp:249-287)
//   bm2_seed_chain_extend_resident  worker_bwt + worker_aln                                           (src/bwamem.cpp:1359-1363)
//   bm2_pestat                    mem_pestat, or the -I values                                        (src/bwamem.cpp:1368-1378)
//   bm2_sam_pe / bm2_sam_se       worker_sam's arithmetic                                             (src/bwamem.cpp:1262-1336)
//   bm2_sam_format_ex             mem_aln2sam's text with RG / the -C comment / XR                    (src/bwamem.cpp:1592-1730)
//     or bm2_bam_format_ex        --bam: the same records as BAM, then bm2_bgzf_compress: BGZF members compressed on the GPU
//        then bm2_bam_sort_compress_ex  --sort: the records in sorted runs, merged, compressed on the GPU, and the BAI (bam_sort.h)
//        with bm2_dup_signatures     --markdup: each chunk's templates' entries, resolved by bm2_dup_resolve at the end; the duplicates' records get
//                                    0x400 in the same sort, which then carries each record's template id (bam_sort.h, markdup_device.cuh)
//        or bm2_dup_signatures_ex    --markdup-metrics: the same with located pair entries and the chunk's record counts, resolved by
//                                    bm2_dup_resolve_ex with the optical pass; Picard's metrics file at the end (markdup_metrics.h)
//        and bm2_bqsr_sites             --recal-file: the --known-sites VCFs, read on a thread of their own while the reads align (known_sites.h),
//                                    go to the sort context before the final sort pass, which then counts the covariates of the sorted
//                                    records on the GPU (bqsr_device.cuh); GATK's recalibration report at the end (bqsr_report.h)
// Chunks in flight: the reference's kt_pipeline runs its three steps (read, process, write) on two worker threads so that one chunk's I/O
// overlaps another's computation (src/fastmap.cpp:952-1003, src/kthread.cpp:122-176).  Here -p workers (default 2) each own a context
// (bm2_create_sibling: one index in HBM) and take whole chunks off a queue; the GPU interleaves the kernels of the two chunks, the host side of
// one (pestat, formatting, fwrite) runs under the GPU stages of the other, and the output is written strictly in chunk order.
// The SAM file equals `bwa-mem2 mem` with the same options and -K except for the @PG line, which names this program
// (tests/test_zz_fastq_sam_gpu.py, tests/test_zz_mem_cli_gpu.py, tests/test_zz_seq_input_gpu.py).  Input: whatever kseq reads - FASTA or
// FASTQ, wrapped or not, plain or gzip - from files or, for `-`, standard input.  The inputs stream (read_input.h): the chunker cuts chunks
// from a window of each input refilled by read() while the workers align earlier chunks, and each chunk owns a copy of its bytes, so host
// memory for input is about (queue + workers) x chunk bytes plus the windows, whatever the input's size.  Gzip (any number of members,
// BGZF included) is inflated by zlib on the chunker's thread, overlapped with the alignment of earlier chunks.
#include "bm2_b200.h"
#include "../csrc/seq_grammar.cuh"
#include "../csrc/read_input.h"
#include "../csrc/bam_sort.h"
#include "../csrc/sort_header.h"
#include "../csrc/markdup_metrics.h"
#include "../csrc/bqsr_report.h"
#include "../csrc/known_sites.h"
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <thread>
#include <cmath>
#include <cctype>
#include <cerrno>
#include <cstdio>
#include <unistd.h>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <zlib.h>
#include <getopt.h>

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

namespace {

struct Shared {
    // work queue (the chunker fills it, bounded), write order, totals
    std::mutex mu; std::condition_variable cv_work, cv_room, cv_turn;
    std::deque<Chunk> queue; bool done = false;
    long long next_to_write = 0;
    double t_loop = 0;
    double t_bam = 0, t_bgzf = 0; long long bam_bytes = 0, bgzf_bytes = 0;       // --bam: encoding (host), compression (device), sizes
    double t_enc = 0, t_aln = 0, t_pes = 0, t_sam = 0, t_fmt = 0, t_write = 0, t_turn = 0;
    std::vector<double> chunk_s, chunk_done_s; std::vector<long long> chunk_reads;
    long long n_processed = 0;
    // constants
    const bm2_mem_opt_t *opt = nullptr; const bm2_index_desc *idx = nullptr; const char *const *cnames = nullptr;
    bool paired = false, smart = false; int threads = 1; FILE *out = nullptr;
    const bm2_pestat_t *pes0 = nullptr;                          // -I: used instead of bm2_pestat
    bm2_sam_text_extra extra{};                                  // -R / -C / -V
    bool copy_comment = false, bam = false;
    BamSortSink *sink = nullptr;                                 // --sort: the records go to the sorted runs instead of the output
    bool markdup = false; double t_dup_sig = 0;                  // --markdup: device time of the signature kernels
    bool metrics = false; long long n_sec_supp = 0, n_unmapped = 0;   // --markdup-metrics: the records' counts of the signature kernels
    double t_split = 0;
    long long seq_chunks = 0;                                    // chunks that went through bm2_seq_encode
    size_t in_flight = 0;                                        // bytes of the chunks queued or being aligned
};

[[noreturn]] void die(const char *what, const bm2_ctx *ctx) { fprintf(stderr, "bm2_mem: %s%s%s\n", what, ctx ? ": " : "", ctx ? bm2_last_error(ctx) : ""); fflush(stderr); _Exit(3); }

struct Times { double aln = 0, pes = 0, sam = 0, fmt = 0, bam = 0; };

// one batch through seams 2, 4 and 5: its SAM text or, with --bam, its BAM records (malloc'd) and, when read_end != nullptr, where the output
// of every read ends; qual_present: NULL, or 0 for the reads without qualities (QUAL '*')
char *align_and_format(Shared *sh, bm2_ctx *ctx, const bm2_fastq_batch &fq, const char *buf0, const char *buf1, const int64_t *cmt_beg,
                       const int32_t *cmt_len, const uint8_t *qual_present, bool paired, long long id_base, int64_t *len, std::vector<int64_t> *read_end, Times &t) {
    const double t1 = now_s();
    bm2_read_batch rb = { fq.n_reads, fq.codes, fq.offsets };
    bm2_reg_result rr;
    if (bm2_seed_chain_extend_resident(ctx, &rb, fq.d_codes, fq.d_offsets, 1, &rr)) die("bm2_seed_chain_extend_resident", ctx);
    const double t2 = now_s();
    double t3 = t2;
    bm2_sam_result sr;
    if (paired) {
        bm2_pestat_t pes[4];
        if (sh->pes0) memcpy(pes, sh->pes0, sizeof pes);
        else if (bm2_pestat(sh->opt, sh->idx->l_pac, fq.n_reads, rr.regs, rr.read_off, pes)) die("bm2_pestat failed", nullptr);
        t3 = now_s();
        if (bm2_sam_pe(ctx, &rb, rr.regs, rr.read_off, pes, id_base, &sr)) die("bm2_sam_pe", ctx);
    } else if (bm2_sam_se(ctx, &rb, rr.regs, rr.read_off, id_base, &sr)) die("bm2_sam_se", ctx);
    const double t4 = now_s();
    bm2_sam_text_in tin; memset(&tin, 0, sizeof tin);
    tin.res = &sr; tin.reads = &rb; tin.quals = fq.quals; tin.contig_names = sh->cnames;
    tin.name_buf[0] = buf0; tin.name_buf[1] = buf1; tin.name_beg = fq.name_beg; tin.name_len = fq.name_len;
    bm2_sam_text_extra x = sh->extra;
    x.comment_beg = cmt_beg; x.comment_len = cmt_len; x.qual_present = qual_present;
    char *text = nullptr;
    if (sh->bam) {
        int64_t *ro = nullptr;
        if (bm2_bam_format_ex(&tin, &x, sh->threads, &text, len, &ro)) { fprintf(stderr, "[E::bm2_mem] %s\n", bm2_last_error(nullptr)); fflush(stderr); _Exit(1); }
        if (read_end) read_end->assign(ro + 1, ro + fq.n_reads + 1);
        bm2_free(ro);
        t.bam += now_s() - t4;
    } else {
        if (bm2_sam_format_ex(&tin, &x, sh->threads, &text, len)) die("bm2_sam_format_ex failed", nullptr);
        if (read_end) {                                                  // lines per read, then where they end
            read_end->assign((size_t) fq.n_reads, 0);
            for (int64_t k = 0; k < sr.n_recs; ++k) ++(*read_end)[(size_t) sr.recs[k].read];
            const char *q = text;
            for (int64_t &e : *read_end) { for (int64_t k = e; k > 0; --k) q = (const char *) memchr(q, '\n', (size_t) (text + *len - q)) + 1; e = q - text; }
        }
        t.fmt += now_s() - t4;
    }
    t.aln += t2 - t1; t.pes += t3 - t2; t.sam += t4 - t3;
    return text;
}

// -p: the single-end set and the pairs of a chunk as the reference's two mem_process_seqs calls (src/fastmap.cpp:260-285), the reads' lines
// (or BAM records) merged back into file order (the records of a read are consecutive); with read_end, where each read's output ends in
// the merged text and each read's mate (-1: none)
char *smart_pair_chunk(Shared *sh, bm2_ctx *ctx, const Chunk &ck, int n_reads, const uint8_t *qual_present, int64_t *len, Times &t,
                       std::vector<int64_t> *read_end = nullptr, std::vector<int64_t> *mate = nullptr) {
    const double t0 = now_s();
    bm2_fastq_split sp;
    if (bm2_fastq_smart_pair(ctx, &sp)) die("bm2_fastq_smart_pair", ctx);
    const double t_split = now_s() - t0;
    char *text[2] = { nullptr, nullptr }; int64_t tl[2] = { 0, 0 }; std::vector<int64_t> ends[2];
    const long long base[2] = { ck.first_read, (ck.first_read + sp.set[0].n_reads) >> 1 };
    std::vector<uint8_t> qp[2];
    for (int s = 0; s < 2 && qual_present; ++s)
        for (int j = 0; j < sp.set[s].n_reads; ++j) qp[s].push_back(qual_present[sp.read_index[s][j]]);
    for (int s = 0; s < 2; ++s)
        if (sp.set[s].n_reads)
            text[s] = align_and_format(sh, ctx, sp.set[s], ck.c1, nullptr, sh->copy_comment ? sp.comment_beg[s] : nullptr,
                                       sh->copy_comment ? sp.comment_len[s] : nullptr, qual_present ? qp[s].data() : nullptr, s == 1, base[s],
                                       &tl[s], &ends[s], t);
    std::vector<int8_t> set_of((size_t) n_reads, -1);
    for (int s = 0; s < 2; ++s) for (int j = 0; j < sp.set[s].n_reads; ++j) set_of[(size_t) sp.read_index[s][j]] = (int8_t) s;
    char *merged = (char *) malloc((size_t) (tl[0] + tl[1]) + 1);
    if (!merged) die("out of memory", nullptr);
    const char *p[2] = { text[0], text[1] }; int next[2] = { 0, 0 }; char *w = merged;
    for (int i = 0; i < n_reads; ++i) {
        const int s = set_of[(size_t) i];
        if (s < 0) die("bm2_fastq_smart_pair: a read in neither set", nullptr);
        const char *q = text[s] + ends[s][(size_t) next[s]++];
        memcpy(w, p[s], (size_t) (q - p[s])); w += q - p[s]; p[s] = q;
        if (read_end) read_end->push_back(w - merged);
    }
    if (mate) {
        mate->assign((size_t) n_reads, -1);
        for (int j = 0; j + 1 < sp.set[1].n_reads; j += 2) {
            const int a = sp.read_index[1][j], b = sp.read_index[1][j + 1];
            (*mate)[(size_t) a] = b; (*mate)[(size_t) b] = a;
        }
    }
    *w = 0; *len = w - merged;
    bm2_free(text[0]); bm2_free(text[1]);
    std::lock_guard<std::mutex> lk(sh->mu);
    sh->t_split += t_split;
    return merged;
}

// --markdup: a chunk's templates (a read, or a read and its mate, which follows it) as record ranges from where each read's records end
// (read_end), each template's id (the global index of its first read) and each record's
struct ChunkTemplates { std::vector<int64_t> starts, first, id, rec_id; };
void chunk_templates(const char *text, int64_t len, const std::vector<int64_t> &read_end, const std::vector<int64_t> &mate, long long first_read,
                     ChunkTemplates &T) {
    for (int64_t q = 0; q + 4 <= len; q += 4 + *(const int32_t *) (text + q)) T.starts.push_back(q);
    size_t k = 0;
    for (size_t i = 0; i < read_end.size(); ++i) {
        const int64_t m = mate.empty() ? -1 : mate[i];
        if (m >= 0 && (size_t) m < i) continue;
        if (m >= 0 && (size_t) m != i + 1) die("--markdup: the mates of a pair are not adjacent in the output", nullptr);
        const int64_t id = first_read + (long long) i, end = read_end[m >= 0 ? i + 1 : i];
        T.first.push_back((int64_t) k); T.id.push_back(id);
        for (; k < T.starts.size() && T.starts[k] < end; ++k) T.rec_id.push_back(id);
    }
    T.first.push_back((int64_t) k);
    if (k != T.starts.size()) die("--markdup: records after the last read", nullptr);
}

void worker(Shared *sh, bm2_ctx *ctx) {
    for (;;) {
        Chunk ck;
        {
            std::unique_lock<std::mutex> lk(sh->mu);
            sh->cv_work.wait(lk, [&] { return !sh->queue.empty() || sh->done; });
            if (sh->queue.empty()) return;
            ck = std::move(sh->queue.front()); sh->queue.pop_front();
            sh->cv_room.notify_one();
        }
        const double t0 = now_s();
        bm2_fastq_batch fq;
        const uint8_t *qp = nullptr;
        if (ck.simple) {
            if (bm2_fastq_encode(ctx, ck.c1, (int64_t) ck.n1, sh->paired ? ck.c2 : nullptr, sh->paired ? (int64_t) ck.n2 : 0, &fq)) die("bm2_fastq_encode", ctx);
        } else if (bm2_seq_encode(ctx, ck.c1, (int64_t) ck.n1, sh->paired ? ck.c2 : nullptr, sh->paired ? (int64_t) ck.n2 : 0, &fq, &qp)) die("bm2_seq_encode", ctx);
        const double t1 = now_s();
        Times t;
        char *text = nullptr; int64_t len = 0;
        std::vector<int64_t> read_end, mate;
        if (sh->smart) text = smart_pair_chunk(sh, ctx, ck, fq.n_reads, qp, &len, t, sh->markdup ? &read_end : nullptr, sh->markdup ? &mate : nullptr);
        else {
            const int64_t *cb = nullptr; const int32_t *cl = nullptr;
            if (sh->copy_comment && bm2_fastq_comments(ctx, &cb, &cl)) die("bm2_fastq_comments", ctx);
            text = align_and_format(sh, ctx, fq, ck.c1, sh->paired ? ck.c2 : nullptr, cb, cl, qp, sh->paired,
                                    sh->paired ? ck.first_read >> 1 : ck.first_read, &len, sh->markdup ? &read_end : nullptr, t);
            if (sh->markdup && sh->paired) { mate.resize(read_end.size()); for (size_t i = 0; i < mate.size(); ++i) mate[i] = (int64_t) (i ^ 1); }
        }
        ChunkTemplates tpl;
        const bm2_dup_entry *dp = nullptr, *df = nullptr; int64_t ndp = 0, ndf = 0;
        const bm2_dup_loc_entry *dlp = nullptr; int64_t counts[2] = { 0, 0 };
        double sig_ms = 0;
        if (sh->markdup) {                                               // the templates' entries, on this worker's context
            chunk_templates(text, len, read_end, mate, ck.first_read, tpl);
            if (sh->metrics) {
                if (bm2_dup_signatures_ex(ctx, (const uint8_t *) text, len, tpl.starts.data(), (int64_t) tpl.starts.size(), tpl.first.data(), tpl.id.data(),
                                          (int64_t) tpl.id.size(), &dlp, &ndp, &df, &ndf, counts)) die("bm2_dup_signatures_ex", ctx);
            } else if (bm2_dup_signatures(ctx, (const uint8_t *) text, len, tpl.starts.data(), (int64_t) tpl.starts.size(), tpl.first.data(), tpl.id.data(),
                                          (int64_t) tpl.id.size(), &dp, &ndp, &df, &ndf)) die("bm2_dup_signatures", ctx);
            bm2_last_dup_stats(ctx, &sig_ms, nullptr);
        }
        const uint8_t *outp = (const uint8_t *) text; int64_t out_len = len;
        double bgzf_ms = 0;
        if (sh->bam && !sh->sink) {                                      // BGZF blocks cut at the records' starts, within the chunk
            std::vector<int64_t> cut;
            for (int64_t q = 0; q + 4 <= len; q += 4 + *(const int32_t *) (text + q)) cut.push_back(q);
            if (bm2_bgzf_compress(ctx, (const uint8_t *) text, len, cut.data(), (int64_t) cut.size(), &outp, &out_len)) die("bm2_bgzf_compress", ctx);
            int64_t members = 0;
            bm2_last_bgzf_stats(ctx, &bgzf_ms, &members);
        }
        const double t5 = now_s();
        {   // the output keeps the chunk order
            std::unique_lock<std::mutex> lk(sh->mu);
            sh->cv_turn.wait(lk, [&] { return sh->next_to_write == ck.index; });
        }
        const double t6 = now_s();
        if (sh->sink) {
            sh->sink->add(outp, out_len, sh->markdup ? tpl.rec_id.data() : nullptr);
            if (sh->metrics) sh->sink->add_sigs_ex(dlp, ndp, df, ndf);
            else if (sh->markdup) sh->sink->add_sigs(dp, ndp, df, ndf);
        }
        else fwrite(outp, 1, (size_t) out_len, sh->out);
        bm2_free(text);
        const double t7 = now_s();
        {
            std::lock_guard<std::mutex> lk(sh->mu);
            sh->t_enc += t1 - t0; sh->t_aln += t.aln; sh->t_pes += t.pes; sh->t_sam += t.sam; sh->t_fmt += t.fmt; sh->t_turn += t6 - t5; sh->t_write += t7 - t6;
            sh->t_bam += t.bam; sh->t_bgzf += bgzf_ms / 1e3; sh->t_dup_sig += sig_ms / 1e3; sh->n_sec_supp += counts[0]; sh->n_unmapped += counts[1]; sh->bam_bytes += sh->bam ? len : 0; sh->bgzf_bytes += sh->bam && !sh->sink ? out_len : 0;
            sh->n_processed += fq.n_reads; sh->seq_chunks += !ck.simple; sh->in_flight -= ck.bytes.size();
            sh->chunk_s.push_back(t7 - t0); sh->chunk_done_s.push_back(t7 - sh->t_loop); sh->chunk_reads.push_back(fq.n_reads);
            ++sh->next_to_write;
        }
        sh->cv_turn.notify_all();
    }
}

// a ByteSource that adds up the time spent reading it
struct TimedSource : ByteSource {
    ByteSource &src; double t = 0;
    explicit TimedSource(ByteSource &s) : src(s) {}
    int64_t read(char *dst, size_t cap) override { const double t0 = now_s(); const int64_t r = src.read(dst, cap); t += now_s() - t0; return r; }
};

// the inputs' streams; a failed read ends the program as a file it cannot open does
struct Inputs {
    InputStream s[2];
    bool open(const char *f1, const char *f2) {
        if (!s[0].open(f1) || (f2 && !s[1].open(f2))) { fail(); return false; }
        return true;
    }
    void fail() const {
        fprintf(stderr, "bm2_mem: cannot read the input files%s%s\n", s[0].error_msg.empty() && s[1].error_msg.empty() ? "" : ": ",
                (s[0].error_msg + s[1].error_msg).c_str());
    }
    long long chunk(bool paired, long long task, const std::function<void(Chunk &&)> &emit, size_t *window_peak, double *read_s) {
        TimedSource t1(s[0]), t2(s[1]);
        std::string err;
        const long long n = chunk_stream(t1, paired ? &t2 : nullptr, task, emit, err, (size_t) 1 << 20, window_peak);
        if (read_s) *read_s = t1.t + t2.t;
        if (n < 0 && (!s[0].error_msg.empty() || !s[1].error_msg.empty())) { fail(); fflush(stderr); _Exit(2); }
        if (n < 0) die(err.c_str(), nullptr);
        for (const InputStream &x : s)                               // read as gzread reads it; the reference's gzclose then reports Z_BUF_ERROR
            if (x.truncated) fprintf(stderr, "[W::bm2_mem] %s ends inside a gzip member: read up to there\n", x.path());
        return n;
    }
};

}  // namespace

namespace {

void usage(const bm2_mem_opt_t &o) {
    fprintf(stderr,
"Usage: bm2_mem [options] <idxbase> <in1.fq> [in2.fq]\n"
"FASTA or FASTQ, wrapped or not, plain or gzip; `-` reads standard input.\n"
"The options of `bwa-mem2 mem`, with the same defaults and the same SAM output:\n"
"  Algorithm:  -t INT threads of the host stages [%d]   -k INT min seed length [%d]   -w INT band width [%d]   -d INT off-diagonal X-dropoff [%d]\n"
"              -r FLOAT re-seed factor [%g]   -y INT 3rd-round seed occurrence [%ld]   -c INT skip seeds with more occurrences [%d]\n"
"              -D FLOAT chain drop ratio [%.2f]   -W INT min chain weight [0]   -m INT mate rescue rounds [%d]   -S skip mate rescue\n"
"              -P skip pairing   -s INT split width [%d]   -G INT max chain gap [%d]   -N INT max chains extended [%d]   -X FLOAT mask level [%.2f]\n"
"              -Q INT mapQ length coefficient\n"
"  Scoring:    -A INT match [%d] (scales -TdBOELU unless given)   -B INT mismatch [%d]   -O INT[,INT] gap open [%d,%d]\n"
"              -E INT[,INT] gap extension [%d,%d]   -L INT[,INT] clipping [%d,%d]   -U INT unpaired pair [%d]\n"
"              -x STR preset: intractg (-B9 -O16 -L5), pacbio / pbref (-k17 -W40 -r10 -A1 -B1 -O1 -E1 -L0), ont2d (-k14 -W20 -r10 -A1 -B1 -O1 -E1 -L0)\n"
"  Input/output: -o / -f FILE output SAM [stdout]   -p smart pairing of one interleaved file (a 2nd file is ignored)\n"
"              -R STR read group line, e.g. '@RG\\tID:foo\\tSM:bar'   -H STR/FILE header line (starts with @) or file of header lines\n"
"              -j ignore the .alt file   -5 take the split alignment with the smallest coordinate as primary   -q keep the mapQ of supplementaries\n"
"              -K INT bases per chunk   -v INT verbosity (accepted, no effect)   -1 (accepted, no effect)   -T INT min score to output [%d]\n"
"              -h INT[,INT] max XA hits [%d,%d]   -a all alignments   -C append the FASTQ comment   -V XR tag with the reference annotation\n"
"              -Y soft clipping for supplementaries   -M mark shorter split hits as secondary   -I FLOAT[,FLOAT[,INT[,INT]]] insert size: mean, std, max, min\n"
"This program's own:\n"
"  -p INT      chunks in flight, one GPU context each (1-4) [2].  A -p given as a separate argument and followed by a positive decimal\n"
"              integer is this count; any other -p (alone, or in a cluster like -5SP) is smart pairing.  An index prefix that is a bare\n"
"              integer must then be written as a path (./2) after a smart-pairing -p.\n"
"  --bam       write BAM (BGZF-compressed on the GPU) instead of SAM; the same records, header and @PG line\n"
"  --sort      write coordinate-sorted BAM (implies --bam), sorted on the GPU in runs merged through temporary files next to -o\n"
"              (<out>.tmp.NNNN) or, on standard output, in ${TMPDIR:-/tmp}; the header's @HD line gets SO:coordinate\n"
"  --sort-mem SIZE  uncompressed BAM bytes per sorted run, with a K, M or G suffix [2G]\n"
"  --write-index  write the BAI index <out>.bai (needs --sort and -o)\n"
"  --markdup   mark duplicates (flag 0x400) in the sorted BAM (implies --sort): templates with the same unclipped 5' ends and strands,\n"
"              the one with the highest sum of base qualities >= 15 kept (ties: the first in the input); Picard MarkDuplicates's\n"
"              defaults, not claimed byte-equal to it (optical duplicates are marked like the others).  Holds --sort-mem / 8 bytes of\n"
"              signatures on the host\n"
"  --markdup-metrics FILE  write Picard's duplication metrics for the one library (-R's LB, else Unknown Library) to FILE, with optical\n"
"              duplicates counted on the GPU from Illumina read names (implies --markdup)\n"
"  --optical-distance N  the largest pixel distance of two optical duplicates, 0 to 2147483647 (needs --markdup-metrics) [100]\n"
"  --recal-file FILE  write GATK BaseRecalibrator's recalibration table (GATKReport, substitution covariates at GATK 4's defaults) of the\n"
"              marked BAM to FILE, with the covariates counted on the GPU (implies --markdup; needs -R and --known-sites)\n"
"  --known-sites VCF  known variant sites skipped by --recal-file, plain, gzip or BGZF; may be given more than once\n"
"  --dump-opt  print the parsed options, the -I values, the read group and the header as JSON, and exit before any GPU work\n"
"  --dump-chunks  print the chunks the input is cut into (first read, byte ranges, whether bm2_fastq_encode takes them) as JSON lines,\n"
"              and exit without loading the index\n",
            o.n_threads, o.min_seed_len, o.w, o.zdrop, o.split_factor, (long) o.max_mem_intv, o.max_occ, o.drop_ratio, o.max_matesw, o.split_width,
            o.max_chain_gap, o.max_chain_extend, o.mask_level, o.a, o.b, o.o_del, o.o_ins, o.e_del, o.e_ins, o.pen_clip5, o.pen_clip3, o.pen_unpaired,
            o.T, o.max_XA_hits, o.max_XA_hits_alt);
}

// bwa_escape (src/bwa.cpp:568-583): \t \n \r \\ decoded, any other escaped character dropped
std::string escape_decode(const char *s) {
    std::string o;
    for (const char *p = s; *p; ++p) {
        if (*p == '\\') {
            ++p;
            if (*p == 't') o += '\t'; else if (*p == 'n') o += '\n'; else if (*p == 'r') o += '\r'; else if (*p == '\\') o += '\\';
            if (!*p) break;
        } else o += *p;
    }
    return o;
}

// bwa_insert_header (src/bwa.cpp:611-625): a line that starts with '@' is appended, escapes decoded
void insert_header(std::string &hdr, bool &have, const char *s) {
    if (!s || s[0] != '@') return;
    if (have) hdr += '\n';
    hdr += escape_decode(s); have = true;
}

std::string json_str(const std::string &s) {
    std::string o = "\"";
    for (unsigned char c : s) {
        if (c == '"' || c == '\\') { o += '\\'; o += (char) c; }
        else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
        else o += (char) c;
    }
    return o + "\"";
}

// "a[,b]" of -O -E -L -h: the second value only after one punctuation character followed by a digit (src/fastmap.cpp:708-728)
void int_pair(const char *arg, int *a, int *b) {
    char *p;
    *a = *b = (int) strtol(arg, &p, 10);
    if (*p != 0 && ispunct((unsigned char) *p) && isdigit((unsigned char) p[1])) *b = (int) strtol(p + 1, &p, 10);
}

// "N" of --optical-distance: a decimal integer in [0, 2^31 - 1]
bool parse_distance(const char *s, long long *v) {
    if (!*s || strlen(s) > 10) return false;
    for (const char *p = s; *p; ++p) if (!isdigit((unsigned char) *p)) return false;
    *v = atoll(s);
    return *v <= INT32_MAX;
}

// the LB field of a read group line, or "" without one
std::string rg_library(const std::string &rg) {
    const size_t at = rg.find("\tLB:");
    if (at == std::string::npos) return std::string();
    const size_t b = at + 4, e = rg.find_first_of("\t\n", b);
    return rg.substr(b, (e == std::string::npos ? rg.size() : e) - b);
}

bool is_count(const char *s) {
    if (!*s) return false;
    for (const char *p = s; *p; ++p) if (!isdigit((unsigned char) *p)) return false;
    return atoi(s) > 0;
}

}  // namespace

int main(int argc, char **argv) {
    static const char *const optstring = "51qpaMCSPVYjk:c:v:s:r:t:R:A:B:O:E:U:w:L:d:T:Q:D:m:I:N:W:x:G:h:y:K:X:H:o:f:";
    // this program's own arguments first: `-p N` (worker count), --bam and --dump-opt are taken out of the list, walking it the way getopt will
    // (option arguments skipped, `--` ends the options), so that everything left is parsed as main_mem parses it
    int workers = 2; bool dump = false, dump_chunks = false, bam = false, sort = false, write_index = false, markdup = false;
    long long sort_mem = 2LL << 30, optical_distance = 100;
    const char *metrics_path = nullptr; bool have_distance = false;
    const char *recal_path = nullptr; std::vector<std::string> known_paths;
    std::vector<char *> av = { argv[0] };
    for (int i = 1; i < argc; ++i) {
        char *s = argv[i];
        if (!strcmp(s, "--")) { for (; i < argc; ++i) av.push_back(argv[i]); break; }
        if (!strcmp(s, "--dump-opt")) { dump = true; continue; }
        if (!strcmp(s, "--bam")) { bam = true; continue; }
        if (!strcmp(s, "--sort")) { sort = bam = true; continue; }
        if (!strcmp(s, "--write-index")) { write_index = true; continue; }
        if (!strcmp(s, "--markdup")) { markdup = sort = bam = true; continue; }
        if (!strcmp(s, "--markdup-metrics")) {
            if (i + 1 >= argc || !*argv[i + 1]) { fprintf(stderr, "[E::bm2_mem] --markdup-metrics takes a file name\n"); return 1; }
            metrics_path = argv[++i]; markdup = sort = bam = true; continue;
        }
        if (!strcmp(s, "--recal-file")) {
            if (i + 1 >= argc || !*argv[i + 1]) { fprintf(stderr, "[E::bm2_mem] --recal-file takes a file name\n"); return 1; }
            recal_path = argv[++i]; markdup = sort = bam = true; continue;
        }
        if (!strcmp(s, "--known-sites")) {
            if (i + 1 >= argc || !*argv[i + 1]) { fprintf(stderr, "[E::bm2_mem] --known-sites takes a VCF file name\n"); return 1; }
            known_paths.push_back(argv[++i]); continue;
        }
        if (!strcmp(s, "--optical-distance")) {
            if (i + 1 >= argc || !parse_distance(argv[i + 1], &optical_distance)) {
                fprintf(stderr, "[E::bm2_mem] --optical-distance takes a decimal integer from 0 to 2147483647\n"); return 1;
            }
            have_distance = true; ++i; continue;
        }
        if (!strcmp(s, "--sort-mem")) {
            if (i + 1 >= argc || !parse_size(argv[i + 1], &sort_mem)) {
                fprintf(stderr, "[E::bm2_mem] --sort-mem takes a positive byte count with an optional K, M or G suffix\n"); return 1;
            }
            ++i; continue;
        }
        if (!strcmp(s, "--dump-chunks")) { dump_chunks = true; continue; }
        if (!strcmp(s, "-p") && i + 1 < argc && is_count(argv[i + 1])) { workers = atoi(argv[++i]); continue; }
        av.push_back(s);
        if (s[0] != '-' || !s[1]) continue;
        for (const char *c = s + 1; *c; ++c) {
            const char *o = strchr(optstring, *c);
            if (o && o[1] == ':') { if (!c[1] && i + 1 < argc) av.push_back(argv[++i]); break; }
        }
    }
    int ac = (int) av.size(); av.push_back(nullptr);
    char **v = av.data();

    bm2_mem_opt_t opt, opt0; bm2_opt_init(&opt); memset(&opt0, 0, sizeof opt0);
    bm2_pestat_t pes[4]; memset(pes, 0, sizeof pes);
    for (auto &p : pes) p.failed = 1;
    bool use_pes = false, ignore_alt = false, copy_comment = false;
    long long fixed_k = -1; const char *out_path = nullptr, *mode = nullptr;
    std::string hdr_line, rg_line, rg_id; bool have_hdr = false, have_rg = false;
    int c; char *p;
    optind = 1;
    while ((c = getopt(ac, v, optstring)) >= 0) {
        if (c == 'k') opt.min_seed_len = atoi(optarg), opt0.min_seed_len = 1;
        else if (c == '1') { }                                        // no_mt_io: the reference's I/O threading
        else if (c == 'x') mode = optarg;
        else if (c == 'w') opt.w = atoi(optarg), opt0.w = 1;
        else if (c == 'A') opt.a = atoi(optarg), opt0.a = 1;
        else if (c == 'B') opt.b = atoi(optarg), opt0.b = 1;
        else if (c == 'T') opt.T = atoi(optarg), opt0.T = 1;
        else if (c == 'U') opt.pen_unpaired = atoi(optarg), opt0.pen_unpaired = 1;
        else if (c == 't') opt.n_threads = atoi(optarg), opt.n_threads = opt.n_threads > 1 ? opt.n_threads : 1;
        else if (c == 'o' || c == 'f') out_path = optarg;
        else if (c == 'P') opt.flag |= 0x4;                           // MEM_F_NOPAIRING
        else if (c == 'a') opt.flag |= 0x8;                           // MEM_F_ALL
        else if (c == 'p') opt.flag |= 0x2 | 0x400;                   // MEM_F_PE | MEM_F_SMARTPE
        else if (c == 'M') opt.flag |= 0x10;                          // MEM_F_NO_MULTI
        else if (c == 'S') opt.flag |= 0x20;                          // MEM_F_NO_RESCUE
        else if (c == 'Y') opt.flag |= 0x200;                         // MEM_F_SOFTCLIP
        else if (c == 'V') opt.flag |= 0x100;                         // MEM_F_REF_HDR
        else if (c == '5') opt.flag |= 0x800 | 0x1000;                // MEM_F_PRIMARY5 | MEM_F_KEEP_SUPP_MAPQ
        else if (c == 'q') opt.flag |= 0x1000;                        // MEM_F_KEEP_SUPP_MAPQ
        else if (c == 'c') opt.max_occ = atoi(optarg), opt0.max_occ = 1;
        else if (c == 'd') opt.zdrop = atoi(optarg), opt0.zdrop = 1;
        else if (c == 'v') { }                                        // verbosity of the reference's stderr
        else if (c == 'j') ignore_alt = true;
        else if (c == 'r') opt.split_factor = (float) atof(optarg), opt0.split_factor = 1.f;
        else if (c == 'D') opt.drop_ratio = (float) atof(optarg), opt0.drop_ratio = 1.f;
        else if (c == 'm') opt.max_matesw = atoi(optarg), opt0.max_matesw = 1;
        else if (c == 's') opt.split_width = atoi(optarg), opt0.split_width = 1;
        else if (c == 'G') opt.max_chain_gap = atoi(optarg), opt0.max_chain_gap = 1;
        else if (c == 'N') opt.max_chain_extend = atoi(optarg), opt0.max_chain_extend = 1;
        else if (c == 'W') opt.min_chain_weight = atoi(optarg), opt0.min_chain_weight = 1;
        else if (c == 'y') opt.max_mem_intv = (uint64_t) atol(optarg), opt0.max_mem_intv = 1;
        else if (c == 'C') copy_comment = true;
        else if (c == 'K') fixed_k = atoll(optarg);
        else if (c == 'X') opt.mask_level = (float) atof(optarg);
        else if (c == 'h') { opt0.max_XA_hits = opt0.max_XA_hits_alt = 1; int_pair(optarg, &opt.max_XA_hits, &opt.max_XA_hits_alt); }
        else if (c == 'Q') {
            opt0.mapQ_coef_len = 1;
            opt.mapQ_coef_len = (float) atoi(optarg);
            opt.mapQ_coef_fac = opt.mapQ_coef_len > 0 ? (int) log(opt.mapQ_coef_len) : 0;
        }
        else if (c == 'O') { opt0.o_del = opt0.o_ins = 1; int_pair(optarg, &opt.o_del, &opt.o_ins); }
        else if (c == 'E') { opt0.e_del = opt0.e_ins = 1; int_pair(optarg, &opt.e_del, &opt.e_ins); }
        else if (c == 'L') { opt0.pen_clip5 = opt0.pen_clip3 = 1; int_pair(optarg, &opt.pen_clip5, &opt.pen_clip3); }
        else if (c == 'R') {                                          // bwa_set_rg (src/bwa.cpp:585-609)
            rg_id.clear(); have_rg = false;
            if (strstr(optarg, "@RG") != optarg) { fprintf(stderr, "[E::bm2_mem] the read group line is not started with @RG\n"); return 1; }
            rg_line = escape_decode(optarg);
            const size_t at = rg_line.find("\tID:");
            if (at == std::string::npos) { fprintf(stderr, "[E::bm2_mem] no ID at the read group line\n"); return 1; }
            const size_t b = at + 4, e = rg_line.find_first_of("\t\n", b);
            rg_id = rg_line.substr(b, (e == std::string::npos ? rg_line.size() : e) - b);
            if (rg_id.size() + 1 > 256) { fprintf(stderr, "[E::bm2_mem] @RG:ID is longer than 255 characters\n"); return 1; }
            have_rg = true;
        }
        else if (c == 'H') {
            if (optarg[0] != '@') {
                FILE *fp = fopen(optarg, "r");
                if (fp) {
                    char buf[0x10000];
                    while (fgets(buf, 0xffff, fp)) { const size_t n = strlen(buf); if (n && buf[n - 1] == '\n') buf[n - 1] = 0; insert_header(hdr_line, have_hdr, buf); }
                    fclose(fp);
                }
            } else insert_header(hdr_line, have_hdr, optarg);
        }
        else if (c == 'I') {                                          // src/fastmap.cpp:760-775, FR orientation only
            use_pes = true;
            pes[1].failed = 0;
            pes[1].avg = strtod(optarg, &p);
            pes[1].std = pes[1].avg * .1;
            if (*p != 0 && ispunct((unsigned char) *p) && isdigit((unsigned char) p[1])) pes[1].std = strtod(p + 1, &p);
            pes[1].high = (int) (pes[1].avg + 4. * pes[1].std + .499);
            pes[1].low = (int) (pes[1].avg - 4. * pes[1].std + .499);
            if (pes[1].low < 1) pes[1].low = 1;
            if (*p != 0 && ispunct((unsigned char) *p) && isdigit((unsigned char) p[1])) pes[1].high = (int) (strtod(p + 1, &p) + .499);
            if (*p != 0 && ispunct((unsigned char) *p) && isdigit((unsigned char) p[1])) pes[1].low = (int) (strtod(p + 1, &p) + .499);
        }
        else { usage(opt); return 1; }
    }
    if (have_rg) insert_header(hdr_line, have_hdr, rg_line.c_str());
    if (opt.n_threads < 1) opt.n_threads = 1;
    if (optind + 2 != ac && optind + 3 != ac) { usage(opt); return 1; }
    if (mode) {                                                       // src/fastmap.cpp:801-843
        if (!strcmp(mode, "intractg")) {
            if (!opt0.o_del) opt.o_del = 16;
            if (!opt0.o_ins) opt.o_ins = 16;
            if (!opt0.b) opt.b = 9;
            if (!opt0.pen_clip5) opt.pen_clip5 = 5;
            if (!opt0.pen_clip3) opt.pen_clip3 = 5;
        } else if (!strcmp(mode, "pacbio") || !strcmp(mode, "pbref") || !strcmp(mode, "ont2d")) {
            if (!opt0.o_del) opt.o_del = 1;
            if (!opt0.e_del) opt.e_del = 1;
            if (!opt0.o_ins) opt.o_ins = 1;
            if (!opt0.e_ins) opt.e_ins = 1;
            if (!opt0.b) opt.b = 1;
            if (opt0.split_factor == 0.f) opt.split_factor = 10.f;
            const bool ont = !strcmp(mode, "ont2d");
            if (!opt0.min_chain_weight) opt.min_chain_weight = ont ? 20 : 40;
            if (!opt0.min_seed_len) opt.min_seed_len = ont ? 14 : 17;
            if (!opt0.pen_clip5) opt.pen_clip5 = 0;
            if (!opt0.pen_clip3) opt.pen_clip3 = 0;
        } else { fprintf(stderr, "[E::bm2_mem] unknown read type '%s'\n", mode); return 1; }
    } else if (opt0.a) {                                              // update_a (src/fastmap.cpp:547-561)
        if (!opt0.b) opt.b *= opt.a;
        if (!opt0.T) opt.T *= opt.a;
        if (!opt0.o_del) opt.o_del *= opt.a;
        if (!opt0.e_del) opt.e_del *= opt.a;
        if (!opt0.o_ins) opt.o_ins *= opt.a;
        if (!opt0.e_ins) opt.e_ins *= opt.a;
        if (!opt0.zdrop) opt.zdrop *= opt.a;
        if (!opt0.pen_clip5) opt.pen_clip5 *= opt.a;
        if (!opt0.pen_clip3) opt.pen_clip3 *= opt.a;
        if (!opt0.pen_unpaired) opt.pen_unpaired *= opt.a;
    }
    {   // bwa_fill_scmat (src/bwa.cpp:246-257)
        int k = 0;
        for (int i = 0; i < 4; ++i) { for (int j = 0; j < 4; ++j) opt.mat[k++] = (int8_t) (i == j ? opt.a : -opt.b); opt.mat[k++] = -1; }
        for (int j = 0; j < 5; ++j) opt.mat[k++] = -1;
    }
    const int threads = opt.n_threads;
    if (workers > 4) workers = 4;
    if (have_distance && !metrics_path) { fprintf(stderr, "[E::bm2_mem] --optical-distance needs --markdup-metrics FILE\n"); return 1; }
    if (!known_paths.empty() && !recal_path) { fprintf(stderr, "[E::bm2_mem] --known-sites needs --recal-file FILE\n"); return 1; }
    if (recal_path && known_paths.empty()) { fprintf(stderr, "[E::bm2_mem] --recal-file needs at least one --known-sites VCF\n"); return 1; }
    if (recal_path && !have_rg) { fprintf(stderr, "[E::bm2_mem] --recal-file needs a read group (-R)\n"); return 1; }
    if (write_index && (!sort || !out_path)) { fprintf(stderr, "[E::bm2_mem] --write-index needs --sort and -o FILE\n"); return 1; }
    const bool smart = (opt.flag & 0x400) != 0;
    const char *prefix = v[optind], *f1 = v[optind + 1], *f2 = optind + 2 < ac ? v[optind + 2] : nullptr;
    if (f2 && smart) { fprintf(stderr, "[W::bm2_mem] when '-p' is in use, the second query file is ignored.\n"); f2 = nullptr; }
    if (f2) opt.flag |= 0x2;                                          // MEM_F_PE
    const long long task = fixed_k > 0 ? fixed_k : (long long) opt.chunk_size * threads;
    opt.chunk_size = task;                                            // as main_mem leaves it (src/fastmap.cpp:949)
    if (dump_chunks) {
        Inputs in;
        if (!in.open(f1, f2)) return 2;
        in.chunk(f2 != nullptr, task, [&](Chunk &&ck) {
            printf("{\"first_read\": %lld, \"offset1\": %lld, \"bytes1\": %zu, \"offset2\": %lld, \"bytes2\": %zu, \"simple\": %s}\n", ck.first_read,
                   (long long) ck.off1, ck.n1, (long long) ck.off2, ck.n2, ck.simple ? "true" : "false");
            fflush(stdout);
        }, nullptr, nullptr);
        return 0;
    }
    const double t_start = now_s();
    bm2_index_desc *idx = nullptr;
    if (bm2_index_load(prefix, &idx)) { fprintf(stderr, "bm2_mem: cannot load the index %s\n", prefix); return 2; }
    if (ignore_alt) memset((void *) idx->ann_is_alt, 0, (size_t) idx->n_seqs * sizeof(int32_t));
    // contig names and annotations: <prefix>.ann (src/bntseq.cpp:106-177): "l_pac n_seqs seed", then per contig "gi name[ anno]" and
    // "offset len n_ambs"; the annotation is the rest of the name line without its first character, "(null)" meaning none
    std::vector<std::string> names, annos; std::vector<long long> lens; std::vector<int64_t> offs;
    {
        FILE *f = fopen((std::string(prefix) + ".ann").c_str(), "r");
        if (!f) { fprintf(stderr, "bm2_mem: cannot open %s.ann\n", prefix); return 2; }
        std::vector<char> line(1 << 16);
        if (!fgets(line.data(), (int) line.size(), f)) return 2;
        for (int i = 0; i < idx->n_seqs; ++i) {
            char nm[8193]; long long gi, off, len; int amb, at = 0;
            if (!fgets(line.data(), (int) line.size(), f) || sscanf(line.data(), "%lld %8192s%n", &gi, nm, &at) != 2) return 2;
            std::string rest(line.data() + at);
            if (!rest.empty() && rest.back() == '\n') rest.pop_back();
            annos.push_back(rest.size() > 1 && rest != " (null)" ? rest.substr(1) : std::string());
            if (!fgets(line.data(), (int) line.size(), f) || sscanf(line.data(), "%lld %lld %d", &off, &len, &amb) != 3) return 2;
            names.push_back(nm); lens.push_back(len); offs.push_back(off);
        }
        fclose(f);
    }
    // the header as bwa_print_sam_hdr (src/bwa.cpp:523-565) writes it: @SQ lines (AH:* on ALT contigs) unless -H gave @SQ lines, the -H lines,
    // the -R line; then this program's @PG line
    std::string header;
    {
        int n_sq = 0;
        for (size_t q = 0; (q = hdr_line.find("@SQ\t", q)) != std::string::npos; q += 4) if (q == 0 || hdr_line[q - 1] == '\n') ++n_sq;
        if (!have_hdr || n_sq == 0)
            for (size_t i = 0; i < names.size(); ++i)
                header += "@SQ\tSN:" + names[i] + "\tLN:" + std::to_string(lens[i]) + (idx->ann_is_alt && idx->ann_is_alt[i] ? "\tAH:*\n" : "\n");
        if (have_hdr) header += hdr_line + "\n";
        if (sort) header = header_with_sort_order(header, "coordinate");
    }
    if (dump) {
        const bm2_mem_opt_t &o = opt;
        printf("{\"a\": %d, \"b\": %d, \"o_del\": %d, \"e_del\": %d, \"o_ins\": %d, \"e_ins\": %d, \"pen_unpaired\": %d, \"pen_clip5\": %d, \"pen_clip3\": %d, "
               "\"w\": %d, \"zdrop\": %d, \"max_mem_intv\": %llu, \"T\": %d, \"flag\": %d, \"min_seed_len\": %d, \"min_chain_weight\": %d, "
               "\"max_chain_extend\": %d, \"split_factor\": %.9g, \"split_width\": %d, \"max_occ\": %d, \"max_chain_gap\": %d, \"n_threads\": %d, "
               "\"chunk_size\": %lld, \"mask_level\": %.9g, \"drop_ratio\": %.9g, \"XA_drop_ratio\": %.9g, \"mask_level_redun\": %.9g, "
               "\"mapQ_coef_len\": %.9g, \"mapQ_coef_fac\": %d, \"max_ins\": %d, \"max_matesw\": %d, \"max_XA_hits\": %d, \"max_XA_hits_alt\": %d, \"mat\": [",
               o.a, o.b, o.o_del, o.e_del, o.o_ins, o.e_ins, o.pen_unpaired, o.pen_clip5, o.pen_clip3, o.w, o.zdrop, (unsigned long long) o.max_mem_intv, o.T,
               o.flag, o.min_seed_len, o.min_chain_weight, o.max_chain_extend, o.split_factor, o.split_width, o.max_occ, o.max_chain_gap, o.n_threads,
               (long long) o.chunk_size, o.mask_level, o.drop_ratio, o.XA_drop_ratio, o.mask_level_redun, o.mapQ_coef_len, o.mapQ_coef_fac, o.max_ins,
               o.max_matesw, o.max_XA_hits, o.max_XA_hits_alt);
        for (int i = 0; i < 25; ++i) printf("%s%d", i ? ", " : "", o.mat[i]);
        printf("], \"pes\": ");
        if (use_pes) printf("{\"low\": %d, \"high\": %d, \"avg\": %.17g, \"std\": %.17g}", pes[1].low, pes[1].high, pes[1].avg, pes[1].std);
        else printf("null");
        printf(", \"rg_id\": %s, \"copy_comment\": %s, \"ignore_alt\": %s, \"smart_pairing\": %s, \"workers\": %d, \"files\": %d, \"bam\": %s, ",
               have_rg ? json_str(rg_id).c_str() : "null", copy_comment ? "true" : "false", ignore_alt ? "true" : "false", smart ? "true" : "false",
               workers, f2 ? 2 : 1, bam ? "true" : "false");
        if (sort) printf("\"sort\": true, \"sort_mem\": %lld, \"write_index\": %s, ", sort_mem, write_index ? "true" : "false");
        if (markdup) printf("\"markdup\": true, ");
        if (metrics_path) printf("\"markdup_metrics\": %s, \"optical_distance\": %lld, ", json_str(metrics_path).c_str(), optical_distance);
        if (recal_path) {
            printf("\"recal_file\": %s, \"known_sites\": [", json_str(recal_path).c_str());
            for (size_t k = 0; k < known_paths.size(); ++k) printf("%s%s", k ? ", " : "", json_str(known_paths[k]).c_str());
            printf("], ");
        }
        printf("\"header\": %s}\n", json_str(header).c_str());
        bm2_index_free(idx);
        return 0;
    }
    if (bam)                                                          // BAM stores l_ref as int32 (SAMv1 §4.2)
        for (size_t i = 0; i < names.size(); ++i)
            if (lens[i] > INT32_MAX) { fprintf(stderr, "[E::bm2_mem] contig %s is %lld bp long: BAM cannot store a contig longer than 2^31-1\n", names[i].c_str(), lens[i]); return 1; }
    if (write_index)                                                  // BAI's bins reach 2^29 (SAMv1 §5.3); longer contigs need CSI
        for (size_t i = 0; i < names.size(); ++i)
            if (lens[i] > (1LL << 29) - 1) { fprintf(stderr, "[E::bm2_mem] contig %s is %lld bp long: BAI cannot index a contig longer than 2^29-1\n", names[i].c_str(), lens[i]); return 1; }
    // --known-sites: the VCFs are read on a thread of their own while the reads align; an error in them ends the program as soon as it is found
    KnownSites known;
    double known_s = 0;
    std::thread known_thread;                                         // started with the workers, joined before the final sort pass
    std::vector<const char *> cnames, canno;
    for (size_t i = 0; i < names.size(); ++i) { cnames.push_back(names[i].c_str()); canno.push_back(annos[i].c_str()); }
    std::vector<bm2_ctx *> ctxs((size_t) workers, nullptr);
    if (bm2_create(&ctxs[0], 0, idx, &opt)) { fprintf(stderr, "bm2_mem: %s\n", bm2_last_error(nullptr)); return 3; }
    for (int w = 1; w < workers; ++w)
        if (bm2_create_sibling(&ctxs[w], ctxs[0])) { fprintf(stderr, "bm2_mem: %s\n", bm2_last_error(ctxs[0])); return 3; }
    bm2_ctx *sort_ctx = nullptr;                                      // --sort: the runs are sorted on a context of their own
    if (sort) {
        if (bm2_create_sibling(&sort_ctx, ctxs[0])) { fprintf(stderr, "bm2_mem: %s\n", bm2_last_error(ctxs[0])); return 3; }
        int64_t need = 0, avail = 0;
        if (bm2_bam_sort_memory_ex(sort_ctx, sort_mem, markdup ? 1 : 0, &need, &avail)) die("bm2_bam_sort_memory", sort_ctx);
        if (need > avail) {
            fprintf(stderr, "[E::bm2_mem] --sort-mem %lld: one run sort needs %lld bytes of device memory, %lld bytes free\n", sort_mem, (long long) need, (long long) avail);
            return 3;
        }
        // --recal-file: the two known-site bitsets (2 bits per reference base) and the counters (1.5 MB) on the sort context too
        const int64_t sites = recal_path ? 2 * ((idx->l_pac + 63) / 64) * 8 + (2 << 20) : 0;
        if (sites && need + sites > avail) {
            fprintf(stderr, "[E::bm2_mem] --recal-file: the run sort and the known-site bitsets need %lld bytes of device memory, %lld bytes free\n",
                    (long long) (need + sites), (long long) avail);
            return 3;
        }
    }
    const double t_index = now_s() - t_start;
    Inputs in;
    if (!in.open(f1, f2)) return 2;
    FILE *out = out_path ? fopen(out_path, "wb") : stdout;
    int64_t header_z = 0;
    if (!out) { fprintf(stderr, "bm2_mem: cannot open %s\n", out_path); return 2; }
    header += std::string("@PG\tID:bm2_mem\tPN:bm2_mem\tVN:b200-r2\tCL:") + argv[0];
    for (int i = 1; i < argc; ++i) header += std::string(" ") + argv[i];
    header += "\n";
    if (!bam) fwrite(header.data(), 1, header.size(), out);
    else {   // SAMv1 §4.2: magic, the header text, then the index's contigs (refIDs index this list, whatever -H put in the text), in blocks of its own
        std::string h("BAM\1", 4);
        auto i32 = [&](int32_t v) { h.append((const char *) &v, 4); };
        i32((int32_t) header.size()); h += header;
        i32((int32_t) names.size());
        for (size_t i = 0; i < names.size(); ++i) { i32((int32_t) names[i].size() + 1); h.append(names[i].c_str(), names[i].size() + 1); i32((int32_t) lens[i]); }
        const uint8_t *z = nullptr; int64_t zl = 0;
        if (bm2_bgzf_compress(ctxs[0], (const uint8_t *) h.data(), (int64_t) h.size(), nullptr, 0, &z, &zl)) die("bm2_bgzf_compress", ctxs[0]);
        fwrite(z, 1, (size_t) zl, out);
        header_z = zl;
    }
    BamSortSink sink;
    if (sort) {
        // without --markdup no template ids are passed, and bm2_bam_sort_compress_ex is bm2_bam_sort_compress
        sink.sort_ex = [sort_ctx, recal_path](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, const int64_t *tids, const uint8_t *c, int64_t cl, int last,
                                  bm2_sort_out *o, const int64_t **tids_out, double *device_s) {
            const int rc = bm2_bam_sort_compress_ex(sort_ctx, r, n, st, nr, tids, c, cl, last, o, tids_out);
            bm2_bqsr_tables_t bt;
            if (rc && recal_path && !bm2_bqsr_tables(sort_ctx, &bt) && bt.err_kind) {       // a read --recal-file cannot count
                fprintf(stderr, "[E::bm2_mem] --recal-file: %s\n", bm2_last_error(sort_ctx)); fflush(stderr); _Exit(1);
            }
            double ms[4] = { 0, 0, 0, 0 };
            bm2_last_sort_stats(sort_ctx, ms);
            *device_s = (ms[0] + ms[1] + ms[2] + ms[3]) / 1e3;
            return rc;
        };
        sink.fail = [sort_ctx](const std::string &m) { die(m.c_str(), m.compare(0, 4, "bm2_") == 0 ? sort_ctx : nullptr); };
        sink.run_bytes = sort_mem; sink.threads = threads;
        if (markdup) {
            sink.dup = [sort_ctx](const bm2_dup_entry *e, int64_t n, int resolve, const bm2_dup_entry **sorted, const int64_t **dups, int64_t *n_dups,
                                  double *device_s) {
                const int rc = bm2_dup_resolve(sort_ctx, e, n, resolve, sorted, dups, n_dups);
                double ms = 0;
                bm2_last_dup_stats(sort_ctx, nullptr, &ms);
                *device_s = ms / 1e3;
                return rc;
            };
            sink.dup_set = [sort_ctx](const uint64_t *bits, int64_t n_bits) { return bm2_dup_set(sort_ctx, bits, n_bits); };
            sink.sig_bytes = sort_mem / 8;
            if (metrics_path)
                sink.dup_ex = [sort_ctx, optical_distance](const bm2_dup_loc_entry *e, int64_t n, int resolve, const bm2_dup_loc_entry **sorted,
                                                           const int64_t **dups, int64_t *n_dups, int64_t *n_optical, double *device_s) {
                    const int rc = bm2_dup_resolve_ex(sort_ctx, e, n, resolve, optical_distance, sorted, dups, n_dups, n_optical);
                    double ms = 0;
                    bm2_last_dup_stats(sort_ctx, nullptr, &ms);
                    *device_s = ms / 1e3;
                    return rc;
                };
        }
        if (recal_path)
            sink.before_final = [&] {
                known_thread.join();
                std::vector<int64_t> holes;                               // <prefix>.amb: "l_pac n_seqs n_holes", then "offset len char" per hole
                FILE *f = fopen((std::string(prefix) + ".amb").c_str(), "r");
                long long a, b, nh = 0; char ch;
                if (!f || fscanf(f, "%lld %lld %lld", &a, &b, &nh) != 3) die("--recal-file: cannot read the index's .amb file", nullptr);
                for (long long k = 0; k < nh; ++k) {
                    if (fscanf(f, "%lld %lld %c", &a, &b, &ch) != 3) die("--recal-file: cannot read the index's .amb file", nullptr);
                    holes.push_back(a); holes.push_back(a + b);
                }
                fclose(f);
                const std::string rg = bqsr_read_group(rg_line);
                if (bm2_bqsr_sites(sort_ctx, known.covered.data(), known.junction.data(), idx->l_pac, holes.data(), (int64_t) holes.size() / 2, rg.c_str()))
                    die("bm2_bqsr_sites", sort_ctx);
            };
        if (out_path) sink.tmp_prefix = std::string(out_path) + ".tmp.";
        else {
            const char *td = getenv("TMPDIR");
            sink.tmp_prefix = std::string(td && *td ? td : "/tmp") + "/bm2_mem." + std::to_string((long long) getpid()) + ".";
        }
    }
    Shared sh;
    sh.opt = &opt; sh.idx = idx; sh.cnames = cnames.data(); sh.paired = f2 != nullptr; sh.smart = smart; sh.threads = threads; sh.out = out;
    sh.pes0 = use_pes ? pes : nullptr; sh.copy_comment = copy_comment; sh.bam = bam; sh.sink = sort ? &sink : nullptr; sh.markdup = markdup;
    sh.metrics = metrics_path != nullptr;
    sh.extra.rg_id = have_rg ? rg_id.c_str() : nullptr; sh.extra.contig_anno = canno.data(); sh.extra.ref_hdr = (opt.flag & 0x100) != 0;
    if (recal_path) {
        std::vector<int64_t> lens64(lens.begin(), lens.end());
        known_thread = std::thread([&known, &known_s, &known_paths, &names, &offs, lens64, l_pac = idx->l_pac] {
            const double t0 = now_s();
            const std::string err = read_known_sites(known_paths, names, offs, lens64, l_pac, known);
            if (!err.empty()) { fprintf(stderr, "[E::bm2_mem] --known-sites: %s\n", err.c_str()); fflush(stderr); _Exit(1); }
            known_s = now_s() - t0;
        });
    }
    sh.t_loop = now_s();
    std::vector<std::thread> pool;
    for (int w = 0; w < workers; ++w) pool.emplace_back(worker, &sh, ctxs[w]);
    size_t window_peak = 0, input_peak = 0; double read_s = 0;
    const long long n_chunks = in.chunk(f2 != nullptr, task, [&](Chunk &&ck) {
        std::unique_lock<std::mutex> lk(sh.mu);
        sh.cv_room.wait(lk, [&] { return (int) sh.queue.size() < workers; });
        sh.in_flight += ck.bytes.size();
        input_peak = std::max(input_peak, sh.in_flight + window_peak + in.s[0].peak_bytes() + in.s[1].peak_bytes());
        sh.queue.push_back(std::move(ck));
        sh.cv_work.notify_one();
    }, &window_peak, &read_s);
    { std::lock_guard<std::mutex> lk(sh.mu); sh.done = true; }
    sh.cv_work.notify_all();
    for (auto &t : pool) t.join();
    const double loop_s = now_s() - sh.t_loop;
    BaiBuilder bai((int) names.size());
    double index_s = 0;
    if (sort) {
        sink.n_reads = sh.n_processed;
        sink.finish(out, (uint64_t) header_z, write_index ? &bai : nullptr);
        if (write_index) {
            const double t0 = now_s();
            const std::string b = bai.bytes(), path = std::string(out_path) + ".bai";
            FILE *f = fopen(path.c_str(), "wb");
            if (!f || fwrite(b.data(), 1, b.size(), f) != b.size() || fclose(f)) { fprintf(stderr, "bm2_mem: cannot write %s\n", path.c_str()); return 2; }
            index_s = now_s() - t0;
        }
    }
    if (bam) {                                                        // the BGZF end-of-file marker (SAMv1 §4.1.2)
        static const uint8_t eof[28] = { 0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0 };
        fwrite(eof, 1, sizeof eof, out);
    }
    if (out != stdout) fclose(out);
    if (metrics_path) {
        fflush(stdout);                                               // after the BAM is complete; through a temporary name, so never partial
        DupMetrics m;
        const std::string lb = have_rg ? rg_library(rg_line) : std::string();
        if (!lb.empty()) m.library = lb;
        m.unpaired_reads = sink.dup_frag_entries; m.read_pairs = sink.dup_pair_entries;
        m.secondary_or_supplementary = sh.n_sec_supp; m.unmapped = sh.n_unmapped;
        m.unpaired_dups = sink.dup_frag_templates; m.pair_dups = sink.dup_pair_templates; m.optical_pairs = sink.dup_optical_pairs;
        std::string args;
        for (int i = 1; i < argc; ++i) args += std::string(i > 1 ? " " : "") + argv[i];
        const std::string text = dup_metrics_text(m, args), path = metrics_path, tmp = path + ".tmp";
        FILE *f = fopen(tmp.c_str(), "wb");
        if (!f || fwrite(text.data(), 1, text.size(), f) != text.size() || fclose(f) || rename(tmp.c_str(), path.c_str())) {
            unlink(tmp.c_str());
            fprintf(stderr, "bm2_mem: cannot write %s\n", path.c_str()); return 2;
        }
    }
    bm2_bqsr_tables_t bt; memset(&bt, 0, sizeof bt);
    if (recal_path) {
        fflush(stdout);                                               // after the BAM is complete; through a temporary name, so never partial
        if (bm2_bqsr_tables(sort_ctx, &bt)) die("bm2_bqsr_tables", sort_ctx);
        const std::string text = bqsr_report_text(bt.read_group, bt.qual_obs, bt.qual_err, bt.ctx_obs, bt.ctx_err, bt.cyc_obs, bt.cyc_err),
                          path = recal_path, tmp = path + ".tmp";
        FILE *f = fopen(tmp.c_str(), "wb");
        if (!f || fwrite(text.data(), 1, text.size(), f) != text.size() || fclose(f) || rename(tmp.c_str(), path.c_str())) {
            unlink(tmp.c_str());
            fprintf(stderr, "bm2_mem: cannot write %s\n", path.c_str()); return 2;
        }
    }
    fprintf(stderr, "{\"reads\": %lld, \"chunks\": %lld, \"workers\": %d, \"loop_s\": %.6f, \"index_and_context_s\": %.3f, \"fastq_encode_s\": %.6f, \"seed_chain_extend_s\": %.6f, "
                    "\"pestat_s\": %.6f, \"sam_stage_s\": %.6f, \"sam_format_s\": %.6f, \"wait_for_turn_s\": %.6f, \"write_s\": %.6f, \"chunk_s\": [",
            sh.n_processed, n_chunks, workers, loop_s, t_index, sh.t_enc, sh.t_aln, sh.t_pes, sh.t_sam, sh.t_fmt, sh.t_turn, sh.t_write);
    for (size_t i = 0; i < sh.chunk_s.size(); ++i) fprintf(stderr, "%s%.6f", i ? ", " : "", sh.chunk_s[i]);
    fprintf(stderr, "], \"chunk_done_s\": [");
    for (size_t i = 0; i < sh.chunk_done_s.size(); ++i) fprintf(stderr, "%s%.6f", i ? ", " : "", sh.chunk_done_s[i]);
    fprintf(stderr, "], \"chunk_reads\": [");
    for (size_t i = 0; i < sh.chunk_reads.size(); ++i) fprintf(stderr, "%s%lld", i ? ", " : "", sh.chunk_reads[i]);
    fprintf(stderr, "], \"smart_pair_split_s\": %.6f, \"seq_encode_chunks\": %lld, \"read_s\": %.6f, \"gzip_members\": %lld, \"input_peak_bytes\": %zu",
            sh.t_split, sh.seq_chunks, read_s, (long long) (in.s[0].gzip_members + in.s[1].gzip_members), input_peak);
    if (bam) fprintf(stderr, ", \"bam_format_s\": %.6f, \"bgzf_s\": %.6f, \"bam_bytes\": %lld, \"bgzf_bytes\": %lld", sh.t_bam, sh.t_bgzf, sh.bam_bytes, sh.bgzf_bytes);
    if (sort)
        fprintf(stderr, ", \"sort_runs\": %lld, \"spill_bytes\": %lld, \"sort_s\": %.6f, \"merge_s\": %.6f, \"merge_windows\": %lld, \"index_s\": %.6f",
                (long long) std::max<size_t>(sink.runs.size(), 1), (long long) sink.spill_bytes, sink.sort_s, sink.merge_s, (long long) sink.merge_windows, index_s);
    if (markdup)
        fprintf(stderr, ", \"markdup_s\": %.6f, \"dup_templates\": %lld, \"dup_pair_templates\": %lld, \"dup_fragment_templates\": %lld, \"dup_records\": %lld, "
                        "\"dup_sig_runs\": %lld, \"dup_sig_bytes\": %lld", sh.t_dup_sig + sink.markdup_s, (long long) sink.dup_templates,
                (long long) sink.dup_pair_templates, (long long) sink.dup_frag_templates, (long long) sink.dup_records, (long long) sink.dup_sig_runs,
                (long long) sink.dup_sig_bytes);
    if (metrics_path) fprintf(stderr, ", \"dup_optical_pairs\": %lld", (long long) sink.dup_optical_pairs);
    if (recal_path)
        fprintf(stderr, ", \"bqsr_s\": %.6f, \"bqsr_reads\": %lld, \"bqsr_bases\": %lld, \"known_sites\": %lld, \"known_sites_s\": %.6f", bt.ms / 1e3,
                (long long) bt.reads, (long long) bt.bases, (long long) known.records, known_s);
    fprintf(stderr, "}\n");
    if (sort_ctx) bm2_destroy(sort_ctx);
    for (int w = workers - 1; w >= 0; --w) bm2_destroy(ctxs[w]);
    bm2_index_free(idx);
    return 0;
}

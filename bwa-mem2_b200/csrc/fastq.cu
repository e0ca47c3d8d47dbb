// fastq.cu — FASTQ bytes -> read batch, parsed and encoded on the GPU (SURVEY 8f item 3: host I/O on the fast side).
//
// Replaces the parsing of bseq_read_orig (reference src/bwa.cpp:170-216 over kseq.h: name up to the first blank, trim_readno :62-66,
// one record = four lines) and the in-place base encoding at the head of mem_kernel1_core (src/bwamem.cpp:992-1000: nst_nt4_table,
// src/bntseq.cpp:54-71).  At the reference's speed (one kseq stream per file) the parser would feed about a million reads per second;
// here the raw bytes of a chunk go to the device once (they have to cross PCIe anyway, as bytes instead of codes) and three small
// kernels do the rest: newline positions by a stream compaction, record spans + validation per record, then one warp per read writes the
// codes 0-4 and the qualities into the flat batch layout of seam 2.  Paired input: reads 2i / 2i+1 come from buffer 1 / buffer 2.
// Restriction (checked, reported as an error): four-line records (no wrapped sequence lines), chunks below 2 GiB per buffer.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "seq_grammar.cuh"
#include <cub/device/device_select.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>
#include <cub/device/device_reduce.cuh>

namespace {

struct IsNewline {
    const char *raw;
    __device__ __forceinline__ bool operator()(const int &i) const { return raw[i] == '\n'; }
};

struct NewlineAsInt {
    const char *raw;
    __device__ __forceinline__ int operator()(const int &i) const { return raw[i] == '\n' ? 1 : 0; }
};

struct Span { int32_t seq_beg, seq_len, qual_beg, name_beg, name_len, cmt_beg, cmt_len, _pad; };

// one thread per record of one buffer: line l of record r spans (nl[4r + l - 1] + 1 .. nl[4r + l])
__global__ void fastq_spans_kernel(const char *__restrict__ raw, const int32_t *__restrict__ nl, int n_rec, int file, int stride, Span *spans,
                                   int64_t *lens, int *err) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rec) return;
    const int l0 = r == 0 ? 0 : nl[4 * r - 1] + 1;
    int e0 = nl[4 * r], l1 = e0 + 1, e1 = nl[4 * r + 1], l2 = e1 + 1, e2 = nl[4 * r + 2], l3 = e2 + 1, e3 = nl[4 * r + 3];
    if (e0 > l0 && raw[e0 - 1] == '\r') --e0;
    if (e1 > l1 && raw[e1 - 1] == '\r') --e1;
    if (e3 > l3 && raw[e3 - 1] == '\r') --e3;
    if (e0 <= l0 || raw[l0] != '@' || e2 <= l2 || raw[l2] != '+' || e3 - l3 != e1 - l1) { atomicExch(err, r + 1); }
    int ne = l0 + 1;
    while (ne < e0 && raw[ne] != ' ' && raw[ne] != '\t') ++ne;                              // the name ends at the first blank (kseq.h)
    // the comment: the rest of the line after that blank; kseq drops a trailing '\r' only from a line longer than one byte (src/kseq.h:148)
    int cb = ne + 1, ce = nl[4 * r];
    if (ne >= e0) cb = ce = 0;
    else if (ce - cb > 1 && raw[ce - 1] == '\r') --ce;
    int nlen = ne - (l0 + 1);
    if (nlen > 2 && raw[l0 + 1 + nlen - 2] == '/' && raw[l0 + nlen] >= '0' && raw[l0 + nlen] <= '9') nlen -= 2;     // trim_readno
    const int read = r * stride + file;
    Span s; s.seq_beg = l1; s.seq_len = e1 - l1; s.qual_beg = l3; s.name_beg = l0 + 1; s.name_len = nlen; s.cmt_beg = cb; s.cmt_len = ce - cb; s._pad = 0;
    spans[read] = s;
    lens[read] = s.seq_len;
}

__device__ __forceinline__ uint8_t nt4(unsigned char c) {        // nst_nt4_table (src/bntseq.cpp:54-71)
    const unsigned char u = c & 0xDF;                            // upper case
    return u == 'A' ? 0 : u == 'C' ? 1 : u == 'G' ? 2 : u == 'T' ? 3 : (c == '-' ? 5 : 4);
}

// one warp per read: codes and qualities into the flat layout
__global__ void fastq_encode_kernel(const char *__restrict__ raw0, const char *__restrict__ raw1, const Span *__restrict__ spans,
                                    const int64_t *__restrict__ offs, int n_reads, int stride, uint8_t *codes, char *quals) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
    for (int rd = w; rd < n_reads; rd += nw) {
        const Span s = spans[rd];
        const char *raw = (stride == 2 && (rd & 1)) ? raw1 : raw0;
        const int64_t o = offs[rd];
        for (int i = lane; i < s.seq_len; i += 32) {
            codes[o + i] = nt4((unsigned char) raw[s.seq_beg + i]);
            quals[o + i] = raw[s.qual_beg + i];
        }
    }
}

// smart pairing (bm2_fastq_smart_pair).  key[i] = i where read i does not share its name with read i-1, else 0: after an inclusive max-scan,
// run[i] is the first read of the run of equal names that read i belongs to
__global__ void fastq_link_kernel(const char *__restrict__ raw, const Span *__restrict__ spans, int n, int *key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool same = false;
    if (i > 0) {
        const Span a = spans[i - 1], b = spans[i];
        same = a.name_len == b.name_len;
        for (int k = 0; same && k < a.name_len; ++k) same = raw[a.name_beg + k] == raw[b.name_beg + k];
    }
    key[i] = same ? 0 : i;
}

// bseq_classify's greedy left-to-right pairing: in a run of equal names starting at read s, read i pairs with read i-1 iff i - s is odd.
// pe[i] = 1 for the reads of a pair, else 0; se[i] = !pe[i]
__global__ void fastq_classify_kernel(const int *__restrict__ run, int n, uint8_t *se, uint8_t *pe) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool with_prev = ((i - run[i]) & 1) != 0;
    const bool with_next = i + 1 < n && ((i + 1 - run[i + 1]) & 1) != 0;
    const uint8_t p = with_prev || with_next;
    pe[i] = p; se[i] = !p;
}

__global__ void fastq_gather_lens_kernel(const int32_t *__restrict__ idx, const int64_t *__restrict__ offs, int n, int64_t *lens) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) lens[j] = offs[idx[j] + 1] - offs[idx[j]];
    if (j == n) lens[j] = 0;
}

// one warp per read of a set: its codes and qualities from the chunk's flat layout
__global__ void fastq_gather_kernel(const int32_t *__restrict__ idx, const int64_t *__restrict__ offs, const int64_t *__restrict__ soffs, int n,
                                    const uint8_t *__restrict__ codes, const char *__restrict__ quals, uint8_t *scodes, char *squals) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
    for (int j = w; j < n; j += nw) {
        const int64_t o = offs[idx[j]], so = soffs[j], len = soffs[j + 1] - so;
        for (int64_t k = lane; k < len; k += 32) { scodes[so + k] = codes[o + k]; squals[so + k] = quals[o + k]; }
    }
}

// slots of bm2_ctx::fq_d: the read batch (buffer b: F_RAW0 + b, F_NL0 + b); smart pairing (set s: F_SFLAG + s, F_SIDX + s, ...);
// bm2_seq_encode (buffer b: S_HP0 + b, S_REC0 + b)
enum FqBuf { F_RAW0, F_RAW1, F_NL0, F_NL1, F_SPANS, F_LENS, F_OFFS, F_CODES, F_QUALS, F_TMP, F_MISC,
             F_KEY, F_RUN, F_SFLAG, F_SCNT = F_SFLAG + 2, F_SIDX, F_SLEN = F_SIDX + 2, F_SOFF = F_SLEN + 2, F_SCODES = F_SOFF + 2,
             F_SQUALS = F_SCODES + 2,
             S_HP0 = F_SQUALS + 2, S_HP1, S_CAND, S_CANDU, S_INFO, S_JUMP, S_MARK, S_FLAG, S_REC0, S_REC1, S_QP, S_CNT, F_COUNT_ };
// the host buffers of one smart-pairing set
enum { SH_OFFS, SH_CODES, SH_QUALS, SH_NAMEBEG, SH_NAMELEN, SH_CMTBEG, SH_CMTLEN, SH_IDX, SH_COUNT_ };
// slots of bm2_ctx::fq_h: the read batch; smart pairing (set s: FH_SPLIT + SH_COUNT_ * s + k); bm2_seq_encode
enum FqHost { FH_OFFS, FH_CODES, FH_QUALS, FH_SPANS, FH_NAMEBEG, FH_NAMELEN, FH_CMTBEG, FH_CMTLEN, FH_SPLIT, FH_QP = FH_SPLIT + 2 * SH_COUNT_, FH_COUNT_ };
static_assert(F_COUNT_ == std::extent<decltype(bm2_ctx::fq_d)>::value, "bm2_ctx::fq_d: one buffer per slot");
static_assert(FH_COUNT_ == std::extent<decltype(bm2_ctx::fq_h)>::value, "bm2_ctx::fq_h: one buffer per slot");

}  // namespace

extern "C" int bm2_fastq_encode(bm2_ctx *ctx, const char *buf1, int64_t n1, const char *buf2, int64_t n2, bm2_fastq_batch *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || !buf1 || n1 < 0 || (buf2 && n2 < 0)) { if (ctx) bm2_set_error(ctx, "bm2_fastq_encode: bad arguments"); return 1; }
    if (n1 >= (1LL << 31) || (buf2 && n2 >= (1LL << 31))) { bm2_set_error(ctx, "bm2_fastq_encode: a chunk must stay below 2 GiB per buffer"); return 1; }
    ctx->fq_n_reads = ctx->fq_n_bufs = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int nbuf = buf2 ? 2 : 1;
    const char *hb[2] = { buf1, buf2 }; const int64_t hn[2] = { n1, buf2 ? n2 : 0 };
    int n_rec[2] = { 0, 0 };
    if (ctx->ensure(ctx->fq_d[F_MISC], 64)) return 1;
    int *d_misc = (int *) ctx->fq_d[F_MISC].p;            // [0], [1]: newline counts; [2]: error flag
    BM2_CUDA_OK(cudaMemsetAsync(d_misc, 0, 64, st));
    for (int b = 0; b < nbuf; ++b) {
        if (ctx->ensure(ctx->fq_d[F_RAW0 + b], (size_t) hn[b] + 16) || ctx->ensure(ctx->fq_d[F_NL0 + b], ((size_t) hn[b] / 2 + 16) * 4)) return 1;
        if (hn[b]) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_d[F_RAW0 + b].p, hb[b], (size_t) hn[b], cudaMemcpyHostToDevice, st));
        if (hn[b]) {
            size_t tmp = 0;
            cub::CountingInputIterator<int> it(0);
            IsNewline pred = { (const char *) ctx->fq_d[F_RAW0 + b].p };
            {   // the position array holds n / 2 + 16 entries (a four-line record has at most one newline per two bytes): count first,
                // so that malformed input is an error and not a write past the array
                NewlineAsInt conv = { (const char *) ctx->fq_d[F_RAW0 + b].p };
                cub::TransformInputIterator<int, NewlineAsInt, cub::CountingInputIterator<int>> cnt_it(it, conv);
                cub::DeviceReduce::Sum(nullptr, tmp, cnt_it, d_misc + 4 + b, (int) hn[b], st);
                if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
                BM2_CUDA_OK(cub::DeviceReduce::Sum(ctx->fq_d[F_TMP].p, tmp, cnt_it, d_misc + 4 + b, (int) hn[b], st));
                int h_n = 0;
                BM2_CUDA_OK(cudaMemcpyAsync(&h_n, d_misc + 4 + b, 4, cudaMemcpyDeviceToHost, st));
                BM2_CUDA_OK(cudaStreamSynchronize(st));
                if ((int64_t) h_n > hn[b] / 2 + 8) { bm2_set_error(ctx, "bm2_fastq_encode: too many line ends for FASTQ records"); return 2; }
                tmp = 0;
            }
            cub::DeviceSelect::If(nullptr, tmp, it, (int32_t *) ctx->fq_d[F_NL0 + b].p, d_misc + b, (int) hn[b], pred, st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::If(ctx->fq_d[F_TMP].p, tmp, it, (int32_t *) ctx->fq_d[F_NL0 + b].p, d_misc + b, (int) hn[b], pred, st));
        }
    }
    int h_cnt[2] = { 0, 0 };
    BM2_CUDA_OK(cudaMemcpyAsync(h_cnt, d_misc, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    for (int b = 0; b < nbuf; ++b) {
        int lines = h_cnt[b];
        if (hn[b] > 0 && hb[b][hn[b] - 1] != '\n') {      // last line without a newline: a virtual one at the end of the buffer
            const int32_t endpos = (int32_t) hn[b];
            BM2_CUDA_OK(cudaMemcpyAsync((int32_t *) ctx->fq_d[F_NL0 + b].p + lines, &endpos, 4, cudaMemcpyHostToDevice, st));
            BM2_CUDA_OK(cudaStreamSynchronize(st));
            ++lines;
        }
        if (lines % 4) { bm2_set_error(ctx, "bm2_fastq_encode: the number of lines is not a multiple of four (wrapped or truncated records)"); return 2; }
        n_rec[b] = lines / 4;
    }
    if (nbuf == 2 && n_rec[0] != n_rec[1]) { bm2_set_error(ctx, "bm2_fastq_encode: the two files hold different numbers of records"); return 2; }
    const int n_reads = n_rec[0] * nbuf;
    out->n_reads = n_reads;
    if (ctx->ensure(ctx->fq_d[F_SPANS], (size_t) (n_reads + 1) * sizeof(Span)) || ctx->ensure(ctx->fq_d[F_LENS], (size_t) (n_reads + 2) * 8) ||
        ctx->ensure(ctx->fq_d[F_OFFS], (size_t) (n_reads + 2) * 8)) return 1;
    Span *d_spans = (Span *) ctx->fq_d[F_SPANS].p; int64_t *d_lens = (int64_t *) ctx->fq_d[F_LENS].p, *d_offs = (int64_t *) ctx->fq_d[F_OFFS].p;
    BM2_CUDA_OK(cudaMemsetAsync(d_lens + n_reads, 0, 8, st));
    for (int b = 0; b < nbuf && n_rec[b] > 0; ++b)
        fastq_spans_kernel<<<(n_rec[b] + 255) / 256, 256, 0, st>>>((const char *) ctx->fq_d[F_RAW0 + b].p, (const int32_t *) ctx->fq_d[F_NL0 + b].p, n_rec[b], b, nbuf,
                                                                      d_spans, d_lens, d_misc + 2);
    {
        size_t tmp = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_lens, d_offs, n_reads + 1, st);
        if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->fq_d[F_TMP].p, tmp, d_lens, d_offs, n_reads + 1, st));
    }
    int64_t total = 0; int h_err = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&total, d_offs + n_reads, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&h_err, d_misc + 2, 4, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    if (h_err) { bm2_set_error(ctx, "bm2_fastq_encode: malformed record " + std::to_string(h_err - 1) + " (expected @name / sequence / + / qualities of the same length)"); return 2; }
    if (ctx->ensure(ctx->fq_d[F_CODES], (size_t) total + 16) || ctx->ensure(ctx->fq_d[F_QUALS], (size_t) total + 16)) return 1;
    if (n_reads > 0) {
        int blocks = (n_reads + 7) / 8; if (blocks > ctx->n_sm * 16) blocks = ctx->n_sm * 16;
        fastq_encode_kernel<<<blocks, 256, 0, st>>>((const char *) ctx->fq_d[F_RAW0].p, (const char *) ctx->fq_d[F_RAW1].p, d_spans, d_offs, n_reads, nbuf,
                                                     (uint8_t *) ctx->fq_d[F_CODES].p, (char *) ctx->fq_d[F_QUALS].p);
    }
    // host copies: offsets, codes, qualities (the SAM stage and the formatter read them), name positions
    if (ctx->ensure_host(ctx->fq_h[FH_OFFS], (size_t) (n_reads + 1) * 8) || ctx->ensure_host(ctx->fq_h[FH_CODES], (size_t) total + 16) ||
        ctx->ensure_host(ctx->fq_h[FH_QUALS], (size_t) total + 16) || ctx->ensure_host(ctx->fq_h[FH_SPANS], (size_t) (n_reads + 1) * sizeof(Span)) ||
        ctx->ensure_host(ctx->fq_h[FH_NAMEBEG], (size_t) (n_reads + 1) * 8) || ctx->ensure_host(ctx->fq_h[FH_NAMELEN], (size_t) (n_reads + 1) * 4)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_OFFS].p, d_offs, (size_t) (n_reads + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (total) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_CODES].p, ctx->fq_d[F_CODES].p, (size_t) total, cudaMemcpyDeviceToHost, st));
    if (total) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_QUALS].p, ctx->fq_d[F_QUALS].p, (size_t) total, cudaMemcpyDeviceToHost, st));
    if (n_reads) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_SPANS].p, d_spans, (size_t) n_reads * sizeof(Span), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaGetLastError());
    const Span *hs = (const Span *) ctx->fq_h[FH_SPANS].p;
    int64_t *nb = (int64_t *) ctx->fq_h[FH_NAMEBEG].p; int32_t *nlv = (int32_t *) ctx->fq_h[FH_NAMELEN].p;
    for (int r = 0; r < n_reads; ++r) { nb[r] = hs[r].name_beg; nlv[r] = hs[r].name_len; }
    out->d_codes = (const uint8_t *) ctx->fq_d[F_CODES].p; out->d_offsets = d_offs;
    out->codes = (const uint8_t *) ctx->fq_h[FH_CODES].p; out->offsets = (const int64_t *) ctx->fq_h[FH_OFFS].p;
    out->quals = (const char *) ctx->fq_h[FH_QUALS].p; out->name_beg = nb; out->name_len = nlv;
    ctx->fq_n_reads = n_reads; ctx->fq_n_bufs = nbuf;
    return 0;
}

extern "C" int bm2_fastq_comments(bm2_ctx *ctx, const int64_t **beg, const int32_t **len) {
    if (!ctx || !beg || !len) { if (ctx) bm2_set_error(ctx, "bm2_fastq_comments: bad arguments"); return 1; }
    const int n = ctx->fq_n_reads;
    if (ctx->ensure_host(ctx->fq_h[FH_CMTBEG], (size_t) (n + 1) * 8) || ctx->ensure_host(ctx->fq_h[FH_CMTLEN], (size_t) (n + 1) * 4)) return 1;
    const Span *hs = (const Span *) ctx->fq_h[FH_SPANS].p;
    int64_t *cb = (int64_t *) ctx->fq_h[FH_CMTBEG].p; int32_t *cl = (int32_t *) ctx->fq_h[FH_CMTLEN].p;
    for (int r = 0; r < n; ++r) { cb[r] = hs[r].cmt_beg; cl[r] = hs[r].cmt_len; }
    *beg = cb; *len = cl;
    return 0;
}

extern "C" int bm2_fastq_smart_pair(bm2_ctx *ctx, bm2_fastq_split *out) {
    if (!ctx || !out) { if (ctx) bm2_set_error(ctx, "bm2_fastq_smart_pair: bad arguments"); return 1; }
    if (ctx->fq_n_bufs != 1) { bm2_set_error(ctx, "bm2_fastq_smart_pair: the last bm2_fastq_encode call was not single-end"); return 1; }
    bm2_ctx *ctx_for_error = ctx;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int n = ctx->fq_n_reads;
    memset(out, 0, sizeof *out);
    if (ctx->ensure(ctx->fq_d[F_KEY], (size_t) (n + 1) * 4) || ctx->ensure(ctx->fq_d[F_RUN], (size_t) (n + 1) * 4) || ctx->ensure(ctx->fq_d[F_SCNT], 16)) return 1;
    for (int s = 0; s < 2; ++s)
        if (ctx->ensure(ctx->fq_d[F_SFLAG + s], (size_t) n + 16) || ctx->ensure(ctx->fq_d[F_SIDX + s], (size_t) (n + 1) * 4) ||
            ctx->ensure(ctx->fq_d[F_SLEN + s], (size_t) (n + 2) * 8) || ctx->ensure(ctx->fq_d[F_SOFF + s], (size_t) (n + 2) * 8)) return 1;
    const Span *d_spans = (const Span *) ctx->fq_d[F_SPANS].p;
    const int64_t *d_offs = (const int64_t *) ctx->fq_d[F_OFFS].p;
    int *d_key = (int *) ctx->fq_d[F_KEY].p, *d_run = (int *) ctx->fq_d[F_RUN].p, *d_cnt = (int *) ctx->fq_d[F_SCNT].p;
    int h_cnt[2] = { 0, 0 };
    if (n > 0) {
        const int blocks = (n + 255) / 256;
        fastq_link_kernel<<<blocks, 256, 0, st>>>((const char *) ctx->fq_d[F_RAW0].p, d_spans, n, d_key);
        size_t tmp = 0;
        cub::DeviceScan::InclusiveScan(nullptr, tmp, d_key, d_run, cub::Max(), n, st);
        if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::InclusiveScan(ctx->fq_d[F_TMP].p, tmp, d_key, d_run, cub::Max(), n, st));
        fastq_classify_kernel<<<blocks, 256, 0, st>>>(d_run, n, (uint8_t *) ctx->fq_d[F_SFLAG].p, (uint8_t *) ctx->fq_d[F_SFLAG + 1].p);
        cub::CountingInputIterator<int32_t> it(0);
        for (int s = 0; s < 2; ++s) {       // stable compaction: the reads of each set in file order
            tmp = 0;
            cub::DeviceSelect::Flagged(nullptr, tmp, it, (const uint8_t *) ctx->fq_d[F_SFLAG + s].p, (int32_t *) ctx->fq_d[F_SIDX + s].p, d_cnt + s, n, st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::Flagged(ctx->fq_d[F_TMP].p, tmp, it, (const uint8_t *) ctx->fq_d[F_SFLAG + s].p, (int32_t *) ctx->fq_d[F_SIDX + s].p,
                                                   d_cnt + s, n, st));
        }
        BM2_CUDA_OK(cudaMemcpyAsync(h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
    }
    const Span *hs = (const Span *) ctx->fq_h[FH_SPANS].p;
    for (int s = 0; s < 2; ++s) {
        const int m = h_cnt[s];
        const int32_t *d_idx = (const int32_t *) ctx->fq_d[F_SIDX + s].p;
        int64_t *d_len = (int64_t *) ctx->fq_d[F_SLEN + s].p, *d_soff = (int64_t *) ctx->fq_d[F_SOFF + s].p;
        fastq_gather_lens_kernel<<<(m + 1 + 255) / 256, 256, 0, st>>>(d_idx, d_offs, m, d_len);
        size_t tmp = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_len, d_soff, m + 1, st);
        if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->fq_d[F_TMP].p, tmp, d_len, d_soff, m + 1, st));
        int64_t total = 0;
        BM2_CUDA_OK(cudaMemcpyAsync(&total, d_soff + m, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        if (ctx->ensure(ctx->fq_d[F_SCODES + s], (size_t) total + 16) || ctx->ensure(ctx->fq_d[F_SQUALS + s], (size_t) total + 16)) return 1;
        if (m > 0) {
            int blocks = (m + 7) / 8; if (blocks > ctx->n_sm * 16) blocks = ctx->n_sm * 16;
            fastq_gather_kernel<<<blocks, 256, 0, st>>>(d_idx, d_offs, d_soff, m, (const uint8_t *) ctx->fq_d[F_CODES].p, (const char *) ctx->fq_d[F_QUALS].p,
                                                        (uint8_t *) ctx->fq_d[F_SCODES + s].p, (char *) ctx->fq_d[F_SQUALS + s].p);
        }
        HostBuf *h = ctx->fq_h + FH_SPLIT + SH_COUNT_ * s;
        if (ctx->ensure_host(h[SH_OFFS], (size_t) (m + 1) * 8) || ctx->ensure_host(h[SH_CODES], (size_t) total + 16) ||
            ctx->ensure_host(h[SH_QUALS], (size_t) total + 16) || ctx->ensure_host(h[SH_NAMEBEG], (size_t) (m + 1) * 8) ||
            ctx->ensure_host(h[SH_NAMELEN], (size_t) (m + 1) * 4) || ctx->ensure_host(h[SH_CMTBEG], (size_t) (m + 1) * 8) ||
            ctx->ensure_host(h[SH_CMTLEN], (size_t) (m + 1) * 4) || ctx->ensure_host(h[SH_IDX], (size_t) (m + 1) * 4)) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(h[SH_OFFS].p, d_soff, (size_t) (m + 1) * 8, cudaMemcpyDeviceToHost, st));
        if (total) BM2_CUDA_OK(cudaMemcpyAsync(h[SH_CODES].p, ctx->fq_d[F_SCODES + s].p, (size_t) total, cudaMemcpyDeviceToHost, st));
        if (total) BM2_CUDA_OK(cudaMemcpyAsync(h[SH_QUALS].p, ctx->fq_d[F_SQUALS + s].p, (size_t) total, cudaMemcpyDeviceToHost, st));
        if (m) BM2_CUDA_OK(cudaMemcpyAsync(h[SH_IDX].p, d_idx, (size_t) m * 4, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        BM2_CUDA_OK(cudaGetLastError());
        const int32_t *idx = (const int32_t *) h[SH_IDX].p;
        int64_t *nb = (int64_t *) h[SH_NAMEBEG].p, *cb = (int64_t *) h[SH_CMTBEG].p;
        int32_t *nlv = (int32_t *) h[SH_NAMELEN].p, *cl = (int32_t *) h[SH_CMTLEN].p;
        for (int j = 0; j < m; ++j) { const Span &sp = hs[idx[j]]; nb[j] = sp.name_beg; nlv[j] = sp.name_len; cb[j] = sp.cmt_beg; cl[j] = sp.cmt_len; }
        bm2_fastq_batch &b = out->set[s];
        b.n_reads = m;
        b.d_codes = (const uint8_t *) ctx->fq_d[F_SCODES + s].p; b.d_offsets = d_soff;
        b.codes = (const uint8_t *) h[SH_CODES].p; b.offsets = (const int64_t *) h[SH_OFFS].p; b.quals = (const char *) h[SH_QUALS].p;
        b.name_beg = nb; b.name_len = nlv;
        out->comment_beg[s] = cb; out->comment_len[s] = cl; out->read_index[s] = idx;
    }
    return 0;
}

// ---- bm2_seq_encode: every input kseq reads (FASTA, wrapped FASTQ, mixed, junk, CRLF), parsed on the GPU by seq_grammar.cuh --------------
// Per buffer: the positions of '\n' and of '>' / '@' by stream compaction; for every line start the first '>' / '@' at or after it - every
// record's header character is one of these candidates (after a FASTQ record kseq skips to the next such byte, after a FASTA record the
// header is the first byte of a line); one thread per candidate runs seq_record, whose next header is again a candidate, so next() is a
// forest pointing right; the records are the chain from the first candidate, marked by pointer doubling (log K jump tables, marks pushed
// from the top level down: the nodes 2^t steps apart are those 2^(t+1) apart plus one jump of 2^t from each); then one warp per record
// walks it again and writes its codes and qualities where the sink puts them.
// Cost of the candidate walks: one walk per line start whose first '>' / '@' differs from the previous line's - about one per record for
// four-line FASTQ (plus one per quality line holding a '>' or '@'), one per record for FASTA (its sequence lines share the candidate),
// and up to one per quality line for wrapped FASTQ; a walk is as long as the record it parses from its candidate.
// sm_90a (ptxas -v), no spills in any of them: seq_gather_kernel 40 registers, seq_walk_kernel 27, seq_span_kernel 26, seq_cand_kernel 22,
// seq_jump_kernel 12, seq_flag_kernel 12, seq_mark_kernel 8.
namespace {

struct IsHeaderChar {
    const char *raw;
    __device__ __forceinline__ bool operator()(const int &i) const { return raw[i] == '>' || raw[i] == '@'; }
};
struct HeaderCharAsInt {
    const char *raw;
    __device__ __forceinline__ int operator()(const int &i) const { return raw[i] == '>' || raw[i] == '@'; }
};

// what a candidate's walk leaves for the record table
struct SeqCand { int32_t h, l_seq, name_beg, name_len, cmt_beg, cmt_len; int8_t status, has_qual, _p[2]; };

// line k (0..n_nl) starts at 0 or nl[k-1] + 1: its first header character at or after the start
__global__ void seq_cand_kernel(SeqTableSrc s, int32_t *cand) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > s.n_nl) return;
    cand[k] = (int32_t) s.hdr(k == 0 ? 0 : (int64_t) s.nl[k - 1] + 1);
}

// one thread per candidate: its record and next(); nxt[K] = K is the end of every chain
__global__ void seq_walk_kernel(SeqTableSrc s, const int32_t *__restrict__ cand, int K, int32_t *nxt, SeqCand *info) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > K) return;
    if (i == K) { nxt[K] = K; return; }
    s.k = 0;
    const SeqRec r = seq_record(s, cand[i], SeqNullSink());
    int j = K;
    if (r.status == SEQ_OK && r.next < s.n) {
        int lo = i + 1, hi = K;
        while (lo < hi) { const int m = (lo + hi) >> 1; if (cand[m] < r.next) lo = m + 1; else hi = m; }
        j = lo;
    }
    nxt[i] = j;
    SeqCand c; c.h = cand[i]; c.l_seq = r.l_seq; c.name_beg = (int32_t) r.name_beg; c.name_len = r.name_len; c.cmt_beg = (int32_t) r.cmt_beg;
    c.cmt_len = r.cmt_len; c.status = r.status; c.has_qual = r.l_qual > 0; c._p[0] = c._p[1] = 0;
    info[i] = c;
}

__global__ void seq_jump_kernel(const int32_t *__restrict__ a, int K, int32_t *b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= K) b[i] = a[a[i]];
}

// level t: every marked node marks its 2^t-th successor (in place: a node marked during this pass only marks nodes of the level above)
__global__ void seq_mark_kernel(const int32_t *__restrict__ jump, int K, uint8_t *mark) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= K && mark[i]) mark[jump[i]] = 1;
}

__global__ void seq_flag_kernel(const uint8_t *__restrict__ mark, const SeqCand *__restrict__ info, int K, uint8_t *flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < K) flag[i] = mark[i] && info[i].status != SEQ_NONE;
}

// records of buffer `file` -> spans, lengths, qualities present
__global__ void seq_span_kernel(const SeqCand *__restrict__ rec, int n_rec, int file, int stride, Span *spans, int64_t *lens, uint8_t *qp) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rec) return;
    const SeqCand c = rec[r];
    const int read = r * stride + file;
    Span s; s.seq_beg = c.h; s.seq_len = c.l_seq; s.qual_beg = 0; s.name_beg = c.name_beg; s.name_len = c.name_len; s.cmt_beg = c.cmt_beg;
    s.cmt_len = c.cmt_len; s._pad = 0;
    spans[read] = s;
    lens[read] = c.l_seq;
    qp[read] = (uint8_t) c.has_qual;
}

struct SeqWarpSink {            // every lane runs the same walk; the lanes split each line's bytes
    uint8_t *codes; char *quals; int lane; const char *raw;
    __device__ void seq(int64_t b, int64_t k, int64_t at) const { for (int64_t i = lane; i < k; i += 32) codes[at + i] = nt4((unsigned char) raw[b + i]); }
    __device__ void qual(int64_t b, int64_t k, int64_t at) const { for (int64_t i = lane; i < k; i += 32) quals[at + i] = raw[b + i]; }
};

// one warp per read: the record walked again from its header, its kept bytes written as codes and qualities
__global__ void seq_gather_kernel(SeqTableSrc s0, SeqTableSrc s1, const Span *__restrict__ spans, const int64_t *__restrict__ offs, int n_reads, int stride,
                                  uint8_t *codes, char *quals) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
    for (int rd = w; rd < n_reads; rd += nw) {
        SeqTableSrc s = (stride == 2 && (rd & 1)) ? s1 : s0;
        s.k = 0;
        const int64_t o = offs[rd];
        SeqWarpSink sink = { codes + o, quals + o, lane, s.raw };
        seq_record(s, spans[rd].seq_beg, sink);
    }
}

}  // namespace

extern "C" int bm2_seq_encode(bm2_ctx *ctx, const char *buf1, int64_t n1, const char *buf2, int64_t n2, bm2_fastq_batch *out, const uint8_t **qual_present) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || !buf1 || n1 < 0 || (buf2 && n2 < 0)) { if (ctx) bm2_set_error(ctx, "bm2_seq_encode: bad arguments"); return 1; }
    if (n1 >= (1LL << 31) - 16 || (buf2 && n2 >= (1LL << 31) - 16)) { bm2_set_error(ctx, "bm2_seq_encode: a chunk must stay below 2 GiB per buffer"); return 1; }
    ctx->fq_n_reads = ctx->fq_n_bufs = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int nbuf = buf2 ? 2 : 1;
    const char *hb[2] = { buf1, buf2 }; const int64_t hn[2] = { n1, buf2 ? n2 : 0 };
    int n_rec[2] = { 0, 0 };
    SeqTableSrc src[2] = {};
    int bad[2] = { -1, -1 };                                       // per buffer: index of the malformed record, -1: none
    if (ctx->ensure(ctx->fq_d[S_CNT], 64)) return 1;
    int *d_cnt = (int *) ctx->fq_d[S_CNT].p;
    // compaction of the positions i < n where pred(raw[i]) into slot `dst` (counted first to size it)
    auto positions = [&](int b, int slot, bool newline, int *count) -> int {
        const char *d_raw = (const char *) ctx->fq_d[F_RAW0 + b].p;
        cub::CountingInputIterator<int> it(0);
        size_t tmp = 0;
        int h_n = 0;
        if (newline) {
            cub::TransformInputIterator<int, NewlineAsInt, cub::CountingInputIterator<int>> cnt_it(it, NewlineAsInt{ d_raw });
            cub::DeviceReduce::Sum(nullptr, tmp, cnt_it, d_cnt, (int) hn[b], st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceReduce::Sum(ctx->fq_d[F_TMP].p, tmp, cnt_it, d_cnt, (int) hn[b], st));
        } else {
            cub::TransformInputIterator<int, HeaderCharAsInt, cub::CountingInputIterator<int>> cnt_it(it, HeaderCharAsInt{ d_raw });
            cub::DeviceReduce::Sum(nullptr, tmp, cnt_it, d_cnt, (int) hn[b], st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceReduce::Sum(ctx->fq_d[F_TMP].p, tmp, cnt_it, d_cnt, (int) hn[b], st));
        }
        BM2_CUDA_OK(cudaMemcpyAsync(&h_n, d_cnt, 4, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        if (ctx->ensure(ctx->fq_d[slot], ((size_t) h_n + 16) * 4)) return 1;
        tmp = 0;
        if (newline) {
            IsNewline pred = { d_raw };
            cub::DeviceSelect::If(nullptr, tmp, it, (int32_t *) ctx->fq_d[slot].p, d_cnt, (int) hn[b], pred, st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::If(ctx->fq_d[F_TMP].p, tmp, it, (int32_t *) ctx->fq_d[slot].p, d_cnt, (int) hn[b], pred, st));
        } else {
            IsHeaderChar pred = { d_raw };
            cub::DeviceSelect::If(nullptr, tmp, it, (int32_t *) ctx->fq_d[slot].p, d_cnt, (int) hn[b], pred, st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::If(ctx->fq_d[F_TMP].p, tmp, it, (int32_t *) ctx->fq_d[slot].p, d_cnt, (int) hn[b], pred, st));
        }
        *count = h_n;
        return 0;
    };
    for (int b = 0; b < nbuf; ++b) {
        if (ctx->ensure(ctx->fq_d[F_RAW0 + b], (size_t) hn[b] + 16)) return 1;
        if (hn[b]) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_d[F_RAW0 + b].p, hb[b], (size_t) hn[b], cudaMemcpyHostToDevice, st));
        int n_nl = 0, n_hp = 0;
        if (hn[b] && (positions(b, F_NL0 + b, true, &n_nl) || positions(b, S_HP0 + b, false, &n_hp))) return 1;
        if (!hn[b] && (ctx->ensure(ctx->fq_d[F_NL0 + b], 64) || ctx->ensure(ctx->fq_d[S_HP0 + b], 64))) return 1;
        SeqTableSrc &s = src[b];
        s.raw = (const char *) ctx->fq_d[F_RAW0 + b].p; s.n = hn[b]; s.nl = (const int32_t *) ctx->fq_d[F_NL0 + b].p; s.n_nl = n_nl;
        s.hp = (const int32_t *) ctx->fq_d[S_HP0 + b].p; s.n_hp = n_hp; s.k = 0;
        if (n_hp == 0) { n_rec[b] = 0; if (ctx->ensure(ctx->fq_d[S_REC0 + b], 64)) return 1; continue; }
        // candidates: the first header character at or after each line start, deduplicated (non-decreasing in the line index)
        const int n_ls = n_nl + 1;
        if (ctx->ensure(ctx->fq_d[S_CAND], (size_t) (n_ls + 16) * 4) || ctx->ensure(ctx->fq_d[S_CANDU], (size_t) (n_ls + 16) * 4)) return 1;
        int32_t *d_cand = (int32_t *) ctx->fq_d[S_CAND].p, *d_cu = (int32_t *) ctx->fq_d[S_CANDU].p;
        seq_cand_kernel<<<(n_ls + 255) / 256, 256, 0, st>>>(s, d_cand);
        {
            size_t tmp = 0;
            cub::DeviceSelect::Unique(nullptr, tmp, d_cand, d_cu, d_cnt, n_ls, st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::Unique(ctx->fq_d[F_TMP].p, tmp, d_cand, d_cu, d_cnt, n_ls, st));
        }
        int K = 0;
        BM2_CUDA_OK(cudaMemcpyAsync(&K, d_cnt, 4, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        int32_t last = 0;
        BM2_CUDA_OK(cudaMemcpyAsync(&last, d_cu + K - 1, 4, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        if (last >= hn[b]) --K;                         // "no header character after this line"
        // next() of every candidate, then the jump tables J_t = next^(2^t), t < T with 2^T > K
        int T = 1; while ((1LL << T) <= K) ++T;
        if (ctx->ensure(ctx->fq_d[S_INFO], (size_t) (K + 1) * sizeof(SeqCand)) || ctx->ensure(ctx->fq_d[S_JUMP], (size_t) T * (K + 1) * 4) ||
            ctx->ensure(ctx->fq_d[S_MARK], (size_t) K + 16) || ctx->ensure(ctx->fq_d[S_FLAG], (size_t) K + 16) ||
            ctx->ensure(ctx->fq_d[S_REC0 + b], (size_t) (K + 1) * sizeof(SeqCand))) return 1;
        int32_t *d_jump = (int32_t *) ctx->fq_d[S_JUMP].p;
        SeqCand *d_info = (SeqCand *) ctx->fq_d[S_INFO].p;
        uint8_t *d_mark = (uint8_t *) ctx->fq_d[S_MARK].p, *d_flag = (uint8_t *) ctx->fq_d[S_FLAG].p;
        const int gK = (K + 1 + 255) / 256;
        seq_walk_kernel<<<gK, 256, 0, st>>>(s, d_cu, K, d_jump, d_info);
        for (int t = 1; t < T; ++t) seq_jump_kernel<<<gK, 256, 0, st>>>(d_jump + (size_t) (t - 1) * (K + 1), K, d_jump + (size_t) t * (K + 1));
        BM2_CUDA_OK(cudaMemsetAsync(d_mark, 0, (size_t) K + 1, st));
        BM2_CUDA_OK(cudaMemsetAsync(d_mark, 1, 1, st));
        for (int t = T - 1; t >= 0; --t) seq_mark_kernel<<<gK, 256, 0, st>>>(d_jump + (size_t) t * (K + 1), K, d_mark);
        seq_flag_kernel<<<gK, 256, 0, st>>>(d_mark, d_info, K, d_flag);
        {
            size_t tmp = 0;
            cub::DeviceSelect::Flagged(nullptr, tmp, d_info, d_flag, (SeqCand *) ctx->fq_d[S_REC0 + b].p, d_cnt, K, st);
            if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::Flagged(ctx->fq_d[F_TMP].p, tmp, d_info, d_flag, (SeqCand *) ctx->fq_d[S_REC0 + b].p, d_cnt, K, st));
        }
        BM2_CUDA_OK(cudaMemcpyAsync(&n_rec[b], d_cnt, 4, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        // a malformed record ends its chain (its next() is K), so only the last record of the buffer can be one
        if (n_rec[b] > 0) {
            SeqCand lastc;
            BM2_CUDA_OK(cudaMemcpyAsync(&lastc, (const SeqCand *) ctx->fq_d[S_REC0 + b].p + n_rec[b] - 1, sizeof lastc, cudaMemcpyDeviceToHost, st));
            BM2_CUDA_OK(cudaStreamSynchronize(st));
            if (lastc.status == SEQ_BAD) bad[b] = n_rec[b] - 1;
        }
    }
    for (int b = 0; b < nbuf; ++b)                                // before the record counts: a malformed record also shortens its file
        if (bad[b] >= 0) {
            bm2_set_error(ctx, "bm2_seq_encode: malformed record " + std::to_string(bad[b]) + (nbuf == 2 ? (b ? " of the 2nd file" : " of the 1st file") : "") +
                               " (a '+' line without qualities, or qualities of another length than the sequence)");
            return 2;
        }
    if (nbuf == 2 && n_rec[0] != n_rec[1]) { bm2_set_error(ctx, "bm2_seq_encode: the two files hold different numbers of records"); return 2; }
    const int n_reads = n_rec[0] * nbuf;
    out->n_reads = n_reads;
    if (ctx->ensure(ctx->fq_d[F_SPANS], (size_t) (n_reads + 1) * sizeof(Span)) || ctx->ensure(ctx->fq_d[F_LENS], (size_t) (n_reads + 2) * 8) ||
        ctx->ensure(ctx->fq_d[F_OFFS], (size_t) (n_reads + 2) * 8) || ctx->ensure(ctx->fq_d[S_QP], (size_t) n_reads + 16)) return 1;
    Span *d_spans = (Span *) ctx->fq_d[F_SPANS].p; int64_t *d_lens = (int64_t *) ctx->fq_d[F_LENS].p, *d_offs = (int64_t *) ctx->fq_d[F_OFFS].p;
    uint8_t *d_qp = (uint8_t *) ctx->fq_d[S_QP].p;
    BM2_CUDA_OK(cudaMemsetAsync(d_lens + n_reads, 0, 8, st));
    for (int b = 0; b < nbuf && n_rec[b] > 0; ++b)
        seq_span_kernel<<<(n_rec[b] + 255) / 256, 256, 0, st>>>((const SeqCand *) ctx->fq_d[S_REC0 + b].p, n_rec[b], b, nbuf, d_spans, d_lens, d_qp);
    {
        size_t tmp = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_lens, d_offs, n_reads + 1, st);
        if (ctx->ensure(ctx->fq_d[F_TMP], tmp)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->fq_d[F_TMP].p, tmp, d_lens, d_offs, n_reads + 1, st));
    }
    int64_t total = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&total, d_offs + n_reads, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    if (ctx->ensure(ctx->fq_d[F_CODES], (size_t) total + 16) || ctx->ensure(ctx->fq_d[F_QUALS], (size_t) total + 16)) return 1;
    if (n_reads > 0) {
        int blocks = (n_reads + 7) / 8; if (blocks > ctx->n_sm * 16) blocks = ctx->n_sm * 16;
        seq_gather_kernel<<<blocks, 256, 0, st>>>(src[0], nbuf == 2 ? src[1] : src[0], d_spans, d_offs, n_reads, nbuf, (uint8_t *) ctx->fq_d[F_CODES].p,
                                                  (char *) ctx->fq_d[F_QUALS].p);
    }
    if (ctx->ensure_host(ctx->fq_h[FH_OFFS], (size_t) (n_reads + 1) * 8) || ctx->ensure_host(ctx->fq_h[FH_CODES], (size_t) total + 16) ||
        ctx->ensure_host(ctx->fq_h[FH_QUALS], (size_t) total + 16) || ctx->ensure_host(ctx->fq_h[FH_SPANS], (size_t) (n_reads + 1) * sizeof(Span)) ||
        ctx->ensure_host(ctx->fq_h[FH_NAMEBEG], (size_t) (n_reads + 1) * 8) || ctx->ensure_host(ctx->fq_h[FH_NAMELEN], (size_t) (n_reads + 1) * 4) ||
        ctx->ensure_host(ctx->fq_h[FH_QP], (size_t) n_reads + 16)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_OFFS].p, d_offs, (size_t) (n_reads + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (total) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_CODES].p, ctx->fq_d[F_CODES].p, (size_t) total, cudaMemcpyDeviceToHost, st));
    if (total) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_QUALS].p, ctx->fq_d[F_QUALS].p, (size_t) total, cudaMemcpyDeviceToHost, st));
    if (n_reads) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_SPANS].p, d_spans, (size_t) n_reads * sizeof(Span), cudaMemcpyDeviceToHost, st));
    if (n_reads) BM2_CUDA_OK(cudaMemcpyAsync(ctx->fq_h[FH_QP].p, d_qp, (size_t) n_reads, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaGetLastError());
    const Span *hs = (const Span *) ctx->fq_h[FH_SPANS].p;
    int64_t *nb = (int64_t *) ctx->fq_h[FH_NAMEBEG].p; int32_t *nlv = (int32_t *) ctx->fq_h[FH_NAMELEN].p;
    for (int r = 0; r < n_reads; ++r) { nb[r] = hs[r].name_beg; nlv[r] = hs[r].name_len; }
    out->d_codes = (const uint8_t *) ctx->fq_d[F_CODES].p; out->d_offsets = d_offs;
    out->codes = (const uint8_t *) ctx->fq_h[FH_CODES].p; out->offsets = (const int64_t *) ctx->fq_h[FH_OFFS].p;
    out->quals = (const char *) ctx->fq_h[FH_QUALS].p; out->name_beg = nb; out->name_len = nlv;
    if (qual_present) *qual_present = (const uint8_t *) ctx->fq_h[FH_QP].p;
    ctx->fq_n_reads = n_reads; ctx->fq_n_bufs = nbuf;
    return 0;
}

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

enum FqBuf { F_RAW0 = 100, F_RAW1, F_NL0, F_NL1, F_SPANS, F_LENS, F_OFFS, F_CODES, F_QUALS, F_TMP, F_MISC };     // slots of bm2_ctx::d[]
enum FqHost { FH_OFFS = 24, FH_CODES, FH_QUALS, FH_SPANS, FH_NAMEBEG, FH_NAMELEN, FH_CMTBEG, FH_CMTLEN };
// smart pairing: device slots 112-126; per set s: F_SIDX + s, F_SLEN + s, ... and host slots FH_SPLIT + 8 s + k
enum FqSplit { F_KEY = 112, F_RUN, F_SFLAG, F_SCNT = F_SFLAG + 2, F_SIDX, F_SLEN = F_SIDX + 2, F_SOFF = F_SLEN + 2, F_SCODES = F_SOFF + 2,
               F_SQUALS = F_SCODES + 2 };
enum FqSplitHost { FH_SPLIT = 32 };
enum { SH_OFFS, SH_CODES, SH_QUALS, SH_NAMEBEG, SH_NAMELEN, SH_CMTBEG, SH_CMTLEN, SH_IDX };
static_assert(F_SQUALS + 1 < 128, "bm2_ctx::d[] slots");

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
    if (ctx->ensure(ctx->d[F_MISC], 64)) return 1;
    int *d_misc = (int *) ctx->d[F_MISC].p;            // [0], [1]: newline counts; [2]: error flag
    BM2_CUDA_OK(cudaMemsetAsync(d_misc, 0, 64, st));
    for (int b = 0; b < nbuf; ++b) {
        if (ctx->ensure(ctx->d[F_RAW0 + b], (size_t) hn[b] + 16) || ctx->ensure(ctx->d[F_NL0 + b], ((size_t) hn[b] / 2 + 16) * 4)) return 1;
        if (hn[b]) BM2_CUDA_OK(cudaMemcpyAsync(ctx->d[F_RAW0 + b].p, hb[b], (size_t) hn[b], cudaMemcpyHostToDevice, st));
        if (hn[b]) {
            size_t tmp = 0;
            cub::CountingInputIterator<int> it(0);
            IsNewline pred = { (const char *) ctx->d[F_RAW0 + b].p };
            {   // the position array holds n / 2 + 16 entries (a four-line record has at most one newline per two bytes): count first,
                // so that malformed input is an error and not a write past the array
                NewlineAsInt conv = { (const char *) ctx->d[F_RAW0 + b].p };
                cub::TransformInputIterator<int, NewlineAsInt, cub::CountingInputIterator<int>> cnt_it(it, conv);
                cub::DeviceReduce::Sum(nullptr, tmp, cnt_it, d_misc + 4 + b, (int) hn[b], st);
                if (ctx->ensure(ctx->d[F_TMP], tmp)) return 1;
                BM2_CUDA_OK(cub::DeviceReduce::Sum(ctx->d[F_TMP].p, tmp, cnt_it, d_misc + 4 + b, (int) hn[b], st));
                int h_n = 0;
                BM2_CUDA_OK(cudaMemcpyAsync(&h_n, d_misc + 4 + b, 4, cudaMemcpyDeviceToHost, st));
                BM2_CUDA_OK(cudaStreamSynchronize(st));
                if ((int64_t) h_n > hn[b] / 2 + 8) { bm2_set_error(ctx, "bm2_fastq_encode: too many line ends for FASTQ records"); return 2; }
                tmp = 0;
            }
            cub::DeviceSelect::If(nullptr, tmp, it, (int32_t *) ctx->d[F_NL0 + b].p, d_misc + b, (int) hn[b], pred, st);
            if (ctx->ensure(ctx->d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::If(ctx->d[F_TMP].p, tmp, it, (int32_t *) ctx->d[F_NL0 + b].p, d_misc + b, (int) hn[b], pred, st));
        }
    }
    int h_cnt[2] = { 0, 0 };
    BM2_CUDA_OK(cudaMemcpyAsync(h_cnt, d_misc, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    for (int b = 0; b < nbuf; ++b) {
        int lines = h_cnt[b];
        if (hn[b] > 0 && hb[b][hn[b] - 1] != '\n') {      // last line without a newline: a virtual one at the end of the buffer
            const int32_t endpos = (int32_t) hn[b];
            BM2_CUDA_OK(cudaMemcpyAsync((int32_t *) ctx->d[F_NL0 + b].p + lines, &endpos, 4, cudaMemcpyHostToDevice, st));
            BM2_CUDA_OK(cudaStreamSynchronize(st));
            ++lines;
        }
        if (lines % 4) { bm2_set_error(ctx, "bm2_fastq_encode: the number of lines is not a multiple of four (wrapped or truncated records)"); return 2; }
        n_rec[b] = lines / 4;
    }
    if (nbuf == 2 && n_rec[0] != n_rec[1]) { bm2_set_error(ctx, "bm2_fastq_encode: the two files hold different numbers of records"); return 2; }
    const int n_reads = n_rec[0] * nbuf;
    out->n_reads = n_reads;
    if (ctx->ensure(ctx->d[F_SPANS], (size_t) (n_reads + 1) * sizeof(Span)) || ctx->ensure(ctx->d[F_LENS], (size_t) (n_reads + 2) * 8) ||
        ctx->ensure(ctx->d[F_OFFS], (size_t) (n_reads + 2) * 8)) return 1;
    Span *d_spans = (Span *) ctx->d[F_SPANS].p; int64_t *d_lens = (int64_t *) ctx->d[F_LENS].p, *d_offs = (int64_t *) ctx->d[F_OFFS].p;
    BM2_CUDA_OK(cudaMemsetAsync(d_lens + n_reads, 0, 8, st));
    for (int b = 0; b < nbuf && n_rec[b] > 0; ++b)
        fastq_spans_kernel<<<(n_rec[b] + 255) / 256, 256, 0, st>>>((const char *) ctx->d[F_RAW0 + b].p, (const int32_t *) ctx->d[F_NL0 + b].p, n_rec[b], b, nbuf,
                                                                      d_spans, d_lens, d_misc + 2);
    {
        size_t tmp = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_lens, d_offs, n_reads + 1, st);
        if (ctx->ensure(ctx->d[F_TMP], tmp)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->d[F_TMP].p, tmp, d_lens, d_offs, n_reads + 1, st));
    }
    int64_t total = 0; int h_err = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&total, d_offs + n_reads, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&h_err, d_misc + 2, 4, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    if (h_err) { bm2_set_error(ctx, "bm2_fastq_encode: malformed record " + std::to_string(h_err - 1) + " (expected @name / sequence / + / qualities of the same length)"); return 2; }
    if (ctx->ensure(ctx->d[F_CODES], (size_t) total + 16) || ctx->ensure(ctx->d[F_QUALS], (size_t) total + 16)) return 1;
    if (n_reads > 0) {
        int blocks = (n_reads + 7) / 8; if (blocks > ctx->n_sm * 16) blocks = ctx->n_sm * 16;
        fastq_encode_kernel<<<blocks, 256, 0, st>>>((const char *) ctx->d[F_RAW0].p, (const char *) ctx->d[F_RAW1].p, d_spans, d_offs, n_reads, nbuf,
                                                     (uint8_t *) ctx->d[F_CODES].p, (char *) ctx->d[F_QUALS].p);
    }
    // host copies: offsets, codes, qualities (the SAM stage and the formatter read them), name positions
    if (ctx->ensure_host(ctx->h[FH_OFFS], (size_t) (n_reads + 1) * 8) || ctx->ensure_host(ctx->h[FH_CODES], (size_t) total + 16) ||
        ctx->ensure_host(ctx->h[FH_QUALS], (size_t) total + 16) || ctx->ensure_host(ctx->h[FH_SPANS], (size_t) (n_reads + 1) * sizeof(Span)) ||
        ctx->ensure_host(ctx->h[FH_NAMEBEG], (size_t) (n_reads + 1) * 8) || ctx->ensure_host(ctx->h[FH_NAMELEN], (size_t) (n_reads + 1) * 4)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->h[FH_OFFS].p, d_offs, (size_t) (n_reads + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (total) BM2_CUDA_OK(cudaMemcpyAsync(ctx->h[FH_CODES].p, ctx->d[F_CODES].p, (size_t) total, cudaMemcpyDeviceToHost, st));
    if (total) BM2_CUDA_OK(cudaMemcpyAsync(ctx->h[FH_QUALS].p, ctx->d[F_QUALS].p, (size_t) total, cudaMemcpyDeviceToHost, st));
    if (n_reads) BM2_CUDA_OK(cudaMemcpyAsync(ctx->h[FH_SPANS].p, d_spans, (size_t) n_reads * sizeof(Span), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaGetLastError());
    const Span *hs = (const Span *) ctx->h[FH_SPANS].p;
    int64_t *nb = (int64_t *) ctx->h[FH_NAMEBEG].p; int32_t *nlv = (int32_t *) ctx->h[FH_NAMELEN].p;
    for (int r = 0; r < n_reads; ++r) { nb[r] = hs[r].name_beg; nlv[r] = hs[r].name_len; }
    out->d_codes = (const uint8_t *) ctx->d[F_CODES].p; out->d_offsets = d_offs;
    out->codes = (const uint8_t *) ctx->h[FH_CODES].p; out->offsets = (const int64_t *) ctx->h[FH_OFFS].p;
    out->quals = (const char *) ctx->h[FH_QUALS].p; out->name_beg = nb; out->name_len = nlv;
    ctx->fq_n_reads = n_reads; ctx->fq_n_bufs = nbuf;
    return 0;
}

extern "C" int bm2_fastq_comments(bm2_ctx *ctx, const int64_t **beg, const int32_t **len) {
    if (!ctx || !beg || !len) { if (ctx) bm2_set_error(ctx, "bm2_fastq_comments: bad arguments"); return 1; }
    const int n = ctx->fq_n_reads;
    if (ctx->ensure_host(ctx->h[FH_CMTBEG], (size_t) (n + 1) * 8) || ctx->ensure_host(ctx->h[FH_CMTLEN], (size_t) (n + 1) * 4)) return 1;
    const Span *hs = (const Span *) ctx->h[FH_SPANS].p;
    int64_t *cb = (int64_t *) ctx->h[FH_CMTBEG].p; int32_t *cl = (int32_t *) ctx->h[FH_CMTLEN].p;
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
    if (ctx->ensure(ctx->d[F_KEY], (size_t) (n + 1) * 4) || ctx->ensure(ctx->d[F_RUN], (size_t) (n + 1) * 4) || ctx->ensure(ctx->d[F_SCNT], 16)) return 1;
    for (int s = 0; s < 2; ++s)
        if (ctx->ensure(ctx->d[F_SFLAG + s], (size_t) n + 16) || ctx->ensure(ctx->d[F_SIDX + s], (size_t) (n + 1) * 4) ||
            ctx->ensure(ctx->d[F_SLEN + s], (size_t) (n + 2) * 8) || ctx->ensure(ctx->d[F_SOFF + s], (size_t) (n + 2) * 8)) return 1;
    const Span *d_spans = (const Span *) ctx->d[F_SPANS].p;
    const int64_t *d_offs = (const int64_t *) ctx->d[F_OFFS].p;
    int *d_key = (int *) ctx->d[F_KEY].p, *d_run = (int *) ctx->d[F_RUN].p, *d_cnt = (int *) ctx->d[F_SCNT].p;
    int h_cnt[2] = { 0, 0 };
    if (n > 0) {
        const int blocks = (n + 255) / 256;
        fastq_link_kernel<<<blocks, 256, 0, st>>>((const char *) ctx->d[F_RAW0].p, d_spans, n, d_key);
        size_t tmp = 0;
        cub::DeviceScan::InclusiveScan(nullptr, tmp, d_key, d_run, cub::Max(), n, st);
        if (ctx->ensure(ctx->d[F_TMP], tmp)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::InclusiveScan(ctx->d[F_TMP].p, tmp, d_key, d_run, cub::Max(), n, st));
        fastq_classify_kernel<<<blocks, 256, 0, st>>>(d_run, n, (uint8_t *) ctx->d[F_SFLAG].p, (uint8_t *) ctx->d[F_SFLAG + 1].p);
        cub::CountingInputIterator<int32_t> it(0);
        for (int s = 0; s < 2; ++s) {       // stable compaction: the reads of each set in file order
            tmp = 0;
            cub::DeviceSelect::Flagged(nullptr, tmp, it, (const uint8_t *) ctx->d[F_SFLAG + s].p, (int32_t *) ctx->d[F_SIDX + s].p, d_cnt + s, n, st);
            if (ctx->ensure(ctx->d[F_TMP], tmp)) return 1;
            BM2_CUDA_OK(cub::DeviceSelect::Flagged(ctx->d[F_TMP].p, tmp, it, (const uint8_t *) ctx->d[F_SFLAG + s].p, (int32_t *) ctx->d[F_SIDX + s].p,
                                                   d_cnt + s, n, st));
        }
        BM2_CUDA_OK(cudaMemcpyAsync(h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
    }
    const Span *hs = (const Span *) ctx->h[FH_SPANS].p;
    for (int s = 0; s < 2; ++s) {
        const int m = h_cnt[s];
        const int32_t *d_idx = (const int32_t *) ctx->d[F_SIDX + s].p;
        int64_t *d_len = (int64_t *) ctx->d[F_SLEN + s].p, *d_soff = (int64_t *) ctx->d[F_SOFF + s].p;
        fastq_gather_lens_kernel<<<(m + 1 + 255) / 256, 256, 0, st>>>(d_idx, d_offs, m, d_len);
        size_t tmp = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_len, d_soff, m + 1, st);
        if (ctx->ensure(ctx->d[F_TMP], tmp)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->d[F_TMP].p, tmp, d_len, d_soff, m + 1, st));
        int64_t total = 0;
        BM2_CUDA_OK(cudaMemcpyAsync(&total, d_soff + m, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        if (ctx->ensure(ctx->d[F_SCODES + s], (size_t) total + 16) || ctx->ensure(ctx->d[F_SQUALS + s], (size_t) total + 16)) return 1;
        if (m > 0) {
            int blocks = (m + 7) / 8; if (blocks > ctx->n_sm * 16) blocks = ctx->n_sm * 16;
            fastq_gather_kernel<<<blocks, 256, 0, st>>>(d_idx, d_offs, d_soff, m, (const uint8_t *) ctx->d[F_CODES].p, (const char *) ctx->d[F_QUALS].p,
                                                        (uint8_t *) ctx->d[F_SCODES + s].p, (char *) ctx->d[F_SQUALS + s].p);
        }
        HostBuf *h = ctx->h + FH_SPLIT + 8 * s;
        if (ctx->ensure_host(h[SH_OFFS], (size_t) (m + 1) * 8) || ctx->ensure_host(h[SH_CODES], (size_t) total + 16) ||
            ctx->ensure_host(h[SH_QUALS], (size_t) total + 16) || ctx->ensure_host(h[SH_NAMEBEG], (size_t) (m + 1) * 8) ||
            ctx->ensure_host(h[SH_NAMELEN], (size_t) (m + 1) * 4) || ctx->ensure_host(h[SH_CMTBEG], (size_t) (m + 1) * 8) ||
            ctx->ensure_host(h[SH_CMTLEN], (size_t) (m + 1) * 4) || ctx->ensure_host(h[SH_IDX], (size_t) (m + 1) * 4)) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(h[SH_OFFS].p, d_soff, (size_t) (m + 1) * 8, cudaMemcpyDeviceToHost, st));
        if (total) BM2_CUDA_OK(cudaMemcpyAsync(h[SH_CODES].p, ctx->d[F_SCODES + s].p, (size_t) total, cudaMemcpyDeviceToHost, st));
        if (total) BM2_CUDA_OK(cudaMemcpyAsync(h[SH_QUALS].p, ctx->d[F_SQUALS + s].p, (size_t) total, cudaMemcpyDeviceToHost, st));
        if (m) BM2_CUDA_OK(cudaMemcpyAsync(h[SH_IDX].p, d_idx, (size_t) m * 4, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        BM2_CUDA_OK(cudaGetLastError());
        const int32_t *idx = (const int32_t *) h[SH_IDX].p;
        int64_t *nb = (int64_t *) h[SH_NAMEBEG].p, *cb = (int64_t *) h[SH_CMTBEG].p;
        int32_t *nlv = (int32_t *) h[SH_NAMELEN].p, *cl = (int32_t *) h[SH_CMTLEN].p;
        for (int j = 0; j < m; ++j) { const Span &sp = hs[idx[j]]; nb[j] = sp.name_beg; nlv[j] = sp.name_len; cb[j] = sp.cmt_beg; cl[j] = sp.cmt_len; }
        bm2_fastq_batch &b = out->set[s];
        b.n_reads = m;
        b.d_codes = (const uint8_t *) ctx->d[F_SCODES + s].p; b.d_offsets = d_soff;
        b.codes = (const uint8_t *) h[SH_CODES].p; b.offsets = (const int64_t *) h[SH_OFFS].p; b.quals = (const char *) h[SH_QUALS].p;
        b.name_beg = nb; b.name_len = nlv;
        out->comment_beg[s] = cb; out->comment_len[s] = cl; out->read_index[s] = idx;
    }
    return 0;
}

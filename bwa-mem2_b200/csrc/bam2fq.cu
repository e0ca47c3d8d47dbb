// bam2fq.cu — the GPU half of bm2_bam2fq: BAM records back to FASTQ text (bam2fq_device.cuh's rule; the host half, the pairing order and
// the streams, is bam2fq.h).
//   bm2_bam2fq_records  one window: one warp per record classifies it, checks its qualities with a vote per 32 bytes, finds its text length
//                       and, for a READ1 or READ2, hashes its QNAME (dup_name_hash, as bm2_markdup_records does).  The first read error by
//                       index is kept with atomicMin.  The window stays on the device for the format calls.
//   bm2_bam2fq_format   one output stream: one thread per listed record gives its text length, a cub inclusive scan the 64-bit offsets, then
//                       one warp per record writes its lines 32 bytes at a time (b2f_write_part) after the stream's carried bytes.  With
//                       compression the carry + text is cut into 65280-byte blocks and the full ones go to bgzf_compress_device, so the text
//                       never crosses PCIe uncompressed; the unfinished block comes back as the tail.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "bam2fq_device.cuh"
#include "bgzf_device.cuh"
#include "markdup_device.cuh"
#include <cub/device/device_scan.cuh>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kRecBytes = 300;              // a short read's record, for bm2_bam2fq_memory's estimate
const char *const kErrText[] = {"has no bases (l_seq 0)", "has a quality above 93"};

__global__ void __launch_bounds__(kWarps * 32) b2f_record_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                                 int suffixes, bm2_bam2fq_rec *out, unsigned long long *err) {
    const int lane = threadIdx.x & 31;
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const uint8_t *r = base + starts[w];
        const B2fView v = b2f_view(r, suffixes);
        bm2_bam2fq_rec o{};
        o.kind = b2f_kind(v.flag);
        int e = B2F_ERR_NONE;
        if (o.kind != B2F_SKIP) {
            if (v.l_seq == 0) e = B2F_ERR_EMPTY;
            else if (__any_sync(kFull, b2f_check_part(v, lane, 32) != B2F_ERR_NONE)) e = B2F_ERR_QUAL;
            o.text_len = b2f_text_len(v);
            if (lane == 0 && o.kind != B2F_OTHER) o.hash = dup_name_hash(v.name, v.name_len);
        }
        if (lane == 0) {
            out[w] = o;
            if (e) atomicMin(err, (unsigned long long) w << 4 | (unsigned) e);
        }
    }
}

__device__ __forceinline__ const uint8_t *b2f_rec(int64_t ref, const uint8_t *win, const int64_t *wst, const uint8_t *extra, const int64_t *xst) {
    return ref >= 0 ? win + wst[ref] : extra + xst[~ref];
}

__global__ void b2f_len_kernel(const int64_t *__restrict__ list, int64_t n, const uint8_t *__restrict__ win, const int64_t *__restrict__ wst,
                               const uint8_t *__restrict__ extra, const int64_t *__restrict__ xst, int suffixes, int64_t *lens) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) lens[i] = b2f_text_len(b2f_view(b2f_rec(list[i], win, wst, extra, xst), suffixes));
}

// offs[i]: the end of record i's text (an inclusive scan), so record i starts at offs[i - 1] (0 for the first)
__global__ void __launch_bounds__(kWarps * 32) b2f_format_kernel(const int64_t *__restrict__ list, int64_t n, const uint8_t *__restrict__ win,
                                                                 const int64_t *__restrict__ wst, const uint8_t *__restrict__ extra,
                                                                 const int64_t *__restrict__ xst, int suffixes, const int64_t *__restrict__ offs,
                                                                 uint8_t *text) {
    const int lane = threadIdx.x & 31;
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const B2fView v = b2f_view(b2f_rec(list[w], win, wst, extra, xst), suffixes);
        b2f_write_part(v, text + (w ? offs[w - 1] : 0), lane, 32);
    }
}

enum { BF_WIN, BF_STARTS, BF_INFO, BF_ERR, BF_LIST, BF_EXTRA, BF_XSTARTS, BF_LENS, BF_OFFS, BF_TEXT, BF_TEMP, BF_END };
enum { BH_INFO, BH_TEXT, BH_END };
static_assert(BF_END == std::extent<decltype(bm2_ctx::b2f_d)>::value, "bm2_ctx::b2f_d: one buffer per slot");
static_assert(BH_END == std::extent<decltype(bm2_ctx::b2f_h)>::value, "bm2_ctx::b2f_h: one buffer per slot");
static_assert(sizeof(bm2_bam2fq_rec) == 24 && sizeof(bm2_bam2fq_out) == 40, "bm2_bam2fq_rec, bm2_bam2fq_out: no padding, as the Python bindings read them");

}  // namespace

extern "C" int bm2_bam2fq_records(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, int32_t suffixes,
                                  const bm2_bam2fq_rec **out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts)) {
        if (ctx) bm2_set_error(ctx, "bm2_bam2fq_records: bad arguments");
        return 1;
    }
    ctx->b2f_n_recs = 0;
    if (bam_check_records(ctx, "bm2_bam2fq_records", recs, n, starts, n_recs)) return 1;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->b2f_d;
    if (ctx->ensure(b[BF_WIN], (size_t) n + 16) || ctx->ensure(b[BF_STARTS], (size_t) n_recs * 8 + 8) ||
        ctx->ensure(b[BF_INFO], (size_t) n_recs * sizeof(bm2_bam2fq_rec) + 8) || ctx->ensure(b[BF_ERR], 8) ||
        ctx->ensure_host(ctx->b2f_h[BH_INFO], (size_t) n_recs * sizeof(bm2_bam2fq_rec) + 16)) return 1;
    for (cudaEvent_t &ev : ctx->b2f_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    ctx->b2f_recs.resize((size_t) n_recs);
    *out = ctx->b2f_recs.data();
    if (!n_recs) return 0;
    const bm2_bam2fq_rec *h_info = (const bm2_bam2fq_rec *) ctx->b2f_h[BH_INFO].p;
    unsigned long long err = ~0ULL;
    BM2_CUDA_OK(cudaMemcpyAsync(b[BF_WIN].p, recs, (size_t) n, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(b[BF_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemsetAsync(b[BF_ERR].p, 0xFF, 8, st));
    const int64_t g = bm2_min<int64_t>((n_recs + kWarps - 1) / kWarps, (int64_t) ctx->n_sm * 16);
    BM2_CUDA_OK(cudaEventRecord(ctx->b2f_ev[0], st));
    b2f_record_kernel<<<(unsigned) g, kWarps * 32, 0, st>>>((const uint8_t *) b[BF_WIN].p, (const int64_t *) b[BF_STARTS].p, n_recs, suffixes ? 1 : 0,
                                                            (bm2_bam2fq_rec *) b[BF_INFO].p, (unsigned long long *) b[BF_ERR].p);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->b2f_ev[1], st));
    BM2_CUDA_OK(cudaMemcpyAsync((void *) h_info, b[BF_INFO].p, (size_t) n_recs * sizeof(bm2_bam2fq_rec), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&err, b[BF_ERR].p, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->b2f_ev[0], ctx->b2f_ev[1]));
    ctx->b2f_record_ms += ms;
    if (err != ~0ULL) {                                                  // a read error: nothing of this window is kept
        const int64_t i = (int64_t) (err >> 4);
        const uint8_t *r = recs + starts[i];
        bm2_set_error(ctx, "bm2_bam2fq_records: read " + std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0) + " (record " + std::to_string(i) +
                               " of the window) " + kErrText[(err & 15) - 1]);
        return 2;
    }
    memcpy(ctx->b2f_recs.data(), h_info, (size_t) n_recs * sizeof(bm2_bam2fq_rec));
    ctx->b2f_n_recs = n_recs;
    return 0;
}

extern "C" int bm2_bam2fq_format(bm2_ctx *ctx, const int64_t *list, int64_t n_list, const uint8_t *extra, int64_t extra_len, const int64_t *extra_starts,
                                 int64_t n_extra, int32_t suffixes, const uint8_t *carry, int64_t carry_len, int32_t compress, int32_t last,
                                 bm2_bam2fq_out *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || n_list < 0 || (n_list && !list) || extra_len < 0 || (extra_len && !extra) || n_extra < 0 || (n_extra && !extra_starts) ||
        carry_len < 0 || carry_len >= BGZF_BLOCK || (carry_len && !carry) || (carry_len && !compress)) {
        if (ctx) bm2_set_error(ctx, "bm2_bam2fq_format: bad arguments");
        return 1;
    }
    if (n_list >= ((int64_t) 1 << 31)) { bm2_set_error(ctx, "bm2_bam2fq_format: 2^31 records or more in one call"); return 1; }
    for (int64_t i = 0; i < n_list; ++i)
        if (list[i] >= ctx->b2f_n_recs || (list[i] < 0 && ~list[i] >= n_extra)) {
            bm2_set_error(ctx, "bm2_bam2fq_format: entry " + std::to_string(i) + " names no record of the window or of extra");
            return 1;
        }
    if (bam_check_records(ctx, "bm2_bam2fq_format", extra, extra_len, extra_starts, n_extra)) return 1;
    memset(out, 0, sizeof *out);
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->b2f_d;
    const int64_t nl = bm2_max<int64_t>(n_list, 1);
    size_t temp = 0;
    BM2_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, temp, (const int64_t *) nullptr, (int64_t *) nullptr, (int) nl, st));
    if (ctx->ensure(b[BF_LIST], (size_t) nl * 8) || ctx->ensure(b[BF_EXTRA], (size_t) extra_len + 16) ||
        ctx->ensure(b[BF_XSTARTS], (size_t) n_extra * 8 + 8) || ctx->ensure(b[BF_LENS], (size_t) nl * 8) || ctx->ensure(b[BF_OFFS], (size_t) nl * 8) ||
        ctx->ensure(b[BF_TEMP], temp + 16) || ctx->ensure(b[BF_WIN], 16) || ctx->ensure(b[BF_STARTS], 8)) return 1;
    for (cudaEvent_t &ev : ctx->b2f_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    int64_t text_len = 0;
    const uint8_t *win = (const uint8_t *) b[BF_WIN].p, *dx = (const uint8_t *) b[BF_EXTRA].p;
    const int64_t *wst = (const int64_t *) b[BF_STARTS].p, *xst = (const int64_t *) b[BF_XSTARTS].p, *dl = (const int64_t *) b[BF_LIST].p;
    int64_t *lens = (int64_t *) b[BF_LENS].p, *offs = (int64_t *) b[BF_OFFS].p;
    if (n_list) {
        BM2_CUDA_OK(cudaMemcpyAsync(b[BF_LIST].p, list, (size_t) n_list * 8, cudaMemcpyHostToDevice, st));
        if (extra_len) BM2_CUDA_OK(cudaMemcpyAsync(b[BF_EXTRA].p, extra, (size_t) extra_len, cudaMemcpyHostToDevice, st));
        if (n_extra) BM2_CUDA_OK(cudaMemcpyAsync(b[BF_XSTARTS].p, extra_starts, (size_t) n_extra * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaEventRecord(ctx->b2f_ev[2], st));
        b2f_len_kernel<<<(unsigned) ((n_list + 255) / 256), 256, 0, st>>>(dl, n_list, win, wst, dx, xst, suffixes ? 1 : 0, lens);
        BM2_CUDA_OK(cudaGetLastError());
        size_t tb = b[BF_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceScan::InclusiveSum(b[BF_TEMP].p, tb, (const int64_t *) lens, offs, (int) n_list, st));
        BM2_CUDA_OK(cudaMemcpyAsync(&text_len, offs + n_list - 1, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
    }
    if (ctx->ensure(b[BF_TEXT], (size_t) (carry_len + text_len) + 16)) return 1;
    uint8_t *text = (uint8_t *) b[BF_TEXT].p;
    if (carry_len) BM2_CUDA_OK(cudaMemcpy(text, carry, (size_t) carry_len, cudaMemcpyHostToDevice));
    if (n_list) {
        const int64_t g = bm2_min<int64_t>((n_list + kWarps - 1) / kWarps, (int64_t) ctx->n_sm * 16);
        b2f_format_kernel<<<(unsigned) g, kWarps * 32, 0, st>>>(dl, n_list, win, wst, dx, xst, suffixes ? 1 : 0, offs, text + carry_len);
        BM2_CUDA_OK(cudaGetLastError());
        BM2_CUDA_OK(cudaEventRecord(ctx->b2f_ev[3], st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        float ms = 0;
        BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->b2f_ev[2], ctx->b2f_ev[3]));
        ctx->b2f_format_ms += ms;
    }
    out->text_len = text_len;
    const int64_t total = carry_len + text_len;
    if (!compress) {
        if (ctx->ensure_host(ctx->b2f_h[BH_TEXT], (size_t) total + 16)) return 1;
        if (total) BM2_CUDA_OK(cudaMemcpy(ctx->b2f_h[BH_TEXT].p, text, (size_t) total, cudaMemcpyDeviceToHost));
        out->data = (const uint8_t *) ctx->b2f_h[BH_TEXT].p; out->len = total;
        return 0;
    }
    // bgzip's cut: blocks of exactly BGZF_BLOCK bytes whatever the line ends, the short one only at the end
    const int64_t full = total / BGZF_BLOCK, nb = full + (last && total % BGZF_BLOCK ? 1 : 0);
    std::vector<int64_t> bst((size_t) nb + 1);
    for (int64_t k = 0; k <= nb; ++k) bst[(size_t) k] = bm2_min<int64_t>(k * BGZF_BLOCK, total);
    const uint8_t *z = nullptr; int64_t zl = 0;
    if (nb) {
        if (bgzf_compress_device(ctx, text, bst.data(), nb, &z, &zl, nullptr)) return 1;
        ctx->b2f_bgzf_ms += ctx->bgzf_ms;
    }
    out->data = z; out->len = zl;
    const int64_t t0 = full * BGZF_BLOCK;
    ctx->b2f_tail.resize((size_t) (last ? 0 : total - t0));
    if (!ctx->b2f_tail.empty()) BM2_CUDA_OK(cudaMemcpy(ctx->b2f_tail.data(), text + t0, ctx->b2f_tail.size(), cudaMemcpyDeviceToHost));
    out->tail = ctx->b2f_tail.data(); out->tail_len = (int64_t) ctx->b2f_tail.size();
    return 0;
}

extern "C" int bm2_last_bam2fq_stats(const bm2_ctx *ctx, bm2_bam2fq_stats_t *out) {
    if (!ctx || !out) return 1;
    out->record_ms = ctx->b2f_record_ms; out->format_ms = ctx->b2f_format_ms; out->bgzf_ms = ctx->b2f_bgzf_ms;
    return 0;
}

extern "C" int bm2_bam2fq_memory(const bm2_ctx *ctx, int64_t window_bytes, int64_t *needed, int64_t *free_bytes) {
    if (!ctx || window_bytes < 0 || !needed || !free_bytes) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // each rounded up by 1.25 as bm2_ctx::ensure allocates: the window; the text of one window, at most 2 x its record bytes (a record holds
    // its name, its bases in half a byte and its qualities, the text its name, bases and qualities and 8 more bytes), plus a carried block;
    // the BGZF slots (one 64 KiB slot per 65280-byte block) and the gathered members; per record 8 bytes of starts, 24 of bm2_bam2fq_rec,
    // 8 of list, 16 of lengths and offsets, and for the pairing (every record a half at most) 24 bytes of half, 16 of sort keys, 8 of order,
    // 4 of partner and about 60 of name and sort scratch.  The carried halves and their names are counted as one more window.
    const double w = (double) window_bytes, text = 2 * w + BGZF_BLOCK, slots = (text / BGZF_BLOCK + 2) * BGZF_MAX_MEMBER;
    const double bytes = 1.25 * (2 * w + text + 2 * slots + (56.0 + 112.0) * (2 * w / kRecBytes + 1)) + 64.0 * (1 << 20);
    size_t fr = 0, tot = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
    *needed = (int64_t) bytes; *free_bytes = (int64_t) fr;
    return 0;
}

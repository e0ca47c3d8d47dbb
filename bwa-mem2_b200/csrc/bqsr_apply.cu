// bqsr_apply.cu — the base qualities of BAM records recalibrated on the GPU from a recalibration table (bm2_applybqsr; bqsr_device.cuh's
// apply rule), then compressed as they leave.
//   bm2_bqsr_apply_set    the dense tables of each read group (bqsr_report.h) and the header's read-group map to the context
//   bm2_bqsr_apply        one window: the records (contiguous, in file order) are uploaded after the carry, rewritten in place, and the stream
//                         carry + records is compressed by bam_compress_stream, the tail bm2_bam_sort_compress uses, so the members, carry and
//                         bm2_sort_rec index data are what SortedWriter and BaiBuilder take
//   bm2_last_bqsr_apply_stats  device times, counts and the first read error since the tables came
// The kernel: one warp per record, grid-stride.  The read-group map (each @RG ID and its table index) sits in shared memory.  Lane 0 finds
// the RG:Z value in the aux data and the lanes compare it against 32 IDs at a time (bqsr_rg_lookup); ballots over the qualities find the low-quality tails
// and the qualities above 93; then the lanes take consecutive bases, each computing its context and cycle (bqsr_covariates, shared with
// the counting kernel), reading its deltas and writing its quality in place.  The contexts read bases, not qualities, so the writes do not
// disturb the other lanes.  The D_cyc table (94 x 1001 doubles per read group) is read from global memory through L2.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "bam_sort_device.cuh"
#include "bqsr_device.cuh"
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int64_t kMapMax = 32768;          // bytes of the read-group map (in shared memory)
constexpr int kRecBytes = 300;              // a short read's record, for bm2_bqsr_apply_memory's estimate
enum { CNT_CHANGED, CNT_RECAL, CNT_KEPT, CNT_ERR, CNT_END };

// map: n_ids int4 {offset of the ID's bytes from the map's start, length, table index or -1, 0}, then the bytes
__global__ void __launch_bounds__(kWarps * 32) bqsr_apply_kernel(uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                                 const int4 *__restrict__ map, int map_bytes, int n_ids, const double *__restrict__ P,
                                                                 const double *__restrict__ Dctx, const double *__restrict__ Dcyc, bm2_sort_rec *info,
                                                                 unsigned long long *cnt, int64_t first) {
    extern __shared__ int4 s_map[];
    for (int i = threadIdx.x; i < map_bytes / 16; i += blockDim.x) s_map[i] = map[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    unsigned long long changed = 0, recal = 0, kept = 0;
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        uint8_t *rec = base + starts[w];
        if (lane == 0) info[w] = bam_sort_rec(rec);
        int32_t len = 0, at = -1;
        if (lane == 0) at = bqsr_aux_rg(rec, &len);
        at = __shfl_sync(kFull, at, 0); len = __shfl_sync(kFull, len, 0);
        const int j = at >= 0 ? bqsr_rg_lookup((const BqsrRgEntry *) s_map, n_ids, rec, at, len) : -1;
        const int rg = j >= 0 ? s_map[j].z : -1;
        BqsrRec r;
        bqsr_apply_prep(rec, r);
        if (rg < 0) r.status = BQSR_KEEP;
        if (r.status == BQSR_APPLY) {                                    // the low-quality tails and the quality check, 32 bases at a time
            int32_t tl = r.hi, tr = r.hi;
            bool bad = false;
            for (int32_t k0 = 0; k0 < r.hi; k0 += 32) {
                const int32_t k = k0 + lane;
                const int q = k < r.hi ? r.qual[k] : 0;
                const unsigned m = __ballot_sync(kFull, q > BQSR_TAIL_Q);
                bad |= __any_sync(kFull, q > BQSR_NQ - 1);
                if (m) { if (tl == r.hi) tl = k0 + __ffs(m) - 1; tr = k0 + 32 - __clz(m); }
            }
            r.tl = tl; r.tr = tr;
            if (bad) r.status = BQSR_ERR_QUAL;
        }
        if (r.status >= BQSR_ERR_NOQUAL) {
            if (lane == 0) atomicMin(&cnt[CNT_ERR], (unsigned long long) (first + w) << 3 | (unsigned) r.status);
            continue;
        }
        if (r.status == BQSR_KEEP) { kept += lane == 0; continue; }
        recal += lane == 0;
        const BqsrApplyView t{P + (size_t) rg * BQSR_NQ, Dctx + (size_t) rg * BQSR_NQ * BQSR_NCTX, Dcyc + (size_t) rg * BQSR_NQ * BQSR_NCYC};
        uint8_t *qual = (uint8_t *) r.qual;
        for (int32_t k = lane; k < r.hi; k += 32) {
            const int q = qual[k];
            int cx, cyc;
            bqsr_covariates(r, k, cx, cyc);
            const int nq = bqsr_recal_q(t, q, cx, cyc);
            if (nq != q) { qual[k] = (uint8_t) nq; ++changed; }
        }
    }
    for (int o = 16; o; o >>= 1) changed += __shfl_xor_sync(kFull, changed, o);
    if (lane == 0) {
        if (changed) atomicAdd(&cnt[CNT_CHANGED], changed);
        if (recal) atomicAdd(&cnt[CNT_RECAL], recal);
        if (kept) atomicAdd(&cnt[CNT_KEPT], kept);
    }
}

enum { AP_P, AP_CTX, AP_CYC, AP_MAP, AP_STREAM, AP_STARTS, AP_INFO, AP_CNT, AP_END };
enum { AH_INFO, AH_END };
static_assert(AP_END == std::extent<decltype(bm2_ctx::bqa_d)>::value, "bm2_ctx::bqa_d: one buffer per slot");
static_assert(AH_END == std::extent<decltype(bm2_ctx::bqa_h)>::value, "bm2_ctx::bqa_h: one buffer per slot");

const char *const kErrText[2] = {"is longer than 500 bases", "has a base quality above 93"};

}  // namespace

extern "C" int bm2_bqsr_apply_set(bm2_ctx *ctx, const bm2_bqsr_apply_tables_t *t) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !t || t->n_rg < 0 || (t->n_rg && (!t->P || !t->ctx || !t->cyc)) || t->n_ids < 0 || (t->n_ids && (!t->ids || !t->id_table))) {
        if (ctx) bm2_set_error(ctx, "bm2_bqsr_apply_set: bad arguments");
        return 1;
    }
    std::vector<int4> map((size_t) t->n_ids);
    std::string bytes;
    for (int32_t i = 0; i < t->n_ids; ++i) {
        if (!t->ids[i] || t->id_table[i] < -1 || t->id_table[i] >= t->n_rg) { bm2_set_error(ctx, "bm2_bqsr_apply_set: a bad read-group entry"); return 1; }
        map[(size_t) i] = int4{(int) bytes.size(), (int) strlen(t->ids[i]), t->id_table[i], 0};
        bytes += t->ids[i];
    }
    const int64_t total = ((16 * (int64_t) t->n_ids + (int64_t) bytes.size()) + 15) / 16 * 16;
    if (total > kMapMax) {
        bm2_set_error(ctx, "bm2_bqsr_apply_set: the header's read-group IDs take " + std::to_string(total) + " bytes, more than " + std::to_string(kMapMax));
        return 1;
    }
    for (int4 &e : map) e.x += 16 * t->n_ids;
    std::vector<uint8_t> blob((size_t) total + 16, 0);
    if (t->n_ids) memcpy(blob.data(), map.data(), map.size() * 16);
    memcpy(blob.data() + 16 * t->n_ids, bytes.data(), bytes.size());
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->bqa_d;
    const size_t np = (size_t) t->n_rg * BQSR_NQ * 8, nc = np * BQSR_NCTX, ny = np * BQSR_NCYC;
    if (ctx->ensure(b[AP_P], np + 8) || ctx->ensure(b[AP_CTX], nc + 8) || ctx->ensure(b[AP_CYC], ny + 8) || ctx->ensure(b[AP_MAP], blob.size()) ||
        ctx->ensure(b[AP_CNT], CNT_END * 8)) return 1;
    if (np) {
        BM2_CUDA_OK(cudaMemcpy(b[AP_P].p, t->P, np, cudaMemcpyHostToDevice));
        BM2_CUDA_OK(cudaMemcpy(b[AP_CTX].p, t->ctx, nc, cudaMemcpyHostToDevice));
        BM2_CUDA_OK(cudaMemcpy(b[AP_CYC].p, t->cyc, ny, cudaMemcpyHostToDevice));
    }
    BM2_CUDA_OK(cudaMemcpy(b[AP_MAP].p, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    const unsigned long long zero[CNT_END] = {0, 0, 0, ~0ULL};
    BM2_CUDA_OK(cudaMemcpy(b[AP_CNT].p, zero, sizeof zero, cudaMemcpyHostToDevice));
    ctx->bqa_map_bytes = total; ctx->bqa_n_ids = t->n_ids;
    ctx->bqa_seen = 0; ctx->bqa_ms = 0; ctx->bqa_bgzf_ms = 0; ctx->bqa_err_kind = 0; ctx->bqa_err_index = -1; ctx->bqa_err_name.clear();
    ctx->bqa_set = true;
    return 0;
}

extern "C" int bm2_bqsr_apply(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry, int64_t carry_len,
                              int last, bm2_sort_out *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts) || carry_len < 0 || carry_len >= BGZF_BLOCK || (carry_len && !carry)) {
        if (ctx) bm2_set_error(ctx, "bm2_bqsr_apply: bad arguments");
        return 1;
    }
    if (!ctx->bqa_set) { bm2_set_error(ctx, "bm2_bqsr_apply: no tables on this context (bm2_bqsr_apply_set)"); return 1; }
    for (int64_t i = 0, at = 0; i <= n_recs; ++i) {                  // whole records, each where the one before ends, the last at n
        if (i == n_recs) { if (at != n) { bm2_set_error(ctx, "bm2_bqsr_apply: the records do not end where the buffer ends"); return 1; } break; }
        const int64_t s = starts[i];
        if (s != at || s + 36 > n) { bm2_set_error(ctx, "bm2_bqsr_apply: record " + std::to_string(i) + " does not start where the one before ends"); return 1; }
        const BamFixed f = bam_fixed(recs + s);
        const int32_t l_seq = bam_le32(recs + s + 20);
        if (f.block_size < 32 || s + 4 + (int64_t) f.block_size > n || l_seq < 0 || f.l_read_name < 1 ||
            32 + (int64_t) f.l_read_name + 4 * (int64_t) f.n_cigar + (l_seq + 1) / 2 + (int64_t) l_seq > (int64_t) f.block_size) {
            bm2_set_error(ctx, "bm2_bqsr_apply: record " + std::to_string(i) + " is malformed");
            return 1;
        }
        at = s + 4 + f.block_size;
    }
    memset(out, 0, sizeof *out);
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->bqa_d;
    if (ctx->ensure(b[AP_STREAM], (size_t) (carry_len + n) + 16) || ctx->ensure(b[AP_STARTS], (size_t) n_recs * 8 + 8) ||
        ctx->ensure(b[AP_INFO], (size_t) n_recs * sizeof(bm2_sort_rec) + 8) ||
        ctx->ensure_host(ctx->bqa_h[AH_INFO], (size_t) n_recs * sizeof(bm2_sort_rec) + 16)) return 1;
    for (cudaEvent_t &ev : ctx->bqa_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    uint8_t *d_stream = (uint8_t *) b[AP_STREAM].p;
    bm2_sort_rec *h_info = (bm2_sort_rec *) ctx->bqa_h[AH_INFO].p;
    if (carry_len) BM2_CUDA_OK(cudaMemcpy(d_stream, carry, (size_t) carry_len, cudaMemcpyHostToDevice));   // carry may be this context's last carry
    unsigned long long cnt[CNT_END] = {0, 0, 0, ~0ULL};
    if (n_recs) {
        BM2_CUDA_OK(cudaMemcpyAsync(d_stream + carry_len, recs, (size_t) n, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[AP_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
        const int smem = (int) ctx->bqa_map_bytes;
        const int64_t g = bm2_min<int64_t>((n_recs + kWarps - 1) / kWarps, (int64_t) ctx->n_sm * 8);
        BM2_CUDA_OK(cudaEventRecord(ctx->bqa_ev[0], st));
        bqsr_apply_kernel<<<(unsigned) g, kWarps * 32, smem, st>>>(d_stream + carry_len, (const int64_t *) b[AP_STARTS].p, n_recs, (const int4 *) b[AP_MAP].p,
                                                                   smem, ctx->bqa_n_ids, (const double *) b[AP_P].p, (const double *) b[AP_CTX].p,
                                                                   (const double *) b[AP_CYC].p, (bm2_sort_rec *) b[AP_INFO].p,
                                                                   (unsigned long long *) b[AP_CNT].p, ctx->bqa_seen);
        BM2_CUDA_OK(cudaGetLastError());
        BM2_CUDA_OK(cudaEventRecord(ctx->bqa_ev[1], st));
        BM2_CUDA_OK(cudaMemcpyAsync(h_info, b[AP_INFO].p, (size_t) n_recs * sizeof(bm2_sort_rec), cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaMemcpyAsync(cnt, b[AP_CNT].p, sizeof cnt, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        float ms = 0;
        BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->bqa_ev[0], ctx->bqa_ev[1]));
        ctx->bqa_ms += ms;
    }
    const int64_t first = ctx->bqa_seen;
    ctx->bqa_seen += n_recs;
    if (cnt[CNT_ERR] != ~0ULL && !ctx->bqa_err_kind) {                 // a read error of this call: name it, write nothing
        const int64_t i = (int64_t) (cnt[CNT_ERR] >> 3) - first;
        ctx->bqa_err_kind = (int) (cnt[CNT_ERR] & 7) - BQSR_ERR_CYCLES + 1;
        ctx->bqa_err_index = (int64_t) (cnt[CNT_ERR] >> 3);
        const uint8_t *r = recs + starts[i];
        ctx->bqa_err_name.assign((const char *) r + 36, r[12] ? r[12] - 1 : 0);
        bm2_set_error(ctx, "bm2_bqsr_apply: read " + ctx->bqa_err_name + " " + kErrText[ctx->bqa_err_kind - 1]);
        return 1;
    }
    if (bam_compress_stream(ctx, d_stream, carry_len, starts, n_recs, n, last, h_info, nullptr, ctx->bqa_carry, ctx->bqa_recs, out)) return 1;
    ctx->bqa_bgzf_ms += ctx->bgzf_ms;
    return 0;
}

extern "C" int bm2_last_bqsr_apply_stats(bm2_ctx *ctx, bm2_bqsr_apply_stats_t *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out) { if (ctx) bm2_set_error(ctx, "bm2_last_bqsr_apply_stats: bad arguments"); return 1; }
    if (!ctx->bqa_set) { bm2_set_error(ctx, "bm2_last_bqsr_apply_stats: no tables on this context (bm2_bqsr_apply_set)"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    unsigned long long cnt[CNT_END];
    BM2_CUDA_OK(cudaMemcpy(cnt, ctx->bqa_d[AP_CNT].p, sizeof cnt, cudaMemcpyDeviceToHost));
    out->apply_ms = ctx->bqa_ms; out->bgzf_ms = ctx->bqa_bgzf_ms;
    out->bases_changed = (int64_t) cnt[CNT_CHANGED]; out->recal_records = (int64_t) cnt[CNT_RECAL]; out->kept_records = (int64_t) cnt[CNT_KEPT];
    out->err_kind = ctx->bqa_err_kind; out->err_index = ctx->bqa_err_index; out->err_name = ctx->bqa_err_name.c_str();
    return 0;
}

extern "C" int bm2_bqsr_apply_memory(const bm2_ctx *ctx, int64_t window_bytes, int32_t n_rg, int64_t *needed, int64_t *free_bytes) {
    if (!ctx || window_bytes < 0 || n_rg < 0 || !needed || !free_bytes) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // each rounded up by 1.25 as bm2_ctx::ensure allocates: the stream (carry + window), the BGZF slots (one 64 KiB slot per 65280-byte block)
    // and the gathered members (at most the slots' bytes, in practice far less), 32 bytes per record of starts and index data, the tables
    const double w = (double) window_bytes, slots = (w / BGZF_BLOCK + 2) * BGZF_MAX_MEMBER;
    const double tables = (double) n_rg * BQSR_NQ * (1 + BQSR_NCTX + BQSR_NCYC) * 8;
    const double bytes = 1.25 * ((w + BGZF_BLOCK) + 2 * slots + 32 * (w / kRecBytes + 1) + tables + kMapMax) + 64.0 * (1 << 20);
    size_t fr = 0, tot = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
    *needed = (int64_t) bytes; *free_bytes = (int64_t) fr;
    return 0;
}

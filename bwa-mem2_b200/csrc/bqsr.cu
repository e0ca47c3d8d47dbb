// bqsr.cu — the covariate counts of bm2_mem --recal-file and bm2_baserecalibrator on the GPU (bqsr_device.cuh's rule).
//   bm2_bqsr_sites    the known-site bitsets ("covered", "junction p|p+1 inside one record"), the .amb holes and the read group to the context;
//                     zeroes the counts and arms counting: from then on bm2_bam_sort_compress_ex counts the records it sorts (bam_sort.cu)
//   bm2_bqsr_count    counts one buffer of records from the host (what the tests compare with the host emulation)
//   bm2_bqsr_tables   the counts as dense tables, the reads and bases counted, the device time, the first read error
// The kernel: one warp per record, grid-stride.  Every lane prepares the record (fixed fields, filters, clipping bounds: the same loads, so
// broadcast), the low-quality tails come from ballots over the qualities, then the warp walks the CIGAR one op at a time with the lanes on
// consecutive bases.  Each base's (quality, context) count goes to a per-CTA table in shared memory, one atomic per group of lanes with the
// same key (__match_any_sync); its (quality, cycle) count, a table of 94 x 1001 too large for shared memory, goes to global memory with
// the same warp aggregation.  Each CTA flushes its shared table once into the 64-bit global counters.  The quality table is the sum of the
// cycle table over the cycles (every counted base has a cycle), taken on the host.  bm2_baserecalibrator (recal.cu) runs the same kernel
// with a read-group map: each record counts into the tables of its covariate, the (quality, context) ones in shared memory up to
// kBqsrSharedCovMax covariates and in global memory above; bm2_mem's path is one covariate and no map.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "bqsr_device.cuh"
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr unsigned kFull = 0xFFFFFFFFu;

// cnt: kBqsrCounts 64-bit counters per covariate (bqsr_count_launch).  map: n_ids BqsrRgEntry {offset of the ID's bytes, length, covariate, 0},
// then the bytes; n_ids 0: no lookup, every record is of covariate 0.  shared_cx: the n_cov (quality, context) tables sit in dynamic shared
// memory, before the map, and are flushed once per CTA; else they are counted in global memory with the same warp aggregation.
__global__ void __launch_bounds__(kWarps * 32) bqsr_count_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                                 BqsrView v, const int4 *__restrict__ map, int map_bytes, int n_ids, int n_cov,
                                                                 bool shared_cx, unsigned long long *cnt, unsigned long long *err, int64_t first) {
    extern __shared__ unsigned long long s_dyn[];
    const int n_s = shared_cx ? n_cov * kBqsrCxTab : 0;
    int4 *s_map = (int4 *) (s_dyn + n_s);
    for (int i = threadIdx.x; i < n_s; i += blockDim.x) s_dyn[i] = 0;
    for (int i = threadIdx.x; i < map_bytes / 16; i += blockDim.x) s_map[i] = map[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    int cur = 0;                                                        // the covariate whose reads and bases the warp is summing
    unsigned long long reads = 0, bases = 0;
    auto flush = [&]() {
        unsigned long long b = bases;
        for (int o = 16; o; o >>= 1) b += __shfl_xor_sync(kFull, b, o);
        if (lane == 0 && reads) {
            atomicAdd(&cnt[(int64_t) cur * kBqsrCounts + kBqsrReads], reads);
            atomicAdd(&cnt[(int64_t) cur * kBqsrCounts + kBqsrBases], b);
        }
        reads = 0; bases = 0;
    };
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const uint8_t *rec = base + starts[w];
        BqsrRec r;
        bqsr_prep(rec, v, r);
        int cov = 0;
        if (n_ids && r.status != BQSR_FILTERED) {                       // the read group, before the read errors
            int32_t len = 0, at = -1;
            if (lane == 0) at = bqsr_aux_rg(rec, &len);
            at = __shfl_sync(kFull, at, 0); len = __shfl_sync(kFull, len, 0);
            const int j = at >= 0 ? bqsr_rg_lookup((const BqsrRgEntry *) s_map, n_ids, rec, at, len) : -1;
            if (j >= 0) cov = s_map[j].z;
            else r.status = at < 0 ? BQSR_ERR_NORG : BQSR_ERR_BADRG;
        }
        if (r.status == BQSR_COUNT) {                                   // the low-quality tails and the quality check, 32 bases at a time
            int32_t tl = r.hi, tr = r.hi;
            bool bad = false;
            for (int32_t k0 = r.lo; k0 < r.hi; k0 += 32) {
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
            if (lane == 0) atomicMin(err, (unsigned long long) (first + w) << 3 | (unsigned) r.status);
            continue;
        }
        if (r.status != BQSR_COUNT) continue;
        if (cov != cur) { flush(); cur = cov; }
        reads += lane == 0;
        unsigned long long *const t_cx = shared_cx ? s_dyn + (int64_t) cov * kBqsrCxTab : cnt + (int64_t) cov * kBqsrCounts;
        unsigned long long *const t_cy = cnt + (int64_t) cov * kBqsrCounts;
        int32_t k = 0; int64_t g = r.g0;
        for (int c = 0; c < r.n_cigar; ++c) {
            const uint32_t o = bqsr_cig(r.cig, c), op = o & 15, len = o >> 4;
            const bool al = op == 0 || op == 7 || op == 8, ins = op == 1;
            if (al || ins) {
                const int32_t a = bm2_max(k, r.lo), b = bm2_min(k + (int32_t) len, r.hi);
                for (int32_t k0 = a; k0 < b; k0 += 32) {
                    const int32_t kk = k0 + lane;
                    int q = 0, cx = -1, cyc = 0, er = 0;
                    const bool ok = kk < b && bqsr_base(r, v, kk, ins, ins ? g - 1 : g + (kk - k), q, cx, cyc, er);
                    bases += ok;
                    const unsigned em = __ballot_sync(kFull, ok && er);
                    const int key = ok && cx >= 0 ? q * BQSR_NCTX + cx : -1;
                    unsigned grp = __match_any_sync(kFull, key);
                    if (key >= 0 && lane == __ffs(grp) - 1) {
                        atomicAdd(&t_cx[kBqsrCxObs + key], (unsigned long long) __popc(grp));
                        if (em & grp) atomicAdd(&t_cx[kBqsrCxErr + key], (unsigned long long) __popc(em & grp));
                    }
                    const int key2 = ok ? q * BQSR_NCYC + cyc + BQSR_MAX_CYCLE : -1;
                    grp = __match_any_sync(kFull, key2);
                    if (key2 >= 0 && lane == __ffs(grp) - 1) {
                        atomicAdd(&t_cy[kBqsrCyObs + key2], (unsigned long long) __popc(grp));
                        if (em & grp) atomicAdd(&t_cy[kBqsrCyErr + key2], (unsigned long long) __popc(em & grp));
                    }
                }
            }
            if (al || ins || op == 4) k += (int32_t) len;
            if (al || op == 2 || op == 3) g += len;
        }
    }
    flush();
    __syncthreads();
    for (int i = threadIdx.x; i < n_s; i += blockDim.x)
        if (s_dyn[i]) atomicAdd(&cnt[(int64_t) (i / kBqsrCxTab) * kBqsrCounts + i % kBqsrCxTab], s_dyn[i]);
}

enum { BQ_COVERED, BQ_JUNCTION, BQ_HOLES, BQ_COUNTS, BQ_ERR, BQ_IN, BQ_STARTS, BQ_END };
static_assert(BQ_END == std::extent<decltype(bm2_ctx::bqsr_d)>::value, "bm2_ctx::bqsr_d: one buffer per slot");

const char *const kErrText[3] = {"has no base qualities", "is longer than 500 cycles after clipping", "has a base quality above 93"};

}  // namespace

int bqsr_count_launch(bm2_ctx *ctx, const uint8_t *d_base, const int64_t *d_starts, int64_t n, const BqsrView &v, const void *d_map, int map_bytes,
                      int n_ids, int n_cov, unsigned long long *cnt, unsigned long long *err, int64_t first, cudaStream_t st) {
    bm2_ctx *ctx_for_error = ctx;
    if (!n) return 0;
    const bool shared_cx = n_cov <= kBqsrSharedCovMax;
    const int smem = (shared_cx ? n_cov * kBqsrCxTab * 8 : 0) + map_bytes;
    if (smem > 48 * 1024)                                               // the opt-in above 48 KB (shared tables beside a large map)
        BM2_CUDA_OK(cudaFuncSetAttribute(bqsr_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int64_t g = bm2_min<int64_t>((n + kWarps - 1) / kWarps, (int64_t) ctx->n_sm * 8);
    bqsr_count_kernel<<<(unsigned) g, kWarps * 32, smem, st>>>(d_base, d_starts, n, v, (const int4 *) d_map, map_bytes, n_ids, n_cov, shared_cx, cnt,
                                                               err, first);
    BM2_CUDA_OK(cudaGetLastError());
    return 0;
}

int bqsr_count_device(bm2_ctx *ctx, const uint8_t *d_base, const int64_t *d_starts, int64_t n, cudaStream_t st) {
    bm2_ctx *ctx_for_error = ctx;
    DevBuf *b = ctx->bqsr_d;
    for (cudaEvent_t &ev : ctx->bqsr_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    BqsrView v;
    v.ref = ctx->idx.ref; v.pac = nullptr; v.ann_off = ctx->idx.ann_off; v.n_seqs = ctx->idx.n_seqs; v.l_pac = ctx->idx.l_pac;
    v.covered = (const uint64_t *) b[BQ_COVERED].p; v.junction = (const uint64_t *) b[BQ_JUNCTION].p;
    v.holes = (const int64_t *) b[BQ_HOLES].p; v.n_holes = ctx->bqsr_n_holes;
    BM2_CUDA_OK(cudaEventRecord(ctx->bqsr_ev[0], st));
    if (bqsr_count_launch(ctx, d_base, d_starts, n, v, nullptr, 0, 0, 1, (unsigned long long *) b[BQ_COUNTS].p, (unsigned long long *) b[BQ_ERR].p,
                          ctx->bqsr_seen, st)) return 1;
    BM2_CUDA_OK(cudaEventRecord(ctx->bqsr_ev[1], st));
    BM2_CUDA_OK(cudaMemcpyAsync(&ctx->bqsr_err_word, b[BQ_ERR].p, 8, cudaMemcpyDeviceToHost, st));
    return 0;
}

int bqsr_count_done(bm2_ctx *ctx, const uint8_t *d_base, const int64_t *h_starts, int64_t n) {
    bm2_ctx *ctx_for_error = ctx;
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->bqsr_ev[0], ctx->bqsr_ev[1]));
    ctx->bqsr_ms += ms;
    const uint64_t e = ctx->bqsr_err_word;
    const int64_t first = ctx->bqsr_seen;
    ctx->bqsr_seen += n;
    if (e == ~(uint64_t) 0 || ctx->bqsr_err_kind) return 0;
    const int64_t i = (int64_t) (e >> 3) - first;
    ctx->bqsr_err_kind = (int) (e & 7) - BQSR_ERR_NOQUAL + 1;
    ctx->bqsr_err_index = (int64_t) (e >> 3);
    uint8_t h[36]; char name[256];
    const uint8_t *r = d_base + h_starts[i];
    BM2_CUDA_OK(cudaMemcpy(h, r, 36, cudaMemcpyDeviceToHost));
    BM2_CUDA_OK(cudaMemcpy(name, r + 36, h[12], cudaMemcpyDeviceToHost));
    name[h[12] ? h[12] - 1 : 0] = 0;
    ctx->bqsr_err_name = name;
    bm2_set_error(ctx, std::string("bm2_bqsr: read ") + name + " " + kErrText[ctx->bqsr_err_kind - 1]);
    return 1;
}

extern "C" int bm2_bqsr_sites(bm2_ctx *ctx, const uint64_t *covered, const uint64_t *junction, int64_t n_bits, const int64_t *holes, int64_t n_holes,
                              const char *rg) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !covered || !junction || n_holes < 0 || (n_holes && !holes) || !rg) { if (ctx) bm2_set_error(ctx, "bm2_bqsr_sites: bad arguments"); return 1; }
    if (!ctx->idx.loaded || n_bits != ctx->idx.l_pac) {
        bm2_set_error(ctx, "bm2_bqsr_sites: the bitsets must have one bit per base of the context's index (" + std::to_string(ctx->idx.l_pac) + ")");
        return 1;
    }
    for (int64_t h = 0; h < n_holes; ++h)
        if (holes[2 * h] < 0 || holes[2 * h + 1] < holes[2 * h] || holes[2 * h + 1] > n_bits || (h && holes[2 * h] < holes[2 * h - 1])) {
            bm2_set_error(ctx, "bm2_bqsr_sites: the holes must be sorted [beg, end) ranges inside the reference"); return 1;
        }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->bqsr_d;
    const size_t words = (size_t) ((n_bits + 63) / 64) * 8, need = 2 * words + (size_t) kBqsrCounts * 8 + (size_t) n_holes * 16;
    if (b[BQ_COVERED].cap < words + 8) {
        size_t fr = 0, tot = 0;
        BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
        if (need > fr) {
            bm2_set_error(ctx, "bm2_bqsr_sites: the known-site bitsets need " + std::to_string(need) + " bytes of device memory, " + std::to_string(fr) +
                               " bytes free");
            return 1;
        }
    }
    if (ctx->ensure(b[BQ_COVERED], words + 8) || ctx->ensure(b[BQ_JUNCTION], words + 8) || ctx->ensure(b[BQ_HOLES], (size_t) n_holes * 16 + 16) ||
        ctx->ensure(b[BQ_COUNTS], (size_t) kBqsrCounts * 8) || ctx->ensure(b[BQ_ERR], 8)) return 1;
    BM2_CUDA_OK(cudaMemcpy(b[BQ_COVERED].p, covered, words, cudaMemcpyHostToDevice));
    BM2_CUDA_OK(cudaMemcpy(b[BQ_JUNCTION].p, junction, words, cudaMemcpyHostToDevice));
    if (n_holes) BM2_CUDA_OK(cudaMemcpy(b[BQ_HOLES].p, holes, (size_t) n_holes * 16, cudaMemcpyHostToDevice));
    BM2_CUDA_OK(cudaMemset(b[BQ_COUNTS].p, 0, (size_t) kBqsrCounts * 8));
    BM2_CUDA_OK(cudaMemset(b[BQ_ERR].p, 0xff, 8));
    ctx->bqsr_n_holes = n_holes; ctx->bqsr_rg = rg;
    ctx->bqsr_seen = 0; ctx->bqsr_ms = 0; ctx->bqsr_err_kind = 0; ctx->bqsr_err_index = -1; ctx->bqsr_err_name.clear();
    ctx->bqsr_armed = true;
    return 0;
}

extern "C" int bm2_bqsr_count(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts)) { if (ctx) bm2_set_error(ctx, "bm2_bqsr_count: bad arguments"); return 1; }
    if (!ctx->bqsr_armed) { bm2_set_error(ctx, "bm2_bqsr_count: no known sites on this context (bm2_bqsr_sites)"); return 1; }
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t s = starts[i];
        if (s < 0 || s + 36 > n || s + 4 + (int64_t) bqsr_le32(recs + s) > n || bqsr_le32(recs + s) < 32) {
            bm2_set_error(ctx, "bm2_bqsr_count: record " + std::to_string(i) + " is not inside the buffer"); return 1;
        }
    }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->bqsr_d;
    if (ctx->ensure(b[BQ_IN], (size_t) n + 16) || ctx->ensure(b[BQ_STARTS], (size_t) n_recs * 8 + 8)) return 1;
    cudaStream_t st = ctx->stream;
    if (n) BM2_CUDA_OK(cudaMemcpyAsync(b[BQ_IN].p, recs, (size_t) n, cudaMemcpyHostToDevice, st));
    if (n_recs) BM2_CUDA_OK(cudaMemcpyAsync(b[BQ_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
    if (bqsr_count_device(ctx, (const uint8_t *) b[BQ_IN].p, (const int64_t *) b[BQ_STARTS].p, n_recs, st)) return 1;
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    bqsr_count_done(ctx, (const uint8_t *) b[BQ_IN].p, starts, n_recs);   // a read error is reported by bm2_bqsr_tables
    return 0;
}

extern "C" int bm2_bqsr_tables(bm2_ctx *ctx, bm2_bqsr_tables_t *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out) { if (ctx) bm2_set_error(ctx, "bm2_bqsr_tables: bad arguments"); return 1; }
    if (!ctx->bqsr_armed) { bm2_set_error(ctx, "bm2_bqsr_tables: no known sites on this context (bm2_bqsr_sites)"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    std::vector<int64_t> &t = ctx->bqsr_tables;
    t.assign((size_t) (kBqsrCounts + 2 * BQSR_NQ), 0);
    BM2_CUDA_OK(cudaMemcpy(t.data(), ctx->bqsr_d[BQ_COUNTS].p, (size_t) kBqsrCounts * 8, cudaMemcpyDeviceToHost));
    int64_t *qo = t.data() + kBqsrCounts, *qe = qo + BQSR_NQ;
    for (int q = 0; q < BQSR_NQ; ++q)
        for (int y = 0; y < BQSR_NCYC; ++y) { qo[q] += t[(size_t) (kBqsrCyObs + q * BQSR_NCYC + y)]; qe[q] += t[(size_t) (kBqsrCyErr + q * BQSR_NCYC + y)]; }
    out->qual_obs = qo; out->qual_err = qe;
    out->ctx_obs = t.data() + kBqsrCxObs; out->ctx_err = t.data() + kBqsrCxErr;
    out->cyc_obs = t.data() + kBqsrCyObs; out->cyc_err = t.data() + kBqsrCyErr;
    out->reads = t[kBqsrReads]; out->bases = t[kBqsrBases];
    out->ms = ctx->bqsr_ms;
    out->err_kind = ctx->bqsr_err_kind; out->err_index = ctx->bqsr_err_index;
    out->err_name = ctx->bqsr_err_name.c_str();
    out->read_group = ctx->bqsr_rg.c_str();
    return 0;
}

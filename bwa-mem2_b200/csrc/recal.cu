// recal.cu — the covariate counts of bm2_baserecalibrator on the GPU: GATK BaseRecalibrator's table of BAM files with several read groups,
// counted by bqsr.cu's kernel (bqsr_device.cuh's rule) with a read-group map.
//   bm2_recal_memory  the device bytes for a reference, a window and the covariates
//   bm2_recal_set     the contigs, the packed reference (2 bits per base), the .amb holes, the known-site bitsets and the read-group map
//                     (each @RG ID and its covariate) to the context; zeroes the counts
//   bm2_recal_add     one window: the records are checked to lie inside their contigs on the host, uploaded and counted, each into the
//                     tables of its covariate; a read error (bqsr_device.cuh's five) fails the call with an error naming the read
//   bm2_recal_tables  one covariate's dense tables, its reads and bases, the device time and the first read error
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "bqsr_recal.h"
#include <vector>

namespace {

enum { RC_PAC, RC_OFF, RC_COVERED, RC_JUNCTION, RC_HOLES, RC_MAP, RC_COUNTS, RC_ERR, RC_IN, RC_STARTS, RC_END };
static_assert(RC_END == std::extent<decltype(bm2_ctx::rcl_d)>::value, "bm2_ctx::rcl_d: one buffer per slot");

constexpr int kRecBytes = 300;              // a short read's record, for bm2_recal_memory's estimate

const char *const kErrText[5] = {"has no base qualities", "is longer than 500 cycles after clipping", "has a base quality above 93",
                                 "has no RG tag", "has an RG tag that is not an @RG ID of the headers"};

}  // namespace

extern "C" int bm2_recal_memory(const bm2_ctx *ctx, int64_t l_pac, int64_t window_bytes, int32_t n_cov, int64_t *needed, int64_t *free_bytes) {
    if (!ctx || l_pac < 0 || window_bytes < 0 || n_cov < 1 || !needed || !free_bytes) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // each rounded up by 1.25 as bm2_ctx::ensure allocates: the packed reference, the two bitsets, the counters, the window and 8 bytes of
    // starts per record; the holes and the map are small
    const double ref = (double) l_pac / 4 + 2.0 * ((double) l_pac / 8), w = (double) window_bytes;
    const double bytes = 1.25 * (ref + (double) n_cov * kBqsrCounts * 8 + w + 8 * (w / kRecBytes + 1) + kBqsrMapMax) + 64.0 * (1 << 20);
    size_t fr = 0, tot = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
    *needed = (int64_t) bytes; *free_bytes = (int64_t) fr;
    return 0;
}

extern "C" int bm2_recal_set(bm2_ctx *ctx, const bm2_recal_set_t *s) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !s || s->n_contigs < 1 || !s->contig_off || !s->contig_len || s->l_pac < 1 || !s->pac || s->n_holes < 0 || (s->n_holes && !s->holes) ||
        !s->covered || !s->junction || s->n_ids < 0 || (s->n_ids && (!s->ids || !s->id_cov)) || s->n_cov < 1) {
        if (ctx) bm2_set_error(ctx, "bm2_recal_set: bad arguments");
        return 1;
    }
    for (int32_t c = 0; c < s->n_contigs; ++c)
        if (s->contig_off[c] < 0 || s->contig_len[c] < 0 || s->contig_off[c] + s->contig_len[c] > s->l_pac) {
            bm2_set_error(ctx, "bm2_recal_set: contig " + std::to_string(c) + " is not inside the reference"); return 1;
        }
    for (int64_t h = 0; h < s->n_holes; ++h)
        if (s->holes[2 * h] < 0 || s->holes[2 * h + 1] < s->holes[2 * h] || s->holes[2 * h + 1] > s->l_pac || (h && s->holes[2 * h] < s->holes[2 * h - 1])) {
            bm2_set_error(ctx, "bm2_recal_set: the holes must be sorted [beg, end) ranges inside the reference"); return 1;
        }
    std::vector<std::string> ids;
    std::vector<int32_t> vals;
    for (int32_t i = 0; i < s->n_ids; ++i) {
        if (!s->ids[i] || s->id_cov[i] < 0 || s->id_cov[i] >= s->n_cov) { bm2_set_error(ctx, "bm2_recal_set: a bad read-group entry"); return 1; }
        ids.push_back(s->ids[i]); vals.push_back(s->id_cov[i]);
    }
    std::vector<uint8_t> blob;
    const std::string e = bqsr_rg_map(ids, vals, blob);
    if (!e.empty()) { bm2_set_error(ctx, "bm2_recal_set: " + e); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->rcl_d;
    const size_t pac = (size_t) (s->l_pac + 3) / 4, words = (size_t) ((s->l_pac + 63) / 64) * 8, counts = (size_t) s->n_cov * kBqsrCounts * 8;
    if (b[RC_PAC].cap < pac + 8) {
        size_t fr = 0, tot = 0;
        BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
        const size_t need = pac + 2 * words + counts;
        if (need > fr) {
            bm2_set_error(ctx, "bm2_recal_set: the reference and the known-site bitsets need " + std::to_string(need) + " bytes of device memory, " +
                               std::to_string(fr) + " bytes free");
            return 1;
        }
    }
    if (ctx->ensure(b[RC_PAC], pac + 8) || ctx->ensure(b[RC_OFF], (size_t) s->n_contigs * 8) || ctx->ensure(b[RC_COVERED], words + 8) ||
        ctx->ensure(b[RC_JUNCTION], words + 8) || ctx->ensure(b[RC_HOLES], (size_t) s->n_holes * 16 + 16) || ctx->ensure(b[RC_MAP], blob.size() + 16) ||
        ctx->ensure(b[RC_COUNTS], counts) || ctx->ensure(b[RC_ERR], 8)) return 1;
    BM2_CUDA_OK(cudaMemcpy(b[RC_PAC].p, s->pac, pac, cudaMemcpyHostToDevice));
    BM2_CUDA_OK(cudaMemcpy(b[RC_OFF].p, s->contig_off, (size_t) s->n_contigs * 8, cudaMemcpyHostToDevice));
    BM2_CUDA_OK(cudaMemcpy(b[RC_COVERED].p, s->covered, words, cudaMemcpyHostToDevice));
    BM2_CUDA_OK(cudaMemcpy(b[RC_JUNCTION].p, s->junction, words, cudaMemcpyHostToDevice));
    if (s->n_holes) BM2_CUDA_OK(cudaMemcpy(b[RC_HOLES].p, s->holes, (size_t) s->n_holes * 16, cudaMemcpyHostToDevice));
    if (!blob.empty()) BM2_CUDA_OK(cudaMemcpy(b[RC_MAP].p, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    BM2_CUDA_OK(cudaMemset(b[RC_COUNTS].p, 0, counts));
    BM2_CUDA_OK(cudaMemset(b[RC_ERR].p, 0xff, 8));
    ctx->rcl_contig_len.assign(s->contig_len, s->contig_len + s->n_contigs);
    ctx->rcl_l_pac = s->l_pac; ctx->rcl_n_holes = s->n_holes; ctx->rcl_n_ids = s->n_ids; ctx->rcl_n_cov = s->n_cov;
    ctx->rcl_map_bytes = (int64_t) blob.size();
    ctx->rcl_seen = 0; ctx->rcl_ms = 0; ctx->rcl_err_kind = 0; ctx->rcl_err_index = -1; ctx->rcl_err_name.clear();
    ctx->rcl_set = true;
    return 0;
}

extern "C" int bm2_recal_add(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts)) { if (ctx) bm2_set_error(ctx, "bm2_recal_add: bad arguments"); return 1; }
    if (!ctx->rcl_set) { bm2_set_error(ctx, "bm2_recal_add: no reference on this context (bm2_recal_set)"); return 1; }
    const int32_t n_seqs = (int32_t) ctx->rcl_contig_len.size();
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t s = starts[i];
        const uint8_t *r = recs + s;
        if (s < 0 || s + 36 > n || bqsr_le32(r) < 32 || s + 4 + (int64_t) bqsr_le32(r) > n || bqsr_le32(r + 20) < 0 || r[12] < 1 ||
            32 + (int64_t) r[12] + 4 * (int64_t) (r[16] | r[17] << 8) + (bqsr_le32(r + 20) + 1) / 2 + (int64_t) bqsr_le32(r + 20) > (int64_t) bqsr_le32(r)) {
            bm2_set_error(ctx, "bm2_recal_add: record " + std::to_string(i) + " is not inside the buffer"); return 1;
        }
        if (bqsr_outside_contig(r, ctx->rcl_contig_len.data(), n_seqs)) {
            bm2_set_error(ctx, "bm2_recal_add: read " + std::string((const char *) r + 36, r[12] - 1) + " is malformed: its alignment is not inside contig " +
                               std::to_string(bqsr_le32(r + 4)));
            return 2;
        }
    }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->rcl_d;
    if (ctx->ensure(b[RC_IN], (size_t) n + 16) || ctx->ensure(b[RC_STARTS], (size_t) n_recs * 8 + 8)) return 1;
    for (cudaEvent_t &ev : ctx->rcl_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    cudaStream_t st = ctx->stream;
    if (n) BM2_CUDA_OK(cudaMemcpyAsync(b[RC_IN].p, recs, (size_t) n, cudaMemcpyHostToDevice, st));
    if (n_recs) BM2_CUDA_OK(cudaMemcpyAsync(b[RC_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
    BqsrView v;
    v.ref = nullptr; v.pac = (const uint8_t *) b[RC_PAC].p; v.ann_off = (const int64_t *) b[RC_OFF].p; v.n_seqs = n_seqs; v.l_pac = ctx->rcl_l_pac;
    v.covered = (const uint64_t *) b[RC_COVERED].p; v.junction = (const uint64_t *) b[RC_JUNCTION].p;
    v.holes = (const int64_t *) b[RC_HOLES].p; v.n_holes = ctx->rcl_n_holes;
    BM2_CUDA_OK(cudaEventRecord(ctx->rcl_ev[0], st));
    if (bqsr_count_launch(ctx, (const uint8_t *) b[RC_IN].p, (const int64_t *) b[RC_STARTS].p, n_recs, v, b[RC_MAP].p, (int) ctx->rcl_map_bytes,
                          ctx->rcl_n_ids, ctx->rcl_n_cov, (unsigned long long *) b[RC_COUNTS].p, (unsigned long long *) b[RC_ERR].p, ctx->rcl_seen, st))
        return 1;
    BM2_CUDA_OK(cudaEventRecord(ctx->rcl_ev[1], st));
    uint64_t e = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&e, b[RC_ERR].p, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->rcl_ev[0], ctx->rcl_ev[1]));
    ctx->rcl_ms += ms;
    const int64_t first = ctx->rcl_seen;
    ctx->rcl_seen += n_recs;
    if (e == ~(uint64_t) 0) return 0;
    if (!ctx->rcl_err_kind) {
        const int64_t i = (int64_t) (e >> 3) - first;
        ctx->rcl_err_kind = (int) (e & 7) - BQSR_ERR_NOQUAL + 1;
        ctx->rcl_err_index = (int64_t) (e >> 3);
        const uint8_t *r = recs + starts[i];
        ctx->rcl_err_name.assign((const char *) r + 36, r[12] - 1);
    }
    bm2_set_error(ctx, "bm2_recal_add: read " + ctx->rcl_err_name + " " + kErrText[ctx->rcl_err_kind - 1]);
    return 2;
}

extern "C" int bm2_recal_tables(bm2_ctx *ctx, int32_t cov, bm2_bqsr_tables_t *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out) { if (ctx) bm2_set_error(ctx, "bm2_recal_tables: bad arguments"); return 1; }
    if (!ctx->rcl_set) { bm2_set_error(ctx, "bm2_recal_tables: no reference on this context (bm2_recal_set)"); return 1; }
    if (cov < 0 || cov >= ctx->rcl_n_cov) { bm2_set_error(ctx, "bm2_recal_tables: covariate " + std::to_string(cov) + " out of range"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    std::vector<int64_t> &t = ctx->rcl_tables;
    t.assign((size_t) (kBqsrCounts + 2 * BQSR_NQ), 0);
    BM2_CUDA_OK(cudaMemcpy(t.data(), (const uint64_t *) ctx->rcl_d[RC_COUNTS].p + (int64_t) cov * kBqsrCounts, (size_t) kBqsrCounts * 8,
                           cudaMemcpyDeviceToHost));
    int64_t *qo = t.data() + kBqsrCounts, *qe = qo + BQSR_NQ;
    for (int q = 0; q < BQSR_NQ; ++q)
        for (int y = 0; y < BQSR_NCYC; ++y) { qo[q] += t[(size_t) (kBqsrCyObs + q * BQSR_NCYC + y)]; qe[q] += t[(size_t) (kBqsrCyErr + q * BQSR_NCYC + y)]; }
    out->qual_obs = qo; out->qual_err = qe;
    out->ctx_obs = t.data() + kBqsrCxObs; out->ctx_err = t.data() + kBqsrCxErr;
    out->cyc_obs = t.data() + kBqsrCyObs; out->cyc_err = t.data() + kBqsrCyErr;
    out->reads = t[kBqsrReads]; out->bases = t[kBqsrBases];
    out->ms = ctx->rcl_ms;
    out->err_kind = ctx->rcl_err_kind; out->err_index = ctx->rcl_err_index;
    out->err_name = ctx->rcl_err_name.c_str();
    out->read_group = "";
    return 0;
}

// cigar.cu — seam 3: CIGAR / NM / MD of a batch of alignments whose end points are known.
//
// Replaces bwa_gen_cigar2 (reference src/bwa.cpp:260-347) + ksw_global2 with backtrack (src/ksw.cpp:545-668) as
// mem_reg2aln calls them per output alignment (src/bwamem.cpp:1757-1768): SURVEY §8(f) item 2, the first widening
// step after the seed-chain-extend path.  One alignment per thread (cigar_device.cuh); the backtrack matrix of a thread
// is a byte column of a matrix interleaved over the threads of the launch (cell c of thread t at z[c * T + t]), the
// operations / MD strings go to worst-case stripes and are compacted by two scans + one gather.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "cigar_device.cuh"
#include <cub/device/device_scan.cuh>
#include <vector>
#include <climits>
#include <cstring>

namespace {
enum { CB_CODES, CB_OFFS, CB_REQS, CB_CAPOFF, CB_OPS_W, CB_MD_W, CB_RECS, CB_Z, CB_HE, CB_CNT, CB_SCAN, CB_CUB, CB_OPS, CB_MD, CB_COUNT_ };
enum { CH_RECS, CH_OPS, CH_MD, CH_COUNT_ };
static_assert(CB_COUNT_ == std::extent<decltype(bm2_ctx::cigar_d)>::value, "bm2_ctx::cigar_d: one buffer per slot");
static_assert(CH_COUNT_ == std::extent<decltype(bm2_ctx::cigar_h)>::value, "bm2_ctx::cigar_h: one buffer per slot");

struct CapOff { int64_t ops, md; };       // start of a request's worst-case stripes

__global__ void __launch_bounds__(128)
cigar_kernel(CigarParams p, int64_t l_pac, const uint8_t *__restrict__ ref, const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs,
             const bm2_cigar_req *__restrict__ reqs, int64_t n, const CapOff *__restrict__ cap, uint32_t *ops_w, char *md_w, bm2_cigar_rec *recs,
             uint8_t *zbuf, int32_t *he_all, int he_stride, int64_t *cnt_ops, int64_t *cnt_md)
{
    const long long T = (long long) gridDim.x * blockDim.x, t = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    CigarZ z = { zbuf + t, T };
    int32_t *he = he_all + t * he_stride;
    for (int64_t r = t; r < n; r += T) {
        const bm2_cigar_req q = reqs[r];
        const int lq = q.qe - q.qb;
        int score = INT_MIN, nc = 0, nm = -1, nmd = 0;
        gen_cigar_d(p, l_pac, ref, q.w, lq, codes + offs[q.read] + q.qb, q.rb, q.re, he, z, &score, ops_w + cap[r].ops, &nc, &nm, md_w + cap[r].md, &nmd);
        bm2_cigar_rec o; o.score = score; o.n_cigar = nc; o.nm = nm; o.n_md = nmd; o.cigar_off = 0; o.md_off = 0;
        recs[r] = o;
        cnt_ops[r] = nc; cnt_md[r] = nmd;
    }
}

__global__ void cigar_gather_kernel(int64_t n, const CapOff *__restrict__ cap, const uint32_t *__restrict__ ops_w, const char *__restrict__ md_w,
                                    const int64_t *__restrict__ off_ops, const int64_t *__restrict__ off_md, bm2_cigar_rec *recs, uint32_t *ops, char *md)
{
    const int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    bm2_cigar_rec o = recs[r];
    o.cigar_off = off_ops[r]; o.md_off = off_md[r];
    recs[r] = o;
    for (int k = 0; k < o.n_cigar; ++k) ops[o.cigar_off + k] = ops_w[cap[r].ops + k];
    for (int k = 0; k < o.n_md; ++k) md[o.md_off + k] = md_w[cap[r].md + k];
}

template <class T> T *P(bm2_ctx *ctx, int b) { return (T *) ctx->cigar_d[b].p; }

}  // namespace

extern "C" int bm2_gen_cigar(bm2_ctx *ctx, const bm2_read_batch *reads, const bm2_cigar_req *reqs, int64_t n, bm2_cigar_result *out)
{
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !reads || !out || (n > 0 && !reqs) || n < 0) { if (ctx) bm2_set_error(ctx, "bm2_gen_cigar: bad arguments"); return 1; }
    if (!ctx->idx.loaded) { bm2_set_error(ctx, "bm2_gen_cigar needs a context created with an index"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    memset(out, 0, sizeof(*out));
    if (ctx->ensure_host(ctx->cigar_h[CH_RECS], sizeof(bm2_cigar_rec)) || ctx->ensure_host(ctx->cigar_h[CH_OPS], 16) || ctx->ensure_host(ctx->cigar_h[CH_MD], 16)) return 1;
    out->recs = (const bm2_cigar_rec *) ctx->cigar_h[CH_RECS].p; out->cigar = (const uint32_t *) ctx->cigar_h[CH_OPS].p; out->md = (const char *) ctx->cigar_h[CH_MD].p;
    if (n == 0) return 0;
    CigarParams p; memcpy(p.mat, ctx->opt.mat, 25); p.o_del = ctx->opt.o_del; p.e_del = ctx->opt.e_del; p.o_ins = ctx->opt.o_ins; p.e_ins = ctx->opt.e_ins;
    if (p.e_del <= 0 || p.e_ins <= 0) { bm2_set_error(ctx, "bm2_gen_cigar: gap extension penalties must be positive"); return 1; }
    // worst-case output stripes and scratch sizes (host: the requests are here anyway)
    const int nr = reads->n_reads;
    std::vector<CapOff> cap((size_t) n + 1);
    int64_t ops_total = 0, md_total = 0; long long zcap = 1; int max_lq = 1;
    for (int64_t r = 0; r < n; ++r) {
        const bm2_cigar_req &q = reqs[r];
        if (q.read < 0 || q.read >= nr) { bm2_set_error(ctx, "bm2_gen_cigar: request names a read outside the batch"); return 1; }
        const int64_t rl = reads->offsets[q.read + 1] - reads->offsets[q.read];
        if (q.qb < 0 || q.qe > rl) { bm2_set_error(ctx, "bm2_gen_cigar: query interval outside its read"); return 1; }
        const int lq = q.qe > q.qb ? q.qe - q.qb : 0;
        const int64_t rlen = q.re > q.rb ? q.re - q.rb : 0;
        if (rlen > (int64_t) 1 << 24 || lq > 1 << 24) { bm2_set_error(ctx, "bm2_gen_cigar: alignment longer than 2^24"); return 1; }
        cap[(size_t) r].ops = ops_total; cap[(size_t) r].md = md_total;
        ops_total += lq + rlen + 2; md_total += 2 * (int64_t) lq + 7 * rlen + 16;
        const long long zc = cigar_z_cells_d(p, ctx->idx.l_pac, q.w, q.qe - q.qb, q.rb, q.re);
        if (zc > zcap) zcap = zc;
        if (lq > max_lq) max_lq = lq;
    }
    cap[(size_t) n].ops = ops_total; cap[(size_t) n].md = md_total;
    if ((size_t) ops_total * 4 + (size_t) md_total > (size_t) 48 << 30) { bm2_set_error(ctx, "bm2_gen_cigar: batch too large (worst-case output over 48 GB): use smaller batches"); return 1; }
    // threads of the launch: as many as the backtrack-matrix budget allows
    const long long z_budget = (long long) 8 << 30;
    if (zcap > z_budget / 128) { bm2_set_error(ctx, "bm2_gen_cigar: backtrack matrix of one alignment over 64 MB"); return 1; }
    long long T = z_budget / zcap / 128 * 128;
    const long long t_max = (long long) ctx->n_sm * 8 * 128, t_need = (n + 127) / 128 * 128;
    if (T > t_max) T = t_max;
    if (T > t_need) T = t_need;
    const int he_stride = 2 * (max_lq + 1);
    const int64_t total = reads->offsets[nr];
    if (ctx->ensure(ctx->cigar_d[CB_CODES], (size_t) total + 16) || ctx->ensure(ctx->cigar_d[CB_OFFS], (size_t) (nr + 1) * 8) ||
        ctx->ensure(ctx->cigar_d[CB_REQS], (size_t) n * sizeof(bm2_cigar_req)) || ctx->ensure(ctx->cigar_d[CB_CAPOFF], (size_t) (n + 1) * sizeof(CapOff)) ||
        ctx->ensure(ctx->cigar_d[CB_OPS_W], (size_t) ops_total * 4 + 16) || ctx->ensure(ctx->cigar_d[CB_MD_W], (size_t) md_total + 16) ||
        ctx->ensure(ctx->cigar_d[CB_RECS], (size_t) n * sizeof(bm2_cigar_rec)) || ctx->ensure(ctx->cigar_d[CB_Z], (size_t) (zcap * T) + 16) ||
        ctx->ensure(ctx->cigar_d[CB_HE], (size_t) T * he_stride * 4) || ctx->ensure(ctx->cigar_d[CB_CNT], (size_t) (n + 1) * 16) ||
        ctx->ensure(ctx->cigar_d[CB_SCAN], (size_t) (n + 1) * 16)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->cigar_d[CB_CODES].p, reads->codes, (size_t) total, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->cigar_d[CB_OFFS].p, reads->offsets, (size_t) (nr + 1) * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->cigar_d[CB_REQS].p, reqs, (size_t) n * sizeof(bm2_cigar_req), cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->cigar_d[CB_CAPOFF].p, cap.data(), (size_t) (n + 1) * sizeof(CapOff), cudaMemcpyHostToDevice, st));
    int64_t *cnt_ops = P<int64_t>(ctx, CB_CNT), *cnt_md = cnt_ops + (n + 1), *off_ops = P<int64_t>(ctx, CB_SCAN), *off_md = off_ops + (n + 1);
    BM2_CUDA_OK(cudaMemsetAsync(cnt_ops + n, 0, 8, st));
    BM2_CUDA_OK(cudaMemsetAsync(cnt_md + n, 0, 8, st));
    cigar_kernel<<<(unsigned) (T / 128), 128, 0, st>>>(p, ctx->idx.l_pac, ctx->idx.ref, P<uint8_t>(ctx, CB_CODES), P<int64_t>(ctx, CB_OFFS),
                                                      P<bm2_cigar_req>(ctx, CB_REQS), n, P<CapOff>(ctx, CB_CAPOFF), P<uint32_t>(ctx, CB_OPS_W),
                                                      P<char>(ctx, CB_MD_W), P<bm2_cigar_rec>(ctx, CB_RECS), P<uint8_t>(ctx, CB_Z),
                                                      P<int32_t>(ctx, CB_HE), he_stride, cnt_ops, cnt_md);
    size_t cub_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, cnt_ops, off_ops, (int) (n + 1));
    if (ctx->ensure(ctx->cigar_d[CB_CUB], cub_bytes)) return 1;
    BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->cigar_d[CB_CUB].p, cub_bytes, cnt_ops, off_ops, (int) (n + 1), st));
    BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->cigar_d[CB_CUB].p, cub_bytes, cnt_md, off_md, (int) (n + 1), st));
    int64_t tot[2] = {0, 0};
    BM2_CUDA_OK(cudaMemcpyAsync(&tot[0], off_ops + n, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&tot[1], off_md + n, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    if (ctx->ensure(ctx->cigar_d[CB_OPS], (size_t) tot[0] * 4 + 16) || ctx->ensure(ctx->cigar_d[CB_MD], (size_t) tot[1] + 16) ||
        ctx->ensure_host(ctx->cigar_h[CH_RECS], (size_t) n * sizeof(bm2_cigar_rec)) || ctx->ensure_host(ctx->cigar_h[CH_OPS], (size_t) tot[0] * 4 + 16) ||
        ctx->ensure_host(ctx->cigar_h[CH_MD], (size_t) tot[1] + 16)) return 1;
    cigar_gather_kernel<<<(unsigned) ((n + 127) / 128), 128, 0, st>>>(n, P<CapOff>(ctx, CB_CAPOFF), P<uint32_t>(ctx, CB_OPS_W), P<char>(ctx, CB_MD_W), off_ops,
                                                                      off_md, P<bm2_cigar_rec>(ctx, CB_RECS), P<uint32_t>(ctx, CB_OPS), P<char>(ctx, CB_MD));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->cigar_h[CH_RECS].p, ctx->cigar_d[CB_RECS].p, (size_t) n * sizeof(bm2_cigar_rec), cudaMemcpyDeviceToHost, st));
    if (tot[0]) BM2_CUDA_OK(cudaMemcpyAsync(ctx->cigar_h[CH_OPS].p, ctx->cigar_d[CB_OPS].p, (size_t) tot[0] * 4, cudaMemcpyDeviceToHost, st));
    if (tot[1]) BM2_CUDA_OK(cudaMemcpyAsync(ctx->cigar_h[CH_MD].p, ctx->cigar_d[CB_MD].p, (size_t) tot[1], cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaGetLastError());
    out->n = n; out->recs = (const bm2_cigar_rec *) ctx->cigar_h[CH_RECS].p;
    out->n_ops = tot[0]; out->cigar = (const uint32_t *) ctx->cigar_h[CH_OPS].p;
    out->n_md = tot[1]; out->md = (const char *) ctx->cigar_h[CH_MD].p;
    return 0;
}

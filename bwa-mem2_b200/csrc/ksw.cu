// ksw.cu — finer seam under seam 4: a batch of the local alignments of mate rescue, one window per warp.
//
// Replaces ksw_align2 (reference src/ksw.cpp:324-381 = ksw_u8 :111-233 / ksw_i16 :235-316 forward, then the same kernel on the reversed
// prefixes) as mem_matesw calls it (src/bwamem_pair.cpp:186-193), for a batch of (query, window) requests - the bring-up seam of the
// second version of bm2_sam_pe, as bm2_extend_pairs is for the extension kernel.  The arithmetic is ksw_warp.cuh (32 lanes split the
// query, two max-plus scans per row), checked on the host against the oracle and the reference's golden vectors.
//
// Parity: tests/test_zzz_ksw_gpu.py.  sam.cu's staged rescue launches the same arithmetic on a job table built on the device.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "ksw_warp.cuh"
#include <vector>
#include <cstring>

namespace {
enum { KB_SEQ, KB_REQ, KB_LISTOFF, KB_LIST, KB_RES, KB_OVF, KB_COUNT_ };
static_assert(KB_COUNT_ == std::extent<decltype(bm2_ctx::ksw_d)>::value, "bm2_ctx::ksw_d: one buffer per slot");
struct KswMat { int8_t m[25]; };

template <int TMAX>
__global__ void __launch_bounds__(128)
ksw_warp_kernel(KswMat mat, int o_del, int e_del, int o_ins, int e_ins, const uint8_t *__restrict__ seqs, const bm2_ksw_req *__restrict__ reqs, int64_t n,
                const int64_t *__restrict__ list_off, int32_t *lists, bm2_ksw_res *res, int *ovf)
{
    __shared__ int8_t smat[32];                               // the passes index the matrix with data (profile set-up): shared, not a local copy
    if (threadIdx.x < 25) smat[threadIdx.x] = mat.m[threadIdx.x];
    __syncthreads();
    const int64_t warps = (int64_t) gridDim.x * (blockDim.x >> 5);
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n; r += warps) {
        const bm2_ksw_req q = reqs[r];
        const int bcap = (int) ((list_off[r + 1] - list_off[r]) >> 1);
        int32_t *bsc = lists + list_off[r], *bpos = bsc + bcap;
        int overflow = 0;
        const KswRes a = ksw_align2_warp_d<TMAX>(q.qlen, seqs + q.qoff, 1, 0, q.tlen, seqs + q.toff, smat, o_del, e_del, o_ins, e_ins, q.xtra, bsc, bpos, bcap, &overflow);
        if (lane == 0) {
            bm2_ksw_res o; o.score = a.score; o.te = a.te; o.qe = a.qe; o.score2 = a.score2; o.te2 = a.te2; o.tb = a.tb; o.qb = a.qb; o._pad = 0;
            res[r] = o;
            if (overflow) atomicOr(ovf, overflow);
        }
        __syncwarp(0xffffffffu);
    }
}
template <class T> T *P(bm2_ctx *ctx, int b) { return (T *) ctx->ksw_d[b].p; }
}  // namespace

extern "C" int bm2_ksw_align2(bm2_ctx *ctx, const uint8_t *seqs, int64_t n_seq_bytes, const bm2_ksw_req *reqs, int64_t n, bm2_ksw_res *out)
{
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n < 0 || n_seq_bytes < 0 || (n > 0 && (!seqs || !reqs || !out))) { if (ctx) bm2_set_error(ctx, "bm2_ksw_align2: bad arguments"); return 1; }
    if (n == 0) return 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const bm2_mem_opt_t &o = ctx->opt;
    if (o.e_del <= 0 || o.e_ins <= 0) { bm2_set_error(ctx, "bm2_ksw_align2: gap extension penalties must be positive"); return 1; }
    std::vector<int64_t> list_off((size_t) n + 1);
    int64_t tot = 0;
    int max_qlen = 1;
    for (int64_t r = 0; r < n; ++r) {
        const bm2_ksw_req &q = reqs[r];
        if (q.qlen <= 0 || q.tlen <= 0 || q.qoff < 0 || q.toff < 0 || q.qoff + q.qlen > n_seq_bytes || q.toff + q.tlen > n_seq_bytes) {
            bm2_set_error(ctx, "bm2_ksw_align2: a request outside the sequence buffer"); return 1;
        }
        if (q.qlen > 32 * BM2_KSW_CMAX - 15) { bm2_set_error(ctx, "bm2_ksw_align2: queries longer than 497 bases are not supported by this entry point yet"); return 1; }
        if (!ksw_scan_ok_d(o.e_ins, q.qlen)) { bm2_set_error(ctx, "bm2_ksw_align2: gap extension penalty too large for this entry point (e_ins * qlen must stay below 2^20)"); return 1; }
        if (q.qlen > max_qlen) max_qlen = q.qlen;
        list_off[(size_t) r] = tot;
        tot += 2 * ((int64_t) q.tlen / 2 + 2);
    }
    list_off[(size_t) n] = tot;
    if (ctx->ensure(ctx->ksw_d[KB_SEQ], (size_t) n_seq_bytes + 16) || ctx->ensure(ctx->ksw_d[KB_REQ], (size_t) n * sizeof(bm2_ksw_req)) ||
        ctx->ensure(ctx->ksw_d[KB_LISTOFF], (size_t) (n + 1) * 8) || ctx->ensure(ctx->ksw_d[KB_LIST], (size_t) tot * 4 + 16) ||
        ctx->ensure(ctx->ksw_d[KB_RES], (size_t) n * sizeof(bm2_ksw_res)) || ctx->ensure(ctx->ksw_d[KB_OVF], 16)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->ksw_d[KB_SEQ].p, seqs, (size_t) n_seq_bytes, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->ksw_d[KB_REQ].p, reqs, (size_t) n * sizeof(bm2_ksw_req), cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->ksw_d[KB_LISTOFF].p, list_off.data(), (size_t) (n + 1) * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemsetAsync(ctx->ksw_d[KB_OVF].p, 0, 4, st));
    KswMat mat; memcpy(mat.m, o.mat, 25);
    const int64_t blocks_need = (n + 3) / 4, blocks_max = (int64_t) ctx->n_sm * 8;
    const unsigned grid = (unsigned) (blocks_need < blocks_max ? blocks_need : blocks_max);
    // the kernel instance whose lanes hold the longest query of the batch (151-bp reads: 5 columns per lane, all in registers)
#define BM2_KSW_LAUNCH(T) ksw_warp_kernel<T><<<grid, 128, 0, st>>>(mat, o.o_del, o.e_del, o.o_ins, o.e_ins, P<uint8_t>(ctx, KB_SEQ), P<bm2_ksw_req>(ctx, KB_REQ), n, \
                                         P<int64_t>(ctx, KB_LISTOFF), P<int32_t>(ctx, KB_LIST), P<bm2_ksw_res>(ctx, KB_RES), P<int>(ctx, KB_OVF))
    switch (ksw_kernel_width_d(max_qlen)) {
    case 5: BM2_KSW_LAUNCH(5); break;
    case 8: BM2_KSW_LAUNCH(8); break;
    default: BM2_KSW_LAUNCH(BM2_KSW_CMAX); break;
    }
#undef BM2_KSW_LAUNCH
    BM2_CUDA_OK(cudaGetLastError());
    int ovf = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(out, ctx->ksw_d[KB_RES].p, (size_t) n * sizeof(bm2_ksw_res), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&ovf, ctx->ksw_d[KB_OVF].p, 4, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    if (ovf) { bm2_set_error(ctx, "bm2_ksw_align2: score-2 list overflow (internal)"); return 1; }
    return 0;
}

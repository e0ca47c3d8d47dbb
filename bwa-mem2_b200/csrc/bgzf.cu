// bgzf.cu — BGZF compression on the GPU (bm2_bgzf_compress): uncompressed bytes and the record starts in, BGZF members out.
//
// BAM out of bm2_mem is about 300 MB/s of uncompressed records at the aligner's rate; single-thread zlib deflates tens of MB/s, so the
// host would need about ten cores to keep up.  Here the blocks are cut on the host by htslib's rule (bgzf_cut_blocks), and one CTA
// compresses one block at a time with the block staged in shared memory:
//   load        the block's bytes into shared memory
//   chain       warps 0-3: the hash chain prev[] of a quarter of the block each (32 positions per step: __match_any_sync finds the lanes
//               with the same hash, the highest earlier lane or the quarter's head table gives prev); warps 4-7 meanwhile: CRC32 of
//               256-byte pieces, combined by multiplication modulo the CRC polynomial.  Then every thread links the positions that
//               start a quarter's chain to the heads of the earlier quarters.
//   parse       thread t: greedy LZ77 of the block's segment t (256 bytes), symbols to global scratch, counts in shared memory
//   codes       two threads: lit/len and distance code lengths (bgzf_huff_lengths); one: canonical codes and the block header
//   pack        each thread's segment bit length, a block-wide scan, then each thread ORs its bits into the shared output words
//   member      gzip header, DEFLATE data (or a stored block when not smaller), CRC32, ISIZE into the block's 64 KiB slot
// A second kernel gathers the members into one buffer, which is what comes back over PCIe.  The per-block logic is bgzf_device.cuh,
// shared with the host emulation tests/host_emul/bgzf_emul.cpp, which gives the same bytes.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "bgzf_device.cuh"
#include <vector>

namespace {

constexpr int kThreads = 256;
constexpr int kQuarters = 4;
constexpr size_t kDataBytes = 65536, kPrevBytes = (size_t) BGZF_BLOCK * 2, kWorkBytes = 32768;
constexpr size_t kSmem = kDataBytes + kPrevBytes + kWorkBytes;

struct BgzfWork {                      // the work area once the head tables are no longer needed
    uint32_t fll[288], fd[32];
    BgzfCodes codes;
    BgzfHuffTmp t[2];
    BgzfHeaderTmp h;
    uint16_t seg_n[kThreads];
};
static_assert(sizeof(BgzfWork) <= kWorkBytes, "BgzfWork fits the head tables' space");
static_assert(kQuarters * (1 << BGZF_HASH_BITS) * 2 <= kWorkBytes, "head tables");
static_assert(BGZF_NSEG <= kThreads, "one segment per thread");

__global__ void __launch_bounds__(kThreads, 1)
bgzf_block_kernel(const uint8_t *__restrict__ in, const int64_t *__restrict__ starts, int nb, BgzfX2n x2n, uint16_t *items_all,
                  uint8_t *slots, int32_t *sizes) {
    extern __shared__ __align__(16) uint8_t sm[];
    uint8_t *d = sm;
    uint16_t *prev = (uint16_t *) (sm + kDataBytes);
    uint32_t *wbuf = (uint32_t *) (sm + kDataBytes);               // the output words, once prev[] is no longer needed
    uint16_t *heads = (uint16_t *) (sm + kDataBytes + kPrevBytes);
    BgzfWork &wk = *(BgzfWork *) (sm + kDataBytes + kPrevBytes);
    __shared__ uint32_t crc_part[4];
    __shared__ unsigned long long warp_sum[kThreads / 32];
    __shared__ unsigned long long s_hbits;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint16_t *items = items_all + (size_t) blockIdx.x * BGZF_BLOCK;
    for (int b = blockIdx.x; b < nb; b += gridDim.x) {
        const int64_t s0 = starts[b];
        const int n = (int) (starts[b + 1] - s0);
        for (int i = tid; i < n; i += kThreads) d[i] = in[s0 + i];
        for (int i = tid; i < kQuarters * (1 << BGZF_HASH_BITS) / 2; i += kThreads) ((uint32_t *) heads)[i] = 0xFFFFFFFFu;
        __syncthreads();
        const int np = n >= 3 ? n - 2 : 0, R = (np + kQuarters - 1) / kQuarters;
        if (warp < kQuarters) {
            uint16_t *hd = heads + warp * (1 << BGZF_HASH_BITS);
            const int lo = warp * R, hi = bm2_min(np, lo + R);
            for (int base = lo; base < hi; base += 32) {
                const int i = base + lane;
                const bool ok = i < hi;
                const uint32_t h = ok ? bgzf_hash3(d + i) : (1u << BGZF_HASH_BITS) + lane;
                const unsigned mask = __match_any_sync(0xFFFFFFFFu, h);
                const unsigned lower = mask & ((1u << lane) - 1);
                const uint16_t p = ok ? (lower ? (uint16_t) (base + 31 - __clz(lower)) : hd[h]) : (uint16_t) BGZF_NONE;
                __syncwarp();
                if (ok && (mask >> lane) == 1u) hd[h] = (uint16_t) i;         // the highest lane of the group
                if (ok) prev[i] = p;
                __syncwarp();
            }
        } else {
            const int t = tid - kQuarters * 32, K = (n + BGZF_SEG - 1) / BGZF_SEG;
            uint32_t acc = 0;
            for (int k = t; k < K; k += kThreads - kQuarters * 32) {
                const int hi = n - BGZF_SEG * k, lo = bm2_max(0, hi - BGZF_SEG);
                acc ^= bgzf_multmodp(bgzf_xpow(x2n, (uint64_t) 8 * BGZF_SEG * k), bgzf_crc_raw(d + lo, hi - lo, 0));
            }
            if (t == 0) acc ^= bgzf_multmodp(bgzf_xpow(x2n, (uint64_t) 8 * n), 0xFFFFFFFFu);      // the initial ~0, n bytes before the end
            for (int o = 16; o; o >>= 1) acc ^= __shfl_xor_sync(0xFFFFFFFFu, acc, o);
            if (lane == 0) crc_part[warp - kQuarters] = acc;
        }
        __syncthreads();
        for (int i = tid; i < np; i += kThreads) {                             // chain starts of a quarter: the heads of the earlier quarters
            if (prev[i] != BGZF_NONE) continue;
            const uint32_t h = bgzf_hash3(d + i);
            for (int q = i / R - 1; q >= 0; --q) { const uint16_t v = heads[q * (1 << BGZF_HASH_BITS) + h]; if (v != BGZF_NONE) { prev[i] = v; break; } }
        }
        __syncthreads();
        for (int i = tid; i < 288; i += kThreads) wk.fll[i] = i == 256;        // the end-of-block symbol
        if (tid < 32) wk.fd[tid] = 0;
        __syncthreads();
        const int nseg = (n + BGZF_SEG - 1) / BGZF_SEG;
        if (tid < nseg) wk.seg_n[tid] = (uint16_t) bgzf_parse_segment(d, n, prev, tid * BGZF_SEG, bm2_min(n, (tid + 1) * BGZF_SEG), items + tid * BGZF_SEG,
                                                                      wk.fll, wk.fd);
        __syncthreads();
        const int n_words = (n + 5) / 4 + 160;                                // and room for the longest header
        for (int i = tid; i < n_words; i += kThreads) wbuf[i] = 0;
        if (tid == 0) bgzf_huff_lengths(wk.fll, 286, 15, wk.codes.ll_len, wk.t[0]);
        if (tid == 32) bgzf_huff_lengths(wk.fd, 30, 15, wk.codes.d_len, wk.t[1]);
        __syncthreads();
        if (tid == 0) s_hbits = bgzf_write_header(wk.codes, wk.h, wk.t[0], wbuf);
        __syncthreads();
        // the segments' bit offsets: a block-wide exclusive scan
        const unsigned long long mine = tid < nseg ? bgzf_segment_bits(items + tid * BGZF_SEG, wk.seg_n[tid], wk.codes) : 0;
        unsigned long long inc = mine;
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long v = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += v; }
        if (lane == 31) warp_sum[warp] = inc;
        __syncthreads();
        unsigned long long before = 0, total = 0;
        for (int w = 0; w < kThreads / 32; ++w) { if (w < warp) before += warp_sum[w]; total += warp_sum[w]; }
        const uint64_t hb = s_hbits, eob = hb + total, bits = eob + wk.codes.ll_len[256];
        const bool stored = (int64_t) ((bits + 7) / 8) >= (int64_t) n + 5;
        if (!stored) {
            if (tid < nseg) bgzf_emit_segment(items + tid * BGZF_SEG, wk.seg_n[tid], wk.codes, wbuf, hb + before + inc - mine);
            if (tid == 0) bgzf_put(wbuf, eob, wk.codes.ll_code[256], wk.codes.ll_len[256]);
        }
        __syncthreads();
        const int body = stored ? n + 5 : (int) ((bits + 7) / 8), member = 18 + body + 8;
        uint8_t *o = slots + (size_t) b * BGZF_MAX_MEMBER;
        if (stored) for (int i = tid; i < n; i += kThreads) o[23 + i] = d[i];
        else for (int i = tid; i < body; i += kThreads) o[18 + i] = ((const uint8_t *) wbuf)[i];
        if (tid == 0) {
            bgzf_member_head(o, member);
            if (stored) bgzf_stored_head(o + 18, n);
            bgzf_put32(o + 18 + body, ~(crc_part[0] ^ crc_part[1] ^ crc_part[2] ^ crc_part[3]));
            bgzf_put32(o + 22 + body, (uint32_t) n);
            sizes[b] = member;
        }
        __syncthreads();
    }
}

// one CTA per member: its slot to its place in the output
__global__ void bgzf_gather_kernel(const uint8_t *__restrict__ slots, const int32_t *__restrict__ sizes, const int64_t *__restrict__ offs, uint8_t *out) {
    const int b = blockIdx.x;
    const uint8_t *s = slots + (size_t) b * BGZF_MAX_MEMBER;
    uint8_t *o = out + offs[b];
    for (int i = threadIdx.x; i < sizes[b]; i += blockDim.x) o[i] = s[i];
}

enum { BG_IN, BG_STARTS, BG_ITEMS, BG_SLOTS, BG_SIZES, BG_OFFS, BG_OUT, BG_END };
enum { BH_SIZES, BH_OUT, BH_END };
static_assert(BG_END == std::extent<decltype(bm2_ctx::bgzf_d)>::value, "bm2_ctx::bgzf_d: one buffer per slot");
static_assert(BH_END == std::extent<decltype(bm2_ctx::bgzf_h)>::value, "bm2_ctx::bgzf_h: one buffer per slot");

}  // namespace

// the members of the nb blocks [starts[b], starts[b+1]) of d_in (device, on ctx's stream) -> *out (host, ctx's) and member sizes (ctx->bgzf_sizes);
// gather: the device buffer the members are gathered into (nullptr: the context's own)
int bgzf_compress_device(bm2_ctx *ctx, const uint8_t *d_in, const int64_t *starts, int64_t nb, const uint8_t **out, int64_t *out_len, DevBuf *gather) {
    bm2_ctx *ctx_for_error = ctx;
    ctx->bgzf_ms = 0; ctx->bgzf_members = 0; ctx->bgzf_sizes.clear();
    *out = nullptr; *out_len = 0;
    if (nb == 0) return 0;
    if (nb >= (1LL << 31)) { bm2_set_error(ctx, "bm2_bgzf_compress: too many blocks"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int grid = (int) bm2_min<int64_t>(nb, ctx->n_sm);
    DevBuf *bg = ctx->bgzf_d;
    if (ctx->ensure(bg[BG_STARTS], (size_t) (nb + 1) * 8) ||
        ctx->ensure(bg[BG_ITEMS], (size_t) grid * BGZF_BLOCK * 2) || ctx->ensure(bg[BG_SLOTS], (size_t) nb * BGZF_MAX_MEMBER) ||
        ctx->ensure(bg[BG_SIZES], (size_t) nb * 4) || ctx->ensure(bg[BG_OFFS], (size_t) (nb + 1) * 8) ||
        ctx->ensure_host(ctx->bgzf_h[BH_SIZES], (size_t) (nb + 1) * 8)) return 1;
    for (cudaEvent_t &ev : ctx->bgzf_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    BM2_CUDA_OK(cudaFuncSetAttribute(bgzf_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) kSmem));
    BM2_CUDA_OK(cudaMemcpyAsync(bg[BG_STARTS].p, starts, (size_t) (nb + 1) * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaEventRecord(ctx->bgzf_ev[0], st));
    bgzf_block_kernel<<<grid, kThreads, kSmem, st>>>(d_in, (const int64_t *) bg[BG_STARTS].p, (int) nb, bgzf_x2n(),
                                                     (uint16_t *) bg[BG_ITEMS].p, (uint8_t *) bg[BG_SLOTS].p, (int32_t *) bg[BG_SIZES].p);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->bgzf_ev[1], st));
    int32_t *hs = (int32_t *) ctx->bgzf_h[BH_SIZES].p;
    BM2_CUDA_OK(cudaMemcpyAsync(hs, bg[BG_SIZES].p, (size_t) nb * 4, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    std::vector<int64_t> offs((size_t) nb + 1, 0);
    for (int64_t b = 0; b < nb; ++b) {
        if (hs[b] < 26 || hs[b] > BGZF_MAX_MEMBER) { bm2_set_error(ctx, "bm2_bgzf_compress: a member of " + std::to_string(hs[b]) + " bytes"); return 2; }
        offs[(size_t) b + 1] = offs[(size_t) b] + hs[b];
    }
    ctx->bgzf_sizes.assign(hs, hs + nb);
    const int64_t total = offs[(size_t) nb];
    DevBuf &dst = gather ? *gather : bg[BG_OUT];
    if (ctx->ensure(dst, (size_t) total + 16) || ctx->ensure_host(ctx->bgzf_h[BH_OUT], (size_t) total + 16)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(bg[BG_OFFS].p, offs.data(), (size_t) (nb + 1) * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaEventRecord(ctx->bgzf_ev[2], st));
    bgzf_gather_kernel<<<(unsigned) nb, 256, 0, st>>>((const uint8_t *) bg[BG_SLOTS].p, (const int32_t *) bg[BG_SIZES].p, (const int64_t *) bg[BG_OFFS].p,
                                                      (uint8_t *) dst.p);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->bgzf_ev[3], st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->bgzf_h[BH_OUT].p, dst.p, (size_t) total, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms0 = 0, ms1 = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms0, ctx->bgzf_ev[0], ctx->bgzf_ev[1]));
    BM2_CUDA_OK(cudaEventElapsedTime(&ms1, ctx->bgzf_ev[2], ctx->bgzf_ev[3]));
    ctx->bgzf_ms = (double) ms0 + ms1; ctx->bgzf_members = nb;
    *out = (const uint8_t *) ctx->bgzf_h[BH_OUT].p; *out_len = total;
    return 0;
}

extern "C" int bm2_bgzf_compress(bm2_ctx *ctx, const uint8_t *in, int64_t n, const int64_t *cut, int64_t n_cut, const uint8_t **out, int64_t *out_len) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || !out_len || n < 0 || (n && !in) || n_cut < 0 || (n_cut && !cut)) { if (ctx) bm2_set_error(ctx, "bm2_bgzf_compress: bad arguments"); return 1; }
    for (int64_t i = 0; i < n_cut; ++i)
        if (cut[i] < 0 || cut[i] > n || (i && cut[i] < cut[i - 1])) { bm2_set_error(ctx, "bm2_bgzf_compress: cut points must ascend within [0, n]"); return 1; }
    ctx->bgzf_ms = 0; ctx->bgzf_members = 0;
    *out = nullptr; *out_len = 0;
    std::vector<int64_t> starts;
    const int64_t nb = bgzf_cut_blocks(n, cut, n_cut, starts);
    if (nb == 0) return 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *bg = ctx->bgzf_d;
    if (ctx->ensure(bg[BG_IN], (size_t) n + 16)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(bg[BG_IN].p, in, (size_t) n, cudaMemcpyHostToDevice, ctx->stream));
    return bgzf_compress_device(ctx, (const uint8_t *) bg[BG_IN].p, starts.data(), nb, out, out_len, nullptr);
}

extern "C" int bm2_last_bgzf_stats(const bm2_ctx *ctx, double *device_ms, int64_t *members) {
    if (!ctx || !device_ms || !members) return 1;
    *device_ms = ctx->bgzf_ms; *members = ctx->bgzf_members;
    return 0;
}

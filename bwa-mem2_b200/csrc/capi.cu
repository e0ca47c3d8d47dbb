// capi.cu — the C ABI of libbm2b200.so (include/bm2_b200.h): context, parameter handling and the
// host side of seam 1 (bm2_extend_pairs).  Seam 2 lives in pipeline.cu.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include <cstdlib>
#include <cstring>
#include <vector>
#include <mutex>

static std::string g_create_error;
static std::mutex g_err_mu;

void bm2_set_error(bm2_ctx *ctx, const std::string &msg) {
    std::lock_guard<std::mutex> lk(g_err_mu);
    if (ctx) ctx->err = msg; else g_create_error = msg;
}

int bsw_launch_with_scratch(bm2_ctx *ctx_for_error, cudaStream_t stream, const BswJob *d_jobs, BswOut *d_out, int n,
                            const uint8_t *d_tbase, const uint8_t *d_qbase, const BswParams &prm,
                            unsigned long long *d_cells, void *scratch, size_t scratch_bytes, int wide_possible);

extern "C" int bm2_abi_version(void) { return BM2_ABI_VERSION; }

extern "C" void bm2_opt_init(bm2_mem_opt_t *o) {
    // mem_opt_init, reference src/bwamem.cpp:107-143
    memset(o, 0, sizeof(*o));
    o->a = 1; o->b = 4;
    o->o_del = o->o_ins = 6;
    o->e_del = o->e_ins = 1;
    o->w = 100;
    o->T = 30;
    o->zdrop = 100;
    o->pen_unpaired = 17;
    o->pen_clip5 = o->pen_clip3 = 5;
    o->max_mem_intv = 20;
    o->min_seed_len = 19;
    o->split_width = 10;
    o->max_occ = 500;
    o->max_chain_gap = 10000;
    o->max_ins = 10000;
    o->mask_level = 0.50f;
    o->drop_ratio = 0.50f;
    o->XA_drop_ratio = 0.80f;
    o->split_factor = 1.5f;
    o->chunk_size = 10000000;
    o->n_threads = 1;
    o->max_XA_hits = 5;
    o->max_XA_hits_alt = 200;
    o->max_matesw = 50;
    o->mask_level_redun = 0.95f;
    o->min_chain_weight = 0;
    o->max_chain_extend = 1 << 30;
    o->mapQ_coef_len = 50;
    o->mapQ_coef_fac = 3;   // (int) log(50)
    // bwa_fill_scmat, reference src/bwa.cpp:248-258
    int k = 0;
    for (int i = 0; i < 4; ++i) {
        for (int j = 0; j < 4; ++j) o->mat[k++] = i == j ? o->a : -o->b;
        o->mat[k++] = -1;
    }
    for (int j = 0; j < 5; ++j) o->mat[k++] = -1;
}

int bm2_ctx::ensure(DevBuf &b, size_t bytes) {
    bm2_ctx *ctx_for_error = this;
    if (b.cap >= bytes) return 0;
    if (b.p) BM2_CUDA_OK(cudaFree(b.p));
    b.p = nullptr; b.cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    BM2_CUDA_OK(cudaMalloc(&b.p, want));
    b.cap = want;
    return 0;
}

int bm2_ctx::ensure_host(HostBuf &b, size_t bytes) {
    bm2_ctx *ctx_for_error = this;
    if (b.cap >= bytes) return 0;
    if (b.p) BM2_CUDA_OK(cudaFreeHost(b.p));
    b.p = nullptr; b.cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    BM2_CUDA_OK(cudaMallocHost(&b.p, want));
    b.cap = want;
    return 0;
}

int bm2_upload_index(bm2_ctx *ctx, const bm2_index_desc *idx, int resident);   // pipeline.cu
void bm2_free_index(bm2_ctx *ctx);

static int create_impl(bm2_ctx **out, int device, const bm2_index_desc *idx, const bm2_mem_opt_t *opt, int resident);
extern "C" int bm2_create(bm2_ctx **out, int device, const bm2_index_desc *idx, const bm2_mem_opt_t *opt) { return create_impl(out, device, idx, opt, 0); }
extern "C" int bm2_create_resident(bm2_ctx **out, int device, const bm2_index_desc *dev_idx, const bm2_mem_opt_t *opt) {
    if (!dev_idx) { bm2_set_error(nullptr, "bm2_create_resident: dev_idx is NULL"); return 1; }
    return create_impl(out, device, dev_idx, opt, 1);
}

static int create_impl(bm2_ctx **out, int device, const bm2_index_desc *idx, const bm2_mem_opt_t *opt, int resident) {
    bm2_ctx *ctx_for_error = nullptr;
    if (!out) { bm2_set_error(nullptr, "bm2_create: out is NULL"); return 1; }
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        bm2_set_error(nullptr, std::string("bm2_create: no usable CUDA device (") + cudaGetErrorString(e) +
                               "); this library has no CPU fallback");
        return 2;
    }
    if (device < 0 || device >= ndev) { bm2_set_error(nullptr, "bm2_create: bad device ordinal"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(device));
    cudaDeviceProp prop;
    BM2_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {      // the library holds an sm_90a cubin only (arch-specific: no forward compatibility)
        bm2_set_error(nullptr, "bm2_create: device is not sm_90 (library is built for sm_90a only)");
        return 2;
    }
    bm2_ctx *ctx = new bm2_ctx();
    ctx->device = device;
    ctx->n_sm = prop.multiProcessorCount;
    if (opt) ctx->opt = *opt; else bm2_opt_init(&ctx->opt);
    if (const char *e = getenv("BM2_SUB_BATCHES")) { int k = atoi(e); if (k >= 1 && k <= 16) ctx->n_lanes = k; }
    ctx_for_error = ctx;
    if (cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
        bm2_set_error(nullptr, "bm2_create: cudaStreamCreate failed"); bm2_destroy(ctx); return 1;
    }
    ctx->stream = ctx->own_stream;
    if (cudaStreamCreateWithFlags(&ctx->side_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming) != cudaSuccess) {
        bm2_set_error(nullptr, "bm2_create: side stream/events failed"); bm2_destroy(ctx); return 1;
    }
    if (idx) {
        if (bm2_upload_index(ctx, idx, resident)) { bm2_set_error(nullptr, "bm2_create: " + ctx->err); bm2_destroy(ctx); return 1; }
    }
    *out = ctx;
    return 0;
}

// A lane: a child context for one sub-batch in flight (own streams, events and scratch; the parent's index by reference).
bm2_ctx *bm2_make_lane(bm2_ctx *parent) {
    bm2_ctx *c = new bm2_ctx();
    c->device = parent->device; c->n_sm = parent->n_sm; c->opt = parent->opt;
    c->idx = parent->idx;                      // device pointers only; idx_allocs stays empty: the parent owns the memory
    c->n_lanes = 1;
    c->parent = parent;
    if (cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->side_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess) {
        bm2_set_error(parent, "sub-batch lane: stream/event creation failed");
        bm2_destroy(c);
        return nullptr;
    }
    c->stream = c->own_stream;
    return c;
}

extern "C" int bm2_create_sibling(bm2_ctx **out, bm2_ctx *ctx) {
    if (!out || !ctx) { bm2_set_error(ctx, "bm2_create_sibling: NULL argument"); return 1; }
    *out = nullptr;
    if (ctx->parent) { bm2_set_error(ctx, "bm2_create_sibling: not on a sub-batch lane"); return 1; }
    if (cudaSetDevice(ctx->device) != cudaSuccess) { bm2_set_error(ctx, "bm2_create_sibling: cudaSetDevice failed"); return 1; }
    bm2_ctx *c = bm2_make_lane(ctx);           // own streams, events and buffers; the index by reference (idx_allocs empty: never freed here)
    if (!c) return 1;
    c->parent = nullptr;                       // a full context of its own: its own sub-batch lanes, its own error text
    c->n_lanes = ctx->n_lanes; c->lane_min_reads = ctx->lane_min_reads; c->sam_staged = ctx->sam_staged;
    *out = c;
    return 0;
}

extern "C" int bm2_set_sub_batches(bm2_ctx *ctx, int k, int min_reads) {
    if (!ctx || k < 1 || k > 16 || min_reads < 512) { if (ctx) bm2_set_error(ctx, "bm2_set_sub_batches: k in 1..16, min_reads >= 512"); return 1; }
    ctx->n_lanes = k; ctx->lane_min_reads = min_reads;
    return 0;
}

extern "C" int bm2_set_sam_staged(bm2_ctx *ctx, int on) {
    if (!ctx || on < -1 || on > 2) { if (ctx) bm2_set_error(ctx, "bm2_set_sam_staged: on in {-1, 0, 1, 2}"); return 1; }
    ctx->sam_staged = on;
    return 0;
}

extern "C" int bm2_last_sam_stats(const bm2_ctx *ctx, double *ms, unsigned long long *counts, int n_ms, int n_counts) {
    if (!ctx || !ms || !counts || n_ms < 4 || n_counts < 6) return 1;
    for (int k = 0; k < 4; ++k) ms[k] = ctx->sam_ms[k];
    for (int k = 0; k < 6; ++k) counts[k] = ctx->sam_counts[k];
    return 0;
}

extern "C" void bm2_destroy(bm2_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (bm2_ctx *l : ctx->lanes) bm2_destroy(l);
    ctx->lanes.clear();
    if (ctx->ev_entry) cudaEventDestroy(ctx->ev_entry);
    for (cudaEvent_t ev : ctx->sam_ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ctx->bgzf_ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ctx->sort_ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ctx->dup_ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ctx->bqa_ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ctx->mm_ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ctx->mdb_ev) if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : ctx->b2f_ev) if (ev) cudaEventDestroy(ev);
    bm2_free_index(ctx);
    for (DevBuf *b : ctx->all_dev()) if (b->p) cudaFree(b->p);
    for (HostBuf *b : ctx->all_host()) if (b->p) cudaFreeHost(b->p);
    for (cudaEvent_t ev : ctx->events) if (ev) cudaEventDestroy(ev);
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    if (ctx->side_stream) cudaStreamDestroy(ctx->side_stream);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    delete ctx;
}

extern "C" const char *bm2_last_error(const bm2_ctx *ctx) {
    // the caller gets a per-thread copy: another thread setting a new message cannot invalidate the returned pointer
    static thread_local std::string copy;
    std::lock_guard<std::mutex> lk(g_err_mu);
    copy = ctx ? ctx->err : g_create_error;
    return copy.c_str();
}

static BswParams bsw_params_of(const bm2_ctx *ctx, int w, int end_bonus) {
    BswParams p;
    p.a = ctx->opt.a; p.b = ctx->opt.b;
    p.o_del = ctx->opt.o_del; p.e_del = ctx->opt.e_del; p.o_ins = ctx->opt.o_ins; p.e_ins = ctx->opt.e_ins;
    p.zdrop = ctx->opt.zdrop; p.end_bonus = end_bonus; p.w = w;
    return p;
}

// ---- seam 1 ------------------------------------------------------------------------------------
__global__ void pairs_to_jobs_kernel(const bm2_seqpair *pairs, int n, BswJob *jobs) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bm2_seqpair sp = pairs[i];
    BswJob j;
    j.toff = sp.idr; j.qoff = sp.idq; j.tlen = sp.len1; j.qlen = sp.len2; j.h0 = sp.h0;
    j.tstride = 1; j.qstride = 1; j._pad = 0;
    jobs[i] = j;
}

__global__ void outs_to_pairs_kernel(const BswOut *outs, int n, bm2_seqpair *pairs) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    BswOut o = outs[i];
    pairs[i].score = o.score; pairs[i].tle = o.tle; pairs[i].gtle = o.gtle; pairs[i].qle = o.qle;
    pairs[i].gscore = o.gscore; pairs[i].max_off = o.max_off;
}

extern "C" int bm2_extend_pairs_device(bm2_ctx *ctx, bm2_seqpair *d_pairs, const uint8_t *d_ref, const uint8_t *d_qer,
                                       int32_t n, int32_t w, int32_t end_bonus, unsigned long long *d_cells) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx) return 1;
    if (n <= 0) return 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    if (ctx->ensure(ctx->bsw_jobs, (size_t) n * sizeof(BswJob))) return 1;
    if (ctx->ensure(ctx->bsw_outs, (size_t) n * sizeof(BswOut))) return 1;
    if (ctx->ensure(ctx->bsw_scratch, bsw_scratch_bytes(n))) return 1;
    pairs_to_jobs_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_pairs, n, (BswJob *) ctx->bsw_jobs.p);
    BswParams p = bsw_params_of(ctx, w, end_bonus);
    if (bsw_launch_with_scratch(ctx, ctx->stream, (const BswJob *) ctx->bsw_jobs.p, (BswOut *) ctx->bsw_outs.p, n, d_ref, d_qer,
                                p, d_cells, ctx->bsw_scratch.p, ctx->bsw_scratch.cap, 1)) return 1;
    outs_to_pairs_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>((const BswOut *) ctx->bsw_outs.p, n, d_pairs);
    BM2_CUDA_OK(cudaGetLastError());
    return 0;
}

extern "C" int bm2_extend_pairs(bm2_ctx *ctx, bm2_seqpair *pairs, const uint8_t *ref, const uint8_t *qer, int32_t n,
                                int32_t w, int32_t end_bonus) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx) return 1;
    if (n <= 0) return 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    // extent of the two byte buffers actually referenced
    int64_t ref_bytes = 0, qer_bytes = 0;
    for (int i = 0; i < n; ++i) {
        if (pairs[i].len1 < 0 || pairs[i].len2 < 0 || pairs[i].idr < 0 || pairs[i].idq < 0) {
            bm2_set_error(ctx, "bm2_extend_pairs: negative length/offset"); return 1;
        }
        int64_t r = (int64_t) pairs[i].idr + pairs[i].len1, q = (int64_t) pairs[i].idq + pairs[i].len2;
        if (r > ref_bytes) ref_bytes = r;
        if (q > qer_bytes) qer_bytes = q;
    }
    if (ctx->ensure(ctx->io_pairs, (size_t) n * sizeof(bm2_seqpair))) return 1;
    if (ctx->ensure(ctx->io_ref, (size_t) ref_bytes + 16)) return 1;
    if (ctx->ensure(ctx->io_qer, (size_t) qer_bytes + 16)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->io_pairs.p, pairs, (size_t) n * sizeof(bm2_seqpair), cudaMemcpyHostToDevice, ctx->stream));
    if (ref_bytes) BM2_CUDA_OK(cudaMemcpyAsync(ctx->io_ref.p, ref, ref_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (qer_bytes) BM2_CUDA_OK(cudaMemcpyAsync(ctx->io_qer.p, qer, qer_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (bm2_extend_pairs_device(ctx, (bm2_seqpair *) ctx->io_pairs.p, (const uint8_t *) ctx->io_ref.p,
                                (const uint8_t *) ctx->io_qer.p, n, w, end_bonus, nullptr)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(pairs, ctx->io_pairs.p, (size_t) n * sizeof(bm2_seqpair), cudaMemcpyDeviceToHost, ctx->stream));
    BM2_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return 0;
}

extern "C" int bm2_set_stream(bm2_ctx *ctx, void *cuda_stream) {
    if (!ctx) return 1;
    ctx->stream = cuda_stream ? (cudaStream_t) cuda_stream : ctx->own_stream;
    return 0;
}

// ---- integer-pipe micro-benchmark: 8 independent dependent-chains of add+max per thread ----------
__global__ void int_pipe_kernel(int *out, int iters, int seed) {
    int a0 = seed + threadIdx.x, a1 = a0 ^ 0x55, a2 = a0 + 7, a3 = a0 * 3, a4 = a0 - 11, a5 = a0 ^ 0x33, a6 = a0 + 101, a7 = a0 - 5;
    const int d = seed | 1, z = seed >> 20;
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            a0 = max(a0 - d, z); a1 = max(a1 - d, z); a2 = max(a2 - d, z); a3 = max(a3 - d, z);
            a4 = max(a4 + d, z); a5 = max(a5 + d, z); a6 = max(a6 + d, z); a7 = max(a7 + d, z);
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

extern "C" int bm2_int_pipe_gops(bm2_ctx *ctx, double *gops) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !gops) return 1;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    const int blocks = ctx->n_sm * 8, threads = 256, iters = 4096;
    if (ctx->ensure(ctx->bsw_outs, (size_t) blocks * threads * 4)) return 1;
    cudaEvent_t e0, e1;
    BM2_CUDA_OK(cudaEventCreate(&e0)); BM2_CUDA_OK(cudaEventCreate(&e1));
    float best = 1e30f;
    for (int rep = 0; rep < 5; ++rep) {
        BM2_CUDA_OK(cudaEventRecord(e0, ctx->stream));
        int_pipe_kernel<<<blocks, threads, 0, ctx->stream>>>((int *) ctx->bsw_outs.p, iters, 12345 + rep);
        BM2_CUDA_OK(cudaEventRecord(e1, ctx->stream));
        BM2_CUDA_OK(cudaEventSynchronize(e1));
        float ms = 0; BM2_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    // per loop iteration and thread: 8 unrolled x 8 chains x 2 ops (add, max)
    double ops = (double) blocks * threads * (double) iters * 8 * 8 * 2;
    *gops = ops / (best * 1e-3) / 1e9;
    return 0;
}

// ---- random 64-byte gather micro-benchmark over the Occ checkpoint table --------------------------------------------------
// The SMEM stage reads two random 64-byte checkpoints per interval extension; this measures what the memory system
// delivers for exactly that access shape when nothing else limits it: every thread keeps `MLP` independent 64-byte
// (4 x 16 B) loads of pseudo-random checkpoints in flight, no dependent address chain, trivial arithmetic.
template <int MLP>
__global__ void __launch_bounds__(256) gather64_kernel(const uint4 *__restrict__ tab, unsigned long long n_entries, int iters, unsigned long long seed,
                                                       unsigned *out) {
    unsigned long long x = seed + (unsigned long long) (blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ull;
    unsigned acc = 0;
    for (int it = 0; it < iters; ++it) {
        uint4 v[MLP][4];
#pragma unroll
        for (int m = 0; m < MLP; ++m) {
            x ^= x << 13; x ^= x >> 7; x ^= x << 17;                 // xorshift64
            const unsigned long long e = (unsigned long long) (((unsigned __int128) x * n_entries) >> 64);
#pragma unroll
            for (int q = 0; q < 4; ++q) v[m][q] = __ldg(tab + e * 4 + q);
        }
#pragma unroll
        for (int m = 0; m < MLP; ++m)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc += v[m][q].x ^ v[m][q].y ^ v[m][q].z ^ v[m][q].w;
    }
    if (acc == 0x12345678u) out[0] = acc;                            // keeps the loads alive
}

extern "C" int bm2_gather64_gbs(bm2_ctx *ctx, unsigned long long span_bytes, double *gbs) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !gbs) return 1;
    if (!ctx->idx.loaded) { bm2_set_error(ctx, "bm2_gather64_gbs needs a context created with an index"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    unsigned long long n_entries = (unsigned long long) (ctx->idx.N >> 6) + 1;
    if (span_bytes && span_bytes / 64 < n_entries) n_entries = span_bytes / 64 ? span_bytes / 64 : 1;     // only the first span_bytes of the table
    const int blocks = ctx->n_sm * 8, threads = 256, iters = 64;
    constexpr int MLP = 4;
    if (ctx->ensure(ctx->bsw_outs, 256)) return 1;
    cudaEvent_t e0, e1;
    BM2_CUDA_OK(cudaEventCreate(&e0)); BM2_CUDA_OK(cudaEventCreate(&e1));
    float best = 1e30f;
    for (int rep = 0; rep < 4; ++rep) {
        BM2_CUDA_OK(cudaEventRecord(e0, ctx->stream));
        gather64_kernel<MLP><<<blocks, threads, 0, ctx->stream>>>((const uint4 *) ctx->idx.cp_occ, n_entries, iters, 777 + rep, (unsigned *) ctx->bsw_outs.p);
        BM2_CUDA_OK(cudaEventRecord(e1, ctx->stream));
        BM2_CUDA_OK(cudaEventSynchronize(e1));
        float ms = 0; BM2_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    *gbs = (double) blocks * threads * (double) iters * MLP * 64.0 / (best * 1e-3) / 1e9;
    return 0;
}

// ---- gather probe with selectable request shape and memory-level parallelism ---------------------------------------------
// shape 0: 64 B per request as four 16-B loads of one thread (the shape of bm2_gather64_gbs); shape 1: 32 B per request as one
// sector read by two 128-bit loads (the half-checkpoint of the device Occ layout, fm_ld256 in fm_device.cuh); shape 2: 64 B per
// request as two such sectors.  `mlp` independent requests per thread are in flight (1, 2, 4 or 8).  Reports GB/s of requested bytes.
__device__ __forceinline__ void ld256(const void *p, unsigned long long &a, unsigned long long &b, unsigned long long &c, unsigned long long &d) {
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%4];\n\t"
                 "ld.global.nc.v2.u64 {%2,%3}, [%4+16];" : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p));
}
template <int MLP, int SHAPE>
__global__ void __launch_bounds__(256) gather_probe_kernel(const char *__restrict__ tab, unsigned long long n_units, int iters, unsigned long long seed,
                                                           unsigned *out) {
    unsigned long long x = seed + (unsigned long long) (blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ull;
    unsigned long long acc = 0;
    constexpr int UNIT = SHAPE == 1 ? 32 : 64;
    for (int it = 0; it < iters; ++it) {
        unsigned long long v[MLP][8];
#pragma unroll
        for (int m = 0; m < MLP; ++m) {
            x ^= x << 13; x ^= x >> 7; x ^= x << 17;
            const unsigned long long e = (unsigned long long) (((unsigned __int128) x * n_units) >> 64);
            const char *p = tab + e * UNIT;
            if (SHAPE == 0) {
#pragma unroll
                for (int q = 0; q < 4; ++q) { const uint4 t = __ldg(reinterpret_cast<const uint4 *>(p) + q); v[m][2 * q] = ((unsigned long long) t.x << 32) | t.y; v[m][2 * q + 1] = ((unsigned long long) t.z << 32) | t.w; }
            } else {
                ld256(p, v[m][0], v[m][1], v[m][2], v[m][3]);
                if (SHAPE == 2) ld256(p + 32, v[m][4], v[m][5], v[m][6], v[m][7]);
                else { v[m][4] = v[m][5] = v[m][6] = v[m][7] = 0; }
            }
        }
#pragma unroll
        for (int m = 0; m < MLP; ++m)
#pragma unroll
            for (int q = 0; q < 8; ++q) acc += v[m][q];
    }
    if (acc == 0x12345678u) out[0] = (unsigned) acc;
}

// shape 3: the same 32-byte requests through the bulk-async (TMA) path: every thread owns MLP 32-byte shared-memory slots and ONE mbarrier,
// announces the bytes (mbarrier.arrive.expect_tx), issues cp.async.bulk.shared::cluster.global per request and waits on the barrier's
// phase - the "Occ blocks TMA-staged to shared memory" shape of the north star, per lane because every lane of the SMEM kernels extends
// its own interval at its own random address (there is no tile to describe with a tensor map).
template <int MLP, bool MIXED>
__global__ void __launch_bounds__(256) gather_probe_bulk_kernel(const char *__restrict__ tab, unsigned long long n_units, int iters, unsigned long long seed,
                                                                unsigned *out) {
    __shared__ __align__(32) unsigned long long slots[256][MLP][4];
    __shared__ __align__(8) unsigned long long bars[256];
    const unsigned bar = (unsigned) __cvta_generic_to_shared(&bars[threadIdx.x]);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    unsigned long long x = seed + (unsigned long long) (blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ull;
    unsigned long long acc = 0;
    unsigned phase = 0;
    for (int it = 0; it < iters; ++it) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(32u * MLP) : "memory");
#pragma unroll
        for (int m = 0; m < MLP; ++m) {
            x ^= x << 13; x ^= x >> 7; x ^= x << 17;
            const unsigned long long e = (unsigned long long) (((unsigned __int128) x * n_units) >> 64);
            const unsigned dst = (unsigned) __cvta_generic_to_shared(&slots[threadIdx.x][m][0]);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], 32, [%2];"
                         :: "r"(dst), "l"(tab + e * 32), "r"(bar) : "memory");
        }
        if (MIXED) {          // shape 4: the same number of 256-bit loads in flight next to the bulk copies (do the two paths add up?)
            unsigned long long v[MLP][4];
#pragma unroll
            for (int m = 0; m < MLP; ++m) {
                x ^= x << 13; x ^= x >> 7; x ^= x << 17;
                const unsigned long long e = (unsigned long long) (((unsigned __int128) x * n_units) >> 64);
                ld256(tab + e * 32, v[m][0], v[m][1], v[m][2], v[m][3]);
            }
#pragma unroll
            for (int m = 0; m < MLP; ++m) acc += v[m][0] + v[m][1] + v[m][2] + v[m][3];
        }
        unsigned done = 0;
        while (!done) {
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(done) : "r"(bar), "r"(phase) : "memory");
        }
        phase ^= 1u;
#pragma unroll
        for (int m = 0; m < MLP; ++m)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc += slots[threadIdx.x][m][q];
    }
    if (acc == 0x12345678u) out[0] = (unsigned) acc;
}

extern "C" int bm2_gather_probe(bm2_ctx *ctx, unsigned long long span_bytes, int mlp, int shape, double *gbs) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !gbs || shape < 0 || shape > 4) return 1;
    if (!ctx->idx.loaded) { bm2_set_error(ctx, "bm2_gather_probe needs a context created with an index"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    const unsigned long long unit = (shape == 1 || shape >= 3) ? 32 : 64;
    unsigned long long n_units = ((unsigned long long) (ctx->idx.N >> 6) + 1) * 64 / unit;
    if (span_bytes && span_bytes / unit < n_units) n_units = span_bytes / unit ? span_bytes / unit : 1;
    const int blocks = ctx->n_sm * 8, threads = 256, iters = 64;
    if (ctx->ensure(ctx->bsw_outs, 256)) return 1;
    cudaEvent_t e0, e1;
    BM2_CUDA_OK(cudaEventCreate(&e0)); BM2_CUDA_OK(cudaEventCreate(&e1));
    float best = 1e30f;
    const char *tab = (const char *) ctx->idx.cp_occ; unsigned *o = (unsigned *) ctx->bsw_outs.p;
    for (int rep = 0; rep < 4; ++rep) {
        BM2_CUDA_OK(cudaEventRecord(e0, ctx->stream));
#define BM2_GP(M, S) gather_probe_kernel<M, S><<<blocks, threads, 0, ctx->stream>>>(tab, n_units, iters, 777 + rep, o)
#define BM2_GPS(M) do { if (shape == 0) BM2_GP(M, 0); else if (shape == 1) BM2_GP(M, 1); else if (shape == 2) BM2_GP(M, 2); \
                        else if (shape == 3) gather_probe_bulk_kernel<(M > 4 ? 4 : M), false><<<blocks, threads, 0, ctx->stream>>>(tab, n_units, iters, 777 + rep, o); \
                        else gather_probe_bulk_kernel<(M > 4 ? 4 : M), true><<<blocks, threads, 0, ctx->stream>>>(tab, n_units, iters, 777 + rep, o); } while (0)
        if (mlp <= 1) BM2_GPS(1); else if (mlp == 2) BM2_GPS(2); else if (mlp <= 4) BM2_GPS(4); else BM2_GPS(8);
#undef BM2_GPS
#undef BM2_GP
        BM2_CUDA_OK(cudaEventRecord(e1, ctx->stream));
        BM2_CUDA_OK(cudaEventSynchronize(e1));
        float ms = 0; BM2_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    int m_eff = mlp <= 1 ? 1 : mlp == 2 ? 2 : mlp <= 4 ? 4 : (shape >= 3 ? 4 : 8);      // (the bulk shapes hold at most 4 slots per thread)
    if (shape == 4) m_eff *= 2;                                                          // mixed: as many loads as bulk copies
    *gbs = (double) blocks * threads * (double) iters * m_eff * (double) unit / (best * 1e-3) / 1e9;
    return 0;
}

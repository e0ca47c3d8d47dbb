// pipeline.cu — seam 2: the seed -> SA -> chain -> extend pipeline on the GPU.
//
// Replaces kt_for(worker_bwt) + kt_for(worker_aln) of mem_process_seqs (reference
// src/bwamem.cpp:1359-1363), i.e. mem_kernel1_core (:976-1091) and mem_kernel2_core (:1093-1172),
// and the 512-read/thread batching of kthread.cpp:81-115: the whole chunk is one batch, every stage
// is one kernel over all reads (or all SMEMs / seed slots / extension jobs) of the chunk.
//
// Stage list (each a kernel or a cub primitive on ctx->stream):
//   A  smem_kernel         one read per thread, 3 SMEM passes (fm_device.cuh)       HBM random 64 B
//   B  radix sort of SMEMs by (read, m, n)  == sortSMEMs + per-read introsort
//   C  sa_kernel           one seed slot per thread, compressed-SA LF walk          HBM random 64 B
//   D  chain_kernel        one read per thread: chaining + chain filter (chain_device.cuh)
//   E  scans + compaction  flat chain / seed / reg / job arrays
//   F  ext_build_kernel    one read per thread: regs + left/right extension jobs
//   G  BSW left  (bsw.cu) + fold + doubled-band retry
//   H  BSW right (bsw.cu) + fold + doubled-band retry
//      (G and H run in waves, with a post-filter walk in between that proves seeds purged before they are extended: lazy extension)
//   I  tail_kernel         one read per thread: post-filter, dedup/patch, ALT marking
//   J  gather of the final regs, D2H
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "fm_device.cuh"
#include "chain_device.cuh"
#include "ext_device.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <vector>
#include <algorithm>
#include <mutex>
#include <thread>
#include <string>
#include <cstring>
#include <cstdlib>
#include <cmath>

static_assert(sizeof(ExtJobRec) == sizeof(BswJob), "ExtJobRec must alias BswJob");

int bsw_launch_with_scratch(bm2_ctx *ctx_for_error, cudaStream_t stream, const BswJob *d_jobs, BswOut *d_out, int n,
                            const uint8_t *d_tbase, const uint8_t *d_qbase, const BswParams &prm,
                            unsigned long long *d_cells, void *scratch, size_t scratch_bytes, int wide_possible);

// ------------------------------------------------------------------------------------------------
// index upload
// ------------------------------------------------------------------------------------------------
// The device layout of the Occ table (FmIndexView::layout 1, fm_device.cuh): words {c0,c1,c2,c3,b0,b1,b2,b3} of every 64-byte
// checkpoint become {c0,c1,b0,b1,c2,c3,b2,b3}, in place, once per upload.  The index files and bm2_index_desc keep the reference's format.
__global__ void occ_relayout_kernel(ulonglong2 *tab, size_t n_entries) {
    const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_entries) return;
    ulonglong2 *e = tab + i * 4;
    const ulonglong2 c23 = e[1], b01 = e[2];
    e[1] = b01; e[2] = c23;
}

// resident != 0: the four big arrays of `idx` are already in this device's memory (bm2_create_resident): adopted, not copied, not owned
int bm2_upload_index(bm2_ctx *ctx, const bm2_index_desc *idx, int resident) {
    bm2_ctx *ctx_for_error = ctx;
    auto up = [&](const void *src, size_t bytes, const void **dst, bool big) -> int {
        if (big && resident) { *dst = src; return 0; }
        void *p = nullptr;
        BM2_CUDA_OK(cudaMalloc(&p, bytes ? bytes : 1));
        ctx->idx_allocs.push_back(p);
        if (bytes) BM2_CUDA_OK(cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice));
        *dst = p;
        return 0;
    };
    DevIndex &d = ctx->idx;
    d.N = idx->reference_seq_len; d.l_pac = idx->l_pac; d.sentinel = idx->sentinel_index;
    for (int i = 0; i < 5; ++i) d.count[i] = idx->count[i];
    d.n_seqs = idx->n_seqs;
    size_t n_occ = (size_t) (d.N >> 6) + 1, n_sa = (size_t) (d.N >> 3) + 1;
    if (up(idx->cp_occ, n_occ * sizeof(bm2_cp_occ), (const void **) &d.cp_occ, true)) return 1;
    {   // BM2_OCC_LAYOUT=0 keeps the file layout on the device (A/B measurements); default: half-checkpoint sectors
        const char *e = getenv("BM2_OCC_LAYOUT");
        d.occ_layout = (e && e[0] == '0') ? 0 : 1;
        if (d.occ_layout) {
            occ_relayout_kernel<<<(unsigned) ((n_occ + 255) / 256), 256>>>((ulonglong2 *) d.cp_occ, n_occ);
            BM2_CUDA_OK(cudaGetLastError());
            BM2_CUDA_OK(cudaDeviceSynchronize());
        }
    }
    if (up(idx->sa_ms_byte, n_sa, (const void **) &d.sa_ms, true)) return 1;
    if (up(idx->sa_ls_word, n_sa * 4, (const void **) &d.sa_ls, true)) return 1;
    if (up(idx->ref_string, (size_t) d.l_pac * 2, (const void **) &d.ref, true)) return 1;
    if (up(idx->ann_offset, (size_t) d.n_seqs * 8, (const void **) &d.ann_off, false)) return 1;
    if (up(idx->ann_len, (size_t) d.n_seqs * 4, (const void **) &d.ann_len, false)) return 1;
    std::vector<int32_t> zeros;
    const int32_t *alt = idx->ann_is_alt;
    if (!alt) { zeros.assign(d.n_seqs, 0); alt = zeros.data(); }
    if (up(alt, (size_t) d.n_seqs * 4, (const void **) &d.ann_alt, false)) return 1;
    d.loaded = true;
    return 0;
}

void bm2_free_index(bm2_ctx *ctx) {
    for (void *p : ctx->idx_allocs) cudaFree(p);
    ctx->idx_allocs.clear();
    ctx->idx.loaded = false;
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
struct Counters {                 // device-side counters of one batch
    unsigned long long n_smem, n_ext, n_lf, n_retry, cells;
    unsigned long long n_pool, n_task, n_task1, n_rtask;     // SMEM stage: interval-list pool, search tasks, re-seed tasks
    unsigned long long n_sel[2], n_walk_done;                // lazy extension: left / right jobs of the wave, reads decided by the first walk
};

struct SearchTask { int32_t read, x, min_intv, n; int64_t off; };     // one backward phase: list pool[off .. off+n)
struct ReseedTask { int32_t read, x, min_intv; };                    // one pass-2 forward search


// A. SMEM passes 1+2 as homogeneous phases (fm_device.cuh): forward chains (one read per thread), backward tasks
// (one search per thread), pass-2 forward searches (one re-seed task per thread), backward tasks again.  The read is
// packed 4 bit/base into shared memory [word][thread] (bank = lane) for the read-per-thread kernels.
struct QShared4 {
    unsigned base, stride;
    __device__ __forceinline__ int operator()(int j) const {
        uint32_t w; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(base + (unsigned) (j >> 3) * stride));
        return (int) ((w >> ((j & 7) * 4)) & 0xFu);
    }
};

struct PoolSink {                 // hands the interval list of one finished forward phase to the backward kernel
    FmPrev *pool; unsigned long long pool_cap; SearchTask *tasks; unsigned long long task_cap; Counters *cnt; int read;
    __device__ __forceinline__ void operator()(int x, int min_intv, const FmPrev *list, int n) {
        if (n <= 0) return;
        const unsigned long long off = atomicAdd(&cnt->n_pool, (unsigned long long) n);
        const unsigned long long t = atomicAdd(&cnt->n_task, 1ULL);
        if (off + n <= pool_cap) for (int i = 0; i < n; ++i) pool[off + i] = list[i];
        if (t < task_cap) { SearchTask k; k.read = read; k.x = x; k.min_intv = min_intv; k.n = n; k.off = (int64_t) off; tasks[t] = k; }
    }
};

__device__ __forceinline__ void pack_read_smem(uint32_t *qsh, const uint8_t *qp, int len) {
    for (int k = 0; k < len; k += 8) {
        uint32_t wv = 0;
#pragma unroll
        for (int u = 0; u < 8; ++u) { uint32_t b = k + u < len ? (uint32_t) qp[k + u] : 4u; wv |= (b > 4u ? 4u : b) << (4 * u); }
        qsh[(k >> 3) * blockDim.x + threadIdx.x] = wv;
    }
}

template <bool USE_SMEM>
__global__ void __launch_bounds__(128, 10)
smem_fwd1_kernel(FmIndexView fm, const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs, int n_reads, int stripe,
                 FmPrev *scratch_all, FmPrev *pool, unsigned long long pool_cap, SearchTask *tasks, unsigned long long task_cap, Counters *cnt)
{
    extern __shared__ uint32_t qsh[];
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
    FmPrev *scratch = scratch_all + (size_t) tid * stripe;
    unsigned n_ext = 0;
    for (int r = tid; r < n_reads; r += nthr) {
        const int64_t o = offs[r];
        const int len = (int) (offs[r + 1] - o);
        PoolSink sink = { pool, pool_cap, tasks, task_cap, cnt, r };
        if (USE_SMEM) {
            pack_read_smem(qsh, codes + o, len);
            QShared4 q = { (unsigned) __cvta_generic_to_shared(qsh + threadIdx.x), (unsigned) blockDim.x * 4u };
            fm_forward(fm, q, len, 0, 1, false, scratch, sink, n_ext);
        } else {
            QPlain q = { codes + o };
            fm_forward(fm, q, len, 0, 1, false, scratch, sink, n_ext);
        }
    }
    if (n_ext) atomicAdd(&cnt->n_ext, (unsigned long long) n_ext);
}

__global__ void __launch_bounds__(128, 10)
smem_fwd2_kernel(FmIndexView fm, const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs, int stripe, FmPrev *scratch_all,
                 const ReseedTask *__restrict__ rtasks, unsigned long long rtask_cap, FmPrev *pool, unsigned long long pool_cap,
                 SearchTask *tasks, unsigned long long task_cap, Counters *cnt)
{
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
    FmPrev *scratch = scratch_all + (size_t) tid * stripe;
    const unsigned long long n = cnt->n_rtask < rtask_cap ? cnt->n_rtask : rtask_cap;
    unsigned n_ext = 0;
    for (unsigned long long t = tid; t < n; t += nthr) {
        const ReseedTask rt = rtasks[t];
        const int64_t o = offs[rt.read];
        const int len = (int) (offs[rt.read + 1] - o);
        PoolSink sink = { pool, pool_cap, tasks, task_cap, cnt, rt.read };
        QPlain q = { codes + o };
        fm_forward(fm, q, len, rt.x, rt.min_intv, true, scratch, sink, n_ext);
    }
    if (n_ext) atomicAdd(&cnt->n_ext, (unsigned long long) n_ext);
}

struct SmemAppend {
    bm2_smem *out; unsigned long long cap; Counters *cnt; uint32_t rid;
    ReseedTask *rtasks; unsigned long long rtask_cap; int split_len, split_width;      // rtasks == nullptr: no re-seeding (pass 2, 3)
    __device__ __forceinline__ void operator()(int m, int n, int64_t k, int64_t l, int64_t s) {
        unsigned long long i = atomicAdd(&cnt->n_smem, 1ULL);
        if (i < cap) { bm2_smem x; x.rid = rid; x.m = (uint32_t) m; x.n = (uint32_t) n; x.k = k; x.l = l; x.s = s; out[i] = x; }
        if (rtasks && n + 1 - m >= split_len && s <= split_width) {                 // src/bwamem.cpp:695-714
            unsigned long long t = atomicAdd(&cnt->n_rtask, 1ULL);
            if (t < rtask_cap) { ReseedTask r; r.read = (int32_t) rid; r.x = (n + 1 + m) >> 1; r.min_intv = (int32_t) (s + 1); rtasks[t] = r; }
        }
    }
};

// Backward phases: one search task per group of BWD_G lanes.  Per row (one base to the left) the lanes extend the
// entries of the interval list INDEPENDENTLY (one DRAM round trip per row instead of one per entry), then apply the
// collapsed keep/emit rule of fm_backward_rows with a ballot.  Lists of up to BWD_CAP entries live in shared memory.
#define BWD_G 8
#define BWD_CAP 32
__global__ void __launch_bounds__(128, 8)
smem_bwd_kernel(FmIndexView fm, SmemParams sp, const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs, int round,
                const SearchTask *__restrict__ tasks, unsigned long long task_cap, FmPrev *pool, unsigned long long pool_cap,
                bm2_smem *out, unsigned long long cap, ReseedTask *rtasks, unsigned long long rtask_cap, Counters *cnt)
{
    __shared__ FmPrev shl[128 / BWD_G][BWD_CAP];
    const int lane = threadIdx.x & 31, gl = lane & (BWD_G - 1), gw = lane / BWD_G;      // lane in group, group in warp
    const unsigned gmask = ((1u << BWD_G) - 1u) << (gw * BWD_G);
    const int grp = (blockIdx.x * blockDim.x + threadIdx.x) / BWD_G, ngrp = gridDim.x * blockDim.x / BWD_G;
    const unsigned long long t0 = round ? cnt->n_task1 : 0ULL;
    const unsigned long long t1 = cnt->n_task < task_cap ? cnt->n_task : task_cap;
    unsigned n_ext = 0;
    for (unsigned long long t = t0 + grp; t < t1; t += ngrp) {
        const SearchTask k = tasks[t];
        if ((unsigned long long) k.off + k.n > pool_cap) continue;                     // overflowed pool: the stage is re-run
        SmemAppend emit = { out, cap, cnt, (uint32_t) k.read, round ? nullptr : rtasks, rtask_cap, sp.split_len, sp.split_width };
        const uint8_t *q = codes + offs[k.read];
        FmPrev *lst = pool + k.off;
        int num_prev = k.n;
        if (num_prev <= BWD_CAP) {
            FmPrev *sl = shl[threadIdx.x / BWD_G];
            for (int p = gl; p < num_prev; p += BWD_G) sl[p] = lst[p];
            lst = sl;
        }
        __syncwarp(gmask);
        for (int j = k.x - 1; j >= 0 && num_prev > 0; --j) {
            const int a = q[j];
            if (a > 3) break;
            const FmPrev first = lst[0];
            __syncwarp(gmask);                                            // everyone has read entry 0 before it is overwritten
            // phase 1: independent extensions, results written back in place (k, l, s)
            int b = num_prev;
            for (int p = gl; p < num_prev; p += BWD_G) {
                FmIv req; req.k = lst[p].k; req.l = lst[p].l; req.s = lst[p].s;
                const FmIv r = fm_backward_ext(fm, req, a);
                ++n_ext;
                lst[p].k = r.k; lst[p].l = r.l; lst[p].s = r.s;
                if (r.s >= k.min_intv && p < b) b = p;
            }
#pragma unroll
            for (int d = BWD_G / 2; d > 0; d >>= 1) b = min(b, __shfl_xor_sync(gmask, b, d));
            __syncwarp(gmask);
            // phase 2: emit entry 0 if it died long enough; keep p >= b iff p == b or s[p] != s[p-1]; compact in place
            if (gl == 0 && b > 0 && first.n - first.m + 1 >= sp.min_seed_len) emit(first.m, first.n, first.k, first.l, first.s);
            int num_curr = 0;
            for (int base = b; base < num_prev; base += BWD_G) {
                const int p = base + gl;
                bool keep = false;
                FmPrev e;
                if (p < num_prev) { e = lst[p]; keep = (p == b) || (lst[p - 1].s != e.s); }
                const unsigned km = __ballot_sync(gmask, keep) >> (gw * BWD_G);
                __syncwarp(gmask);                                        // all reads of this round before any write
                if (keep) { e.m = j; lst[num_curr + __popc(km & ((1u << gl) - 1u))] = e; }
                num_curr += __popc(km);
                __syncwarp(gmask);
            }
            num_prev = num_curr;
        }
        if (gl == 0 && num_prev != 0) {
            const FmPrev s0 = lst[0];
            if (s0.n - s0.m + 1 >= sp.min_seed_len) emit(s0.m, s0.n, s0.k, s0.l, s0.s);
        }
        __syncwarp(gmask);
    }
    n_ext = __reduce_add_sync(0xffffffffu, n_ext);
    if (lane == 0 && n_ext) atomicAdd(&cnt->n_ext, (unsigned long long) n_ext);
}

__global__ void mark_task1_kernel(Counters *cnt) { if (threadIdx.x == 0 && blockIdx.x == 0) cnt->n_task1 = cnt->n_task; }

// A'. pass 3 (forward-only seeding) as its own kernel on a second stream: lean state, high occupancy
template <bool USE_SMEM>
__global__ void __launch_bounds__(128, 12)
smem_pass3_kernel(FmIndexView fm, SmemParams sp, const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs, int n_reads,
                  bm2_smem *out, unsigned long long cap, Counters *cnt)
{
    extern __shared__ uint32_t qsh[];
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
    unsigned n_ext = 0;
    for (int r = tid; r < n_reads; r += nthr) {
        const int64_t o = offs[r];
        const int len = (int) (offs[r + 1] - o);
        SmemAppend emit = { out, cap, cnt, (uint32_t) r, nullptr, 0, 0, 0 };
        if (USE_SMEM) {
            pack_read_smem(qsh, codes + o, len);
            QShared4 q = { (unsigned) __cvta_generic_to_shared(qsh + threadIdx.x), (unsigned) blockDim.x * 4u };
            fm_smem_pass3(fm, q, len, sp, emit, n_ext);
        } else {
            QPlain q = { codes + o };
            fm_smem_pass3(fm, q, len, sp, emit, n_ext);
        }
    }
    if (n_ext) atomicAdd(&cnt->n_ext, (unsigned long long) n_ext);
}

// B. sort keys: (rid, m, n) -> the order of sortSMEMs + ks_introsort(mem_intv1) (src/bwamem.cpp:785-799)
__global__ void smem_keys_kernel(const bm2_smem *sm, int64_t n, uint64_t *keys, uint32_t *vals) {
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = (uint64_t) sm[i].rid << 32 | (uint64_t) (sm[i].m & 0xFFFFu) << 16 | (uint64_t) (sm[i].n & 0xFFFFu);
    vals[i] = (uint32_t) i;
}

__global__ void smem_gather_kernel(const bm2_smem *in, const uint32_t *perm, int64_t n, int max_occ, bm2_smem *out, int64_t *slot_cnt) {
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bm2_smem x = in[perm[i]];
    out[i] = x;
    slot_cnt[i] = x.s < max_occ ? x.s : max_occ;          // rows sampled per SMEM (src/bwamem.cpp:892-893)
}

__global__ void read_smem_off_kernel(const uint64_t *keys_sorted, int64_t n_smem, int n_reads, int64_t *read_smem_off) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_reads) return;
    const uint64_t key = (uint64_t) r << 32;               // first SMEM with rid >= r
    int64_t lo = 0, hi = n_smem;
    while (lo < hi) { int64_t mid = (lo + hi) >> 1; if (keys_sorted[mid] < key) lo = mid + 1; else hi = mid; }
    read_smem_off[r] = lo;
}

// C. one seed slot per thread.  owner[slot] = index of the SMEM the slot belongs to, by a scatter of the SMEM
// indices to their first slot followed by an inclusive max-scan (no per-thread binary search over slot_off).
__global__ void slot_head_kernel(const int64_t *__restrict__ slot_off, int64_t n_smem, int32_t *owner) {
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_smem) return;
    if (slot_off[i + 1] > slot_off[i]) owner[slot_off[i]] = (int32_t) i;
}

__global__ void __launch_bounds__(256)
sa_kernel(FmIndexView fm, const bm2_smem *__restrict__ sm, const int64_t *__restrict__ slot_off, const int32_t *__restrict__ owner,
          int64_t n_slots, int max_occ, int64_t *sa, Counters *cnt)
{
    int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    int lf = 0;
    if (t < n_slots) {
        const int32_t o = owner[t];
        const bm2_smem x = sm[o];
        const int64_t step = x.s > max_occ ? x.s / max_occ : 1;
        sa[t] = fm_sa_of_row(fm, x.k + (t - slot_off[o]) * step, &lf);
    }
    // one atomic per warp (millions of same-address atomics per step are not free)
    lf = __reduce_add_sync(0xffffffffu, lf);
    if ((threadIdx.x & 31) == 0 && lf) atomicAdd(&cnt->n_lf, (unsigned long long) lf);
}

// D. one read per thread
struct ChainBufs {
    WSeed *wseed; WChain *wchain; int32_t *ord, *srt, *kv; int64_t *ordpos; FltRec *flt;
    bm2_chain *fin_chain; bm2_seed *fin_seed;
    int32_t *n_chain, *n_seed, *n_left, *n_right;
};

__global__ void __launch_bounds__(128)
chain_kernel(ContigView cv, ChainParams cp, const bm2_smem *__restrict__ sm, const int64_t *__restrict__ read_smem_off,
             const int64_t *__restrict__ slot_off, const int64_t *__restrict__ sa, const int64_t *__restrict__ offs, int n_reads,
             const int32_t *__restrict__ perm, ChainBufs b, SwParams sw, const uint8_t *__restrict__ ref, const uint8_t *__restrict__ codes,
             const int32_t *__restrict__ min_hsp, int mode, int heavy_thr, int coop_min, int light_sorted)
{
    // mode 0: light reads, one per thread; mode 1: heavy reads (many seed occurrences: O(n^2) chain insertion and
    // filtering), one per WARP, taken from the list sorted by decreasing work: lane 0 runs the sequential chaining, ALL lanes share the
    // local alignments of mem_flt_chained_seeds (long reads: hundreds of independent <= 200 x 200 alignments per read)
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const int stride = mode ? (gridDim.x * blockDim.x) >> 5 : gridDim.x * blockDim.x;
    for (int t = mode ? tid >> 5 : tid; t < n_reads; t += stride) {
    // (mode 0 with light_sorted: the light reads in work order too, so that the 32 reads of a warp have similar numbers of seed occurrences)
    const int r = (mode || light_sorted) ? perm[t] : t;
    {
        const int64_t nslot = slot_off[read_smem_off[r + 1]] - slot_off[read_smem_off[r]];
        if (mode) { if (nslot <= heavy_thr) break; }                  // perm is sorted by decreasing work (warp-uniform)
        else if (nslot > heavy_thr) continue;
    }
    int nk = 0, ns = 0, nl = 0, nr = 0;
    const int64_t sb = read_smem_off[r], se = read_smem_off[r + 1];
    const int len = (int) (offs[r + 1] - offs[r]);
    // reference quirk: a 512-read block whose SMEM total is exactly 1 yields no chain (src/bwamem.cpp:835)
    const int b0 = (r / 512) * 512, b1 = min(n_reads, b0 + 512);
    const bool skip = (read_smem_off[b1] - read_smem_off[b0]) <= 1;
    const bool lead = !mode || lane == 0;
    if (se > sb && !skip && len >= cp.min_seed_len) {
        const int64_t base = slot_off[sb];
        ChainStripe ws = { b.wseed + base, b.wchain + base, b.ord + base, b.ordpos + base, b.srt + base, b.kv + base, b.flt + base };
        float frac = 0.f;
        // reads with very many seed occurrences (long reads): all 32 lanes run the chaining on the same data and share its O(chains)
        // scans and shifts (ChainWarp); otherwise one thread runs it
        const bool coop = mode && (slot_off[se] - base) > coop_min;
        if (coop) { ChainWarp cw = { lane }; nk = chain_read_d(cv, cp, sm + sb, (int) (se - sb), sa + base, len, ws, &frac, cw); __syncwarp(); }
        else if (lead) nk = chain_read_d(cv, cp, sm + sb, (int) (se - sb), sa + base, len, ws, &frac);
        const bool flt = min_hsp && min_hsp[r] >= 0;
        if (!mode) {
            if (flt) chain_flt_seeds_d(cv, sw, ref, len, codes + offs[r], min_hsp[r], ws, nk);
        } else if (flt) {
            nk = __shfl_sync(0xffffffffu, nk, 0);
            int T = 0;
            if (lane == 0) T = chain_flt_list_d(ws, nk);
            T = __shfl_sync(0xffffffffu, T, 0);                      // (the shuffle also orders lane 0's writes before the others' reads)
            __syncwarp();
            chain_flt_score_d(cv, sw, ref, len, codes + offs[r], ws, T, lane, 32);
            __syncwarp();
            if (lane == 0) chain_flt_apply_d(sw, min_hsp[r], ws, nk);
        }
        if (lead) chain_finalize_d(ws, nk, frac, r, len, b.fin_chain + base, b.fin_seed + base, &ns, &nl, &nr);
    }
    if (lead) { b.n_chain[r] = nk; b.n_seed[r] = ns; b.n_left[r] = nl; b.n_right[r] = nr; }
    if (mode) __syncwarp();
    }
}


// E. compaction of the per-read stripes into flat arrays
__global__ void chain_compact_kernel(const int64_t *__restrict__ read_smem_off, const int64_t *__restrict__ slot_off, int n_reads,
                                     const bm2_chain *fin_chain, const bm2_seed *fin_seed, const int64_t *chain_off, const int64_t *reg_off,
                                     bm2_chain *chains, bm2_seed *seeds)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    const int64_t c0 = chain_off[r], c1 = chain_off[r + 1];
    if (c1 == c0) return;
    const int64_t base = slot_off[read_smem_off[r]];
    const int64_t s0 = reg_off[r], s1 = reg_off[r + 1];
    for (int64_t k = 0; k < c1 - c0; ++k) { bm2_chain c = fin_chain[base + k]; c.seed_off += (int32_t) s0; chains[c0 + k] = c; }
    for (int64_t k = 0; k < s1 - s0; ++k) { bm2_seed s = fin_seed[base + k]; s.chain += (int32_t) c0; seeds[s0 + k] = s; }
}

// F. one read per thread
struct ExtBufs {
    bm2_alnreg_t *regs; int32_t *reg_chain, *reg_seed; uint64_t *srt;
    ExtJobRec *left, *right; int32_t *left_reg, *right_reg;
    uint8_t *state;                  // per-reg extension state of the lazy extension (null: every job runs)
};

__global__ void __launch_bounds__(128)
ext_build_kernel(ContigView cv, ExtParams ep, const bm2_chain *__restrict__ chains, const bm2_seed *__restrict__ seeds,
                 const int64_t *__restrict__ chain_off, const int64_t *__restrict__ reg_off, const int64_t *__restrict__ left_off,
                 const int64_t *__restrict__ right_off, const int64_t *__restrict__ offs, int n_reads, const int32_t *__restrict__ perm, ExtBufs b)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_reads) return;
    const int r = perm[t];
    const int64_t c0 = chain_off[r], c1 = chain_off[r + 1];
    if (c1 == c0) return;
    const int64_t g0 = reg_off[r];
    ext_build_read_d(cv, ep, chains + c0, (int) (c1 - c0), seeds, (int) (offs[r + 1] - offs[r]), offs[r], c0, g0, b.regs + g0,
                     b.reg_chain + g0, b.reg_seed + g0, b.left + left_off[r], b.left_reg + left_off[r], b.right + right_off[r],
                     b.right_reg + right_off[r], b.srt + g0, b.state ? b.state + g0 : nullptr);
}

// G/H. fold one finished job into its reg; rejected jobs are appended to the retry list
__global__ void right_h0_kernel(ExtJobRec *jobs, const int32_t *job_reg, int n, const bm2_alnreg_t *regs) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) jobs[i].h0 = regs[job_reg[i]].score;       // src/bwamem.cpp:2672-2677
}

__global__ void fold_kernel(ExtParams ep, const ExtJobRec *jobs, const int32_t *job_reg, const BswOut *outs, const int32_t *sel, int n,
                            int is_right, int w, int last_try, bm2_alnreg_t *regs, const int32_t *reg_chain, const bm2_chain *chains,
                            const bm2_seed *seeds, const int64_t *offs, int32_t *retry, Counters *cnt)
{
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int j = sel ? sel[t] : t;                        // job index; outs[] is indexed like the launch (t)
    const BswOut o = outs[t];
    const int g = job_reg[j];
    const bm2_chain c = chains[reg_chain[g]];
    const int l_query = (int) (offs[c.seqid + 1] - offs[c.seqid]);
    bm2_alnreg_t a = regs[g];
    const bool ok = ext_fold_d(ep, a, is_right, jobs[j].h0, o.score, o.qle, o.tle, o.gtle, o.gscore, o.max_off, w, last_try, l_query,
                               seeds + c.seed_off, c.n_seeds);
    regs[g] = a;
    if (!ok) { unsigned long long k = atomicAdd(&cnt->n_retry, 1ULL); retry[k] = j; }
}

__global__ void gather_jobs_kernel(const ExtJobRec *jobs, const int32_t *sel, int n, ExtJobRec *out) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) out[t] = jobs[sel[t]];
}

// ---- lazy extension (ext_walk_read_d, ext_device.cuh): the extension runs in waves ------------------------------------------------
// The jobs of one wave: those whose reg is EXT_NEED or, in the last wave, any reg not extended yet (EXT_TODO), appended with their reg
// ids to a compact list, one atomic per warp.  The order of the list does not matter: the extension kernels sort their jobs by size.
__global__ void ext_select_kernel(const ExtJobRec *__restrict__ jobs, const int32_t *__restrict__ job_reg, int n,
                                  const uint8_t *__restrict__ state, int last, ExtJobRec *out, int32_t *out_reg, unsigned long long *n_out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
    int g = 0;
    bool take = false;
    if (i < n) { g = job_reg[i]; const uint8_t s = state[g]; take = s == EXT_NEED || (last && s == EXT_TODO); }
    const unsigned m = __ballot_sync(0xffffffffu, take);
    if (!m) return;
    const int leader = __ffs(m) - 1;
    unsigned long long at = 0;
    if (lane == leader) at = atomicAdd(n_out, (unsigned long long) __popc(m));
    at = __shfl_sync(0xffffffffu, at, leader);
    if (take) { const unsigned long long k = at + __popc(m & ((1u << lane) - 1u)); out[k] = jobs[i]; out_reg[k] = g; }
}

// after a wave: its regs are extended
__global__ void ext_mark_done_kernel(uint8_t *state, int64_t n) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && state[i] == EXT_NEED) state[i] = EXT_DONE;
}

// The scan of pf_seed_purged_d by a whole warp: the same v, for seed s against box[0..n_reg) with lim kept regs so far.  The
// scan - O(regs) per seed, O(regs^2) per read - is split over the lanes, 32 boxes per step: each lane classifies its box as skipped /
// counted (v++) / hit (break), and a ballot pair per step goes to pf_scan_step_d, which stops where the sequential loop stops.
// The boxes of FOUR steps are classified before the first of them is resolved (the loads and tests of a lane's four boxes overlap; a read
// inside a high-copy repeat has thousands of regs and its scan - one dependent load -> test -> ballot chain per step - is the critical path
// of the kernels that call this); the resolution keeps the sequential loop's order.  Called by all lanes with the same arguments.
__device__ int pf_scan_warp(const ExtParams &p, const bm2_seed &s, const PfBox *box, int n_reg, int lim, int l_query)
{
    const int lane = threadIdx.x & 31;
    int v = 0;
    bool stop = false;
    for (int i0 = 0; i0 < n_reg && v < lim && !stop; i0 += 128) {
        int kind[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            const int i = i0 + 32 * g + lane;
            kind[g] = i < n_reg ? pf_box_kind_d(p, s, box[i], l_query) : 0;      // 0 skipped, 1 counted, 2 hit
        }
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            const unsigned cm = __ballot_sync(0xFFFFFFFFu, kind[g] == 1), hm = __ballot_sync(0xFFFFFFFFu, kind[g] == 2);
            if (!stop) stop = pf_scan_step_d(cm, hm, v, lim);       // (warp-uniform: the ballots above are taken by all lanes)
        }
    }
    return v;
}

// ext_walk_read_d by a whole warp, for the reads with many regs: the same decisions, states, srt2, boxes and cursor.  The box scan runs
// on all lanes (pf_scan_warp); every lane computes the same decision, and lane 0 writes state, srt2 and box.  Called by all lanes.
__device__ bool ext_walk_read_warp(const ExtParams &p, const bm2_chain *chains, int n_chain, const bm2_seed *seeds, int l_query,
                                   const bm2_alnreg_t *regs, const int32_t *reg_seed, uint8_t *state, int32_t *srt2, PfBox *box, PfCursor &cur)
{
    const int lane = threadIdx.x & 31;
    int ci = cur.ci, k = cur.k, lim = cur.lim, base = cur.base;
    for (; ci < n_chain; ++ci, k = -1) {
        const bm2_chain &c = chains[ci];
        const bm2_seed *cs = seeds + c.seed_off;
        const int n = c.n_seeds;
        if (n == 0) continue;
        if (k < 0) {
            for (int kk = n - 1 - lane; kk >= 0; kk -= 32) srt2[kk] = reg_seed[base + (n - 1 - kk)];
            __syncwarp();
            k = n - 1;
        }
        for (; k >= 0; --k) {
            const int ai = base + (n - 1 - k);
            const bm2_seed s = cs[srt2[k]];
            // the scan ends before box[ai]: the lim kept regs are all earlier ones, and the boxes from ai on are not written yet
            const bool purged = pf_scan_warp(p, s, box, ai, lim, l_query) < lim && !pf_chain_overlap_d(cs, n, srt2, k, s);
            const uint8_t st = state[ai];
            __syncwarp();
            if (purged) {
                if (lane == 0) { box[ai].qb = box[ai].qe = -1; srt2[k] = -1; if (st != EXT_DONE) state[ai] = EXT_SKIP; }
                __syncwarp();
                continue;
            }
            if (st != EXT_DONE) {
                if (lane == 0) state[ai] = EXT_NEED;
                cur.ci = ci; cur.k = k; cur.lim = lim; cur.base = base;
                return false;
            }
            if (lane == 0) box[ai] = pf_box_d(regs[ai]);
            __syncwarp();
            lim++;
        }
        base += n;
    }
    cur.ci = ci; cur.k = -1; cur.lim = lim; cur.base = base;
    return true;
}

// The post-filter walk, resumed from cur[r] (first: from the start).  Reads with at most heavy_thr regs are walked one per thread, in input
// order (mode 0); the others one per warp (mode 1), in perm's order of decreasing regs, so that the heaviest start first.
template <int mode>
__global__ void __launch_bounds__(128)
ext_walk_kernel(ExtParams ep, const bm2_chain *__restrict__ chains, const bm2_seed *__restrict__ seeds, const int64_t *__restrict__ chain_off,
                const int64_t *__restrict__ reg_off, const int64_t *__restrict__ offs, int n_reads, const bm2_alnreg_t *regs,
                const int32_t *__restrict__ reg_seed, uint8_t *state, int32_t *srt2_all, PfBox *box_all, PfCursor *cur,
                const int32_t *__restrict__ perm, int heavy_thr, int first, Counters *cnt)
{
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    const int unit = mode ? tid >> 5 : tid, nunit = mode ? nthr >> 5 : nthr;
    unsigned n_done = 0;
    for (int t = unit; t < n_reads; t += nunit) {
        const int r = mode ? perm[t] : t;
        const int64_t c0 = chain_off[r], g0 = reg_off[r];
        const int n_reg = (int) (reg_off[r + 1] - g0), n_chain = (int) (chain_off[r + 1] - c0);
        if (mode) { if (n_reg <= heavy_thr) break; }       // perm is sorted by decreasing n_reg
        else if (n_reg > heavy_thr) continue;
        if (n_chain == 0) continue;
        PfCursor c;
        if (first) { c.ci = 0; c.k = -1; c.lim = 0; c.base = 0; } else c = cur[r];
        if (c.ci >= n_chain) continue;
        const int l_query = (int) (offs[r + 1] - offs[r]);
        bool done;
        if (mode) done = ext_walk_read_warp(ep, chains + c0, n_chain, seeds, l_query, regs + g0, reg_seed + g0, state + g0, srt2_all + g0, box_all + g0, c);
        else done = ext_walk_read_d(ep, chains + c0, n_chain, seeds, l_query, regs + g0, n_reg, reg_seed + g0, state + g0, srt2_all + g0, box_all + g0, c);
        if (!mode || lane == 0) { cur[r] = c; n_done += done; }
    }
    if (first) {
        n_done = __reduce_add_sync(0xffffffffu, n_done);
        if (lane == 0 && n_done) atomicAdd(&cnt->n_walk_done, (unsigned long long) n_done);
    }
}

// Post-filter of one read by a whole warp (same result as ext_postfilter_read_d, src/bwamem.cpp:2895-2989): the box scan of each seed
// is pf_scan_warp; the rest runs on every lane, and lane 0 writes.
__device__ void ext_postfilter_read_warp(const ExtParams &p, const bm2_chain *chains, int n_chain, const bm2_seed *seeds, int l_query,
                                         bm2_alnreg_t *regs, int n_reg, const int32_t *reg_seed, int32_t *srt2, PfBox *box)
{
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < n_reg; i += 32) box[i] = pf_box_d(regs[i]);
    __syncwarp();
    int lim = 0, base = 0;
    for (int ci = 0; ci < n_chain; ++ci) {
        const bm2_chain &c = chains[ci];
        const bm2_seed *cs = seeds + c.seed_off;
        const int n = c.n_seeds;
        if (n == 0) continue;
        for (int k = n - 1 - lane; k >= 0; k -= 32) srt2[k] = reg_seed[base + (n - 1 - k)];
        __syncwarp();
        for (int k = n - 1; k >= 0; --k) {
            const bm2_seed s = cs[srt2[k]];
            const int v = pf_scan_warp(p, s, box, n_reg, lim, l_query);
            if (v < lim) {
                if (!pf_chain_overlap_d(cs, n, srt2, k, s)) {
                    __syncwarp();
                    if (lane == 0) {
                        const int ai = base + (n - 1 - k);
                        regs[ai].qb = regs[ai].qe = -1;
                        box[ai].qb = box[ai].qe = -1;
                        srt2[k] = -1;
                    }
                    __syncwarp();
                    continue;
                }
            }
            lim++;
        }
        __syncwarp();
        base += n;
    }
}

// ---- the tail of one heavy read by a whole warp ---------------------------------------------------------------------------------
// Same result as ext_tail_read_d (ext_device.cuh; src/bwamem.cpp:1141-1169 + mem_sort_dedup_patch, :292-353).  The passes that touch every record
// once - the three compactions, the key arrays of the two sorts, the two in-place permutations, n_comp = 1, the equal-neighbour test, the ALT
// marks - run on all lanes (ncu r2i: they were 36 % of the heavy pass's samples with ONE lane active); the two introsorts and the
// dedup / patch scan, whose steps depend on each other, stay on lane 0.

// keep the records with qe > qb, in order, in place; returns the count.  A block of 32 records is read completely before any of it is written,
// and a record only moves towards the front.
__device__ int tail_compact_warp(bm2_alnreg_t *a, int n, int lane) {
    int m = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        uint4 v[7];
        bool keep = false;
        if (i < n) {
            const uint4 *s4 = reinterpret_cast<const uint4 *>(a + i);
#pragma unroll
            for (int k = 0; k < 7; ++k) v[k] = s4[k];
            keep = a[i].qe > a[i].qb;
        }
        const unsigned km = __ballot_sync(0xffffffffu, keep);
        __syncwarp();
        if (keep) {
            const int d = m + __popc(km & ((1u << lane) - 1u));
            if (d != i) {
                uint4 *d4 = reinterpret_cast<uint4 *>(a + d);
#pragma unroll
                for (int k = 0; k < 7; ++k) d4[k] = v[k];
            }
        }
        m += __popc(km);
        __syncwarp();
    }
    return m;
}

// a[i] <- a[idx[i]] in place (permute_regs_d's cycle walk, every lane walking the same cycle); lanes 0..6 move one 16-byte word of the
// record each, the displaced first record of a cycle waits in their registers; idx is destroyed
__device__ void tail_permute_warp(bm2_alnreg_t *a, int32_t *idx, int n, int lane) {
    for (int i = 0; i < n; ++i) {
        const int first = idx[i];
        if (first < 0 || first == i) continue;
        uint4 tmp = make_uint4(0, 0, 0, 0);
        if (lane < 7) tmp = reinterpret_cast<const uint4 *>(a + i)[lane];
        int j = i;
        for (;;) {
            const int src = idx[j];
            __syncwarp();
            if (lane == 0) idx[j] = -1;
            if (src == i) { if (lane < 7) reinterpret_cast<uint4 *>(a + j)[lane] = tmp; break; }
            if (lane < 7) reinterpret_cast<uint4 *>(a + j)[lane] = reinterpret_cast<const uint4 *>(a + src)[lane];
            j = src;
        }
        __syncwarp();
    }
}

__device__ int ext_tail_read_warp(const ContigView &cv, const ExtParams &p, const uint8_t *ref, const uint8_t *query, bm2_alnreg_t *a, int n_reg,
                                  int32_t *he, int32_t *idx, TailSortKey *keys)
{
    const int lane = threadIdx.x & 31;
    int n = tail_compact_warp(a, n_reg, lane);
    if (n > 1) {
        for (int i = lane; i < n; i += 32) { idx[i] = i; keys[i].r = a[i].re; }
        __syncwarp();
        if (lane == 0) {
            const TailSortKey *rk = keys;
            ks_introsort_d(idx, (long) n, [rk](int x, int y) { return rk[x].r < rk[y].r; });
        }
        __syncwarp();
        tail_permute_warp(a, idx, n, lane);
        for (int i = lane; i < n; i += 32) reg_set_n_comp_d(a[i], 1);
        __syncwarp();
        if (lane == 0) sort_dedup_scan_d(cv, p, ref, query, n, a, he);
        __syncwarp();
        n = tail_compact_warp(a, n, lane);
        for (int i = lane; i < n; i += 32) { idx[i] = i; keys[i].r = a[i].rb; keys[i].score = a[i].score; keys[i].qb = a[i].qb; }
        __syncwarp();
        if (lane == 0) {
            const TailSortKey *rk = keys;
            ks_introsort_d(idx, (long) n, [rk](int xi, int yi) {
                const TailSortKey x = rk[xi], y = rk[yi];
                return x.score > y.score || (x.score == y.score && (x.r < y.r || (x.r == y.r && x.qb < y.qb)));
            });
        }
        __syncwarp();
        tail_permute_warp(a, idx, n, lane);
        // equal neighbours (score, rb, qb): the test reads fields the marking does not change, so all pairs are independent
        for (int i0 = 0; i0 < n; i0 += 32) {
            const int i = i0 + lane;
            const bool dup = i >= 1 && i < n && a[i].score == a[i - 1].score && a[i].rb == a[i - 1].rb && a[i].qb == a[i - 1].qb;
            __syncwarp();
            if (dup) a[i].qe = a[i].qb;
        }
        __syncwarp();
        // (the reference's last compaction starts at index 1: a[0] stays whatever its qe is)
        if (n > 1) n = 1 + tail_compact_warp(a + 1, n - 1, lane);
    }
    for (int i = lane; i < n; i += 32)
        if (a[i].rid >= 0 && cv.ann_alt && cv.ann_alt[a[i].rid]) reg_set_is_alt_d(a[i], 1);
    __syncwarp();
    return n;
}

// I. one read per thread (grid-stride: the NW scratch `he` is per thread)
template <int mode>             // separate instances: the warp-per-read code (more registers) must not cost the per-thread pass its occupancy (96)
// (mode 1 at 4 CTAs per SM = 128 registers.  Compiled for 6 / 8 CTAs - 80 / 64 registers, 350-470 B of spills - it was no faster: 13.0 / 13.4 against
// no faster in an A/B: more resident warps do not help this kernel.)
__global__ void __launch_bounds__(128, mode ? 4 : 1)
tail_kernel(ContigView cv, ExtParams ep, const uint8_t *__restrict__ ref, const uint8_t *__restrict__ codes, const int64_t *__restrict__ offs,
            const bm2_chain *__restrict__ chains, const bm2_seed *__restrict__ seeds, const int64_t *__restrict__ chain_off,
            const int64_t *__restrict__ reg_off, int n_reads, bm2_alnreg_t *regs, const int32_t *reg_seed, int32_t *srt2_all, int32_t *he_all,
            int he_stride, const int32_t *__restrict__ perm, PfBox *box_all, int32_t *n_final, int heavy_thr, int light_sorted, int coop_tail)
{
    // Heavy reads (many regs: O(regs^2) post-filter, sorts, patch DP) would serialise with the 31 other reads of their
    // warp (ncu: 1.9 active lanes per instruction), so they get a WARP each (mode 1: reads in decreasing-work order; the
    // post-filter scan runs on all lanes, the rest on lane 0); light reads run one per thread (mode 0).
    // (The heavy reads in SHARED memory - records, sort keys and index array copied in and out by the warp - were no faster at the
    // same number of resident warps, and slower with fewer: the
    // records of one read stay in L1 between lane 0's passes, so the sequential part is bound by its instructions, not by memory latency.)
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    int32_t *he = he_all + (size_t) (mode ? tid >> 5 : tid) * he_stride;
    const int unit = mode ? tid >> 5 : tid, nunit = mode ? nthr >> 5 : nthr;
    for (int t = unit; t < n_reads; t += nunit) {
        const int r = (mode || light_sorted) ? perm[t] : t;      // (the light reads in work order too: similar reads share a warp)
        const int64_t c0 = chain_off[r], c1 = chain_off[r + 1], g0 = reg_off[r];
        const int n_reg = (int) (reg_off[r + 1] - g0);
        if (mode) { if (n_reg <= heavy_thr) break; }       // perm is sorted by decreasing n_reg
        else if (n_reg > heavy_thr) continue;
        int m = 0;
        if (c1 > c0) {
            const int l_query = (int) (offs[r + 1] - offs[r]);
            if (mode) {
                ext_postfilter_read_warp(ep, chains + c0, (int) (c1 - c0), seeds, l_query, regs + g0, n_reg, reg_seed + g0, srt2_all + g0, box_all + g0);
                __syncwarp();
                if (coop_tail) m = ext_tail_read_warp(cv, ep, ref, codes + offs[r], regs + g0, n_reg, he, srt2_all + g0, reinterpret_cast<TailSortKey *>(box_all + g0));
                else if (lane == 0) m = ext_tail_read_d(cv, ep, ref, codes + offs[r], regs + g0, n_reg, he, srt2_all + g0, reinterpret_cast<TailSortKey *>(box_all + g0));
                __syncwarp();
            } else {
                ext_postfilter_read_d(ep, chains + c0, (int) (c1 - c0), seeds, l_query, regs + g0, n_reg, reg_seed + g0, srt2_all + g0, box_all + g0);
                m = ext_tail_read_d(cv, ep, ref, codes + offs[r], regs + g0, n_reg, he, srt2_all + g0, reinterpret_cast<TailSortKey *>(box_all + g0));
            }
        }
        if (!mode || lane == 0) n_final[r] = m;
    }
}

__global__ void regs_gather_kernel(const bm2_alnreg_t *regs, const int64_t *reg_off, const int64_t *out_off, int n_reads, bm2_alnreg_t *out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    const int64_t o0 = out_off[r], o1 = out_off[r + 1], g0 = reg_off[r];
    for (int64_t k = 0; k < o1 - o0; ++k) reg_copy(&out[o0 + k], &regs[g0 + k]);
}

// reads ordered by decreasing work (heavy reads first, similar reads share a warp)
__global__ void work_keys_slots_kernel(const int64_t *read_smem_off, const int64_t *slot_off, int n, uint32_t *keys, int32_t *vals) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    int64_t w = slot_off[read_smem_off[r + 1]] - slot_off[read_smem_off[r]];
    keys[r] = 0xFFFFFFFFu - (uint32_t) (w > 0x7FFFFFFF ? 0x7FFFFFFF : w);
    vals[r] = r;
}
__global__ void work_keys_off_kernel(const int64_t *off, int n, uint32_t *keys, int32_t *vals) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    int64_t w = off[r + 1] - off[r];
    keys[r] = 0xFFFFFFFFu - (uint32_t) (w > 0x7FFFFFFF ? 0x7FFFFFFF : w);
    vals[r] = r;
}

__global__ void widen_kernel(const int32_t *in, int n, int64_t *out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i];
    if (i == n) out[i] = 0;
}

// ------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------
namespace {
enum Buf {
    B_CODES, B_OFFS, B_CNT, B_PREV, B_SMEM_RAW, B_KEYS_IN, B_KEYS_OUT, B_VALS_IN, B_VALS_OUT, B_CUB, B_SMEM, B_SLOT_CNT,
    B_SLOT_OFF, B_READ_SMEM_OFF, B_SA, B_WSEED, B_WCHAIN, B_ORD, B_SRT, B_KV, B_FIN_CHAIN, B_FIN_SEED, B_PER_READ, B_SCAN, B_CHAINS,
    B_SEEDS, B_REGS, B_REG_AUX, B_JOBS, B_NW, B_OUT, B_PERM, B_ORDPOS, B_FLT, B_MINHSP, B_OWNER, B_POOL, B_TASKS, B_RTASKS, B_COUNT_
};
enum HBuf { H_OUT_REGS, H_OUT_OFF, H_SMEM, H_CHAINS, H_SEEDS, H_COUNT_ };
static_assert(B_COUNT_ == std::extent<decltype(bm2_ctx::pipe_d)>::value, "bm2_ctx::pipe_d: one buffer per slot");
static_assert(H_COUNT_ == std::extent<decltype(bm2_ctx::pipe_h)>::value, "bm2_ctx::pipe_h: one buffer per slot");

struct Stages {
    bm2_ctx *ctx; std::vector<cudaEvent_t> &ev; std::vector<const char *> &names;
    int n = 0;
    int mark(const char *name) {
        bm2_ctx *ctx_for_error = ctx;
        if ((int) ev.size() <= n) { cudaEvent_t e; BM2_CUDA_OK(cudaEventCreate(&e)); ev.push_back(e); }
        BM2_CUDA_OK(cudaEventRecord(ev[n], ctx->stream));
        if ((int) names.size() <= n) names.push_back(name); else names[n] = name;
        ++n;
        return 0;
    }
};

template <class T> T *P(bm2_ctx *ctx, int b) { return (T *) ctx->pipe_d[b].p; }

}  // namespace

namespace {

struct Params { FmIndexView fm; ContigView cv; SmemParams sp; ChainParams cp; ExtParams ep; SwParams sw; };

Params make_params(const bm2_ctx *ctx) {
    Params v;
    const DevIndex &d = ctx->idx; const bm2_mem_opt_t &o = ctx->opt;
    v.fm.cp_occ = d.cp_occ; v.fm.layout = d.occ_layout; v.fm.sa_ms = d.sa_ms; v.fm.sa_ls = d.sa_ls; v.fm.sentinel = d.sentinel;
    for (int i = 0; i < 5; ++i) v.fm.count[i] = d.count[i];
    v.cv.l_pac = d.l_pac; v.cv.n_seqs = d.n_seqs; v.cv.ann_off = d.ann_off; v.cv.ann_len = d.ann_len; v.cv.ann_alt = d.ann_alt;
    v.sp.min_seed_len = o.min_seed_len; v.sp.split_len = (int) (o.min_seed_len * o.split_factor + .499);
    v.sp.split_width = o.split_width; v.sp.max_mem_intv = (int) o.max_mem_intv;
    v.cp.w = o.w; v.cp.max_chain_gap = o.max_chain_gap; v.cp.max_occ = o.max_occ; v.cp.min_chain_weight = o.min_chain_weight;
    v.cp.max_chain_extend = o.max_chain_extend; v.cp.min_seed_len = o.min_seed_len; v.cp.mask_level = o.mask_level; v.cp.drop_ratio = o.drop_ratio;
    v.ep.a = o.a; v.ep.b = o.b; v.ep.o_del = o.o_del; v.ep.e_del = o.e_del; v.ep.o_ins = o.o_ins; v.ep.e_ins = o.e_ins; v.ep.w = o.w;
    v.ep.pen_clip5 = o.pen_clip5; v.ep.pen_clip3 = o.pen_clip3; v.ep.max_chain_gap = o.max_chain_gap; v.ep.mask_level_redun = o.mask_level_redun;
    memcpy(v.ep.mat, o.mat, 25);
    v.sw.a = o.a; v.sw.o_del = o.o_del; v.sw.e_del = o.e_del; v.sw.o_ins = o.o_ins; v.sw.e_ins = o.e_ins; memcpy(v.sw.mat, o.mat, 25);
    return v;
}

inline size_t al(size_t x) { return (x + 255) / 256 * 256; }

// tuning knobs read from the environment at every batch (experiments toggle them between calls of one process)
inline int env_int(const char *name, int def, int lo, int hi) {
    const char *e = getenv(name);
    if (!e || !*e) return def;
    const int v = atoi(e);
    return v < lo ? lo : (v > hi ? hi : v);
}

// exclusive scan of n int64 counts into n+1 offsets (last = total)
int scan64(bm2_ctx *ctx, const int64_t *in, int64_t *out, int64_t n) {
    bm2_ctx *ctx_for_error = ctx;
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int) (n + 1));
    if (ctx->ensure(ctx->pipe_d[B_CUB], bytes)) return 1;
    BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(ctx->pipe_d[B_CUB].p, bytes, in, out, (int) (n + 1), ctx->stream));
    return 0;
}

// sorts (keys, vals) of n reads; result permutation in vals_out
// Measured: grouping heavy reads into the same warps makes the thread-per-read
// chain/tail kernels 2-7x SLOWER (32 private n^2 scans per warp thrash L1/L2), so until those kernels are
// warp-cooperative the reads keep their input order (the permutation is the identity).
static const bool kSortReadsByWork = false;

int sort_work(bm2_ctx *ctx, uint32_t *keys_in, uint32_t *keys_out, int32_t *vals_in, int32_t *vals_out, int n, bool force = false) {
    bm2_ctx *ctx_for_error = ctx;
    if (!kSortReadsByWork && !force) {
        BM2_CUDA_OK(cudaMemcpyAsync(vals_out, vals_in, (size_t) n * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        return 0;
    }
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys_in, keys_out, vals_in, vals_out, n);
    if (ctx->ensure(ctx->pipe_d[B_CUB], bytes)) return 1;
    BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(ctx->pipe_d[B_CUB].p, bytes, keys_in, keys_out, vals_in, vals_out, n, 0, 32, ctx->stream));
    return 0;
}

enum UpTo { UPTO_SMEM, UPTO_CHAIN, UPTO_REGS };

// A stage token of the parent context, held while a lane's stage is enqueued and until its closing host sync.
struct StageToken {
    std::mutex *m;
    explicit StageToken(std::mutex *mu) : m(mu) { if (m) m->lock(); }
    ~StageToken() { release(); }
    void release() { if (m) { m->unlock(); m = nullptr; } }
    StageToken(const StageToken &) = delete; StageToken &operator=(const StageToken &) = delete;
};

struct BatchState {       // host-visible sizes of the batch in flight
    int n = 0, max_len = 0; int64_t n_smem = 0, n_slots = 0, n_chains = 0, n_regs = 0, n_left = 0, n_right = 0, n_out = 0;
};

int run_pipeline(bm2_ctx *ctx, const bm2_read_batch *rb, UpTo upto, BatchState &bs, const uint8_t *ext_codes = nullptr,
                 const int64_t *ext_offs = nullptr, bool copy_out = true) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx->idx.loaded) { bm2_set_error(ctx, "seam 2 needs a context created with an index"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const int n = rb->n_reads;
    bs = BatchState(); bs.n = n;
    if (n <= 0) return 0;
    const int64_t total = rb->offsets[n];
    int max_len = 1;
    bool any_flt = false;
    std::vector<int32_t> min_hsp_host;
    {
        // mem_flt_chained_seeds (src/bwamem.cpp:472-504) applies to reads with min_l <= 0.05 * l (>= 725 bp by default):
        // min_HSP_score is computed here with the reference's double arithmetic (log() on the host), once per distinct
        // consecutive length (a batch of equal-length reads costs one log(), not a million)
        int64_t memo_l = -1; int memo_hsp = -1;
        for (int r = 0; r < n; ++r) {
            const int64_t l = rb->offsets[r + 1] - rb->offsets[r];
            if (l < 0 || l > 32767) { bm2_set_error(ctx, "read length out of range (0..32767)"); return 1; }
            if (l > max_len) max_len = (int) l;
            if (l != memo_l) {
                const double min_l = ctx->opt.min_chain_weight ? 1.1f * ctx->opt.min_chain_weight : 5.5f * log((double) (l > 0 ? l : 1));
                memo_l = l; memo_hsp = -1;
                if (l > 0 && !(min_l > 0.05f * l)) memo_hsp = (int) (ctx->opt.a * min_l + .499);
            }
            if (memo_hsp >= 0 && !any_flt) { any_flt = true; min_hsp_host.assign((size_t) n, -1); }
            if (any_flt) min_hsp_host[r] = memo_hsp;
        }
    }
    bs.max_len = max_len;
    Params pv = make_params(ctx);
    // unique-interval shortcut of the forward SMEM passes (fm_device.cuh): on for the whole-path entries; the staged bm2_collect_smems entry,
    // whose callers see the SMEMs' l values, runs the plain search (BM2_SMEM_TEXT=0 turns it off everywhere: A/B measurements)
    if (upto != UPTO_SMEM && env_int("BM2_SMEM_TEXT", 1, 0, 1)) { pv.fm.text = ctx->idx.ref; pv.fm.text_len = 2 * ctx->idx.l_pac; }
    Stages sg = { ctx, ctx->events, ctx->stage_names };
    if (sg.mark("h2d")) return 1;

    if (ctx->ensure(ctx->pipe_d[B_CNT], sizeof(Counters))) return 1;
    const uint8_t *d_codes = ext_codes; const int64_t *d_offs = ext_offs;
    if (!ext_codes) {
        if (ctx->ensure(ctx->pipe_d[B_CODES], (size_t) total + 16)) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(ctx->pipe_d[B_CODES].p, rb->codes, (size_t) total, cudaMemcpyHostToDevice, st));
        d_codes = P<uint8_t>(ctx, B_CODES);
    }
    if (!ext_offs) {     // (a sub-batch of a device-resident batch brings its codes pointer but re-based offsets from the host)
        if (ctx->ensure(ctx->pipe_d[B_OFFS], (size_t) (n + 1) * 8)) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(ctx->pipe_d[B_OFFS].p, rb->offsets, (size_t) (n + 1) * 8, cudaMemcpyHostToDevice, st));
        d_offs = P<int64_t>(ctx, B_OFFS);
    }
    if (any_flt) {
        if (ctx->ensure(ctx->pipe_d[B_MINHSP], (size_t) n * 4)) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(ctx->pipe_d[B_MINHSP].p, min_hsp_host.data(), (size_t) n * 4, cudaMemcpyHostToDevice, st));
    }
    BM2_CUDA_OK(cudaMemsetAsync(ctx->pipe_d[B_CNT].p, 0, sizeof(Counters), st));
    Counters *d_cnt = P<Counters>(ctx, B_CNT);
    Counters h_cnt;

    // ---- A. SMEMs -------------------------------------------------------------------------------------------
    if (sg.mark("smem")) return 1;
    const int stripe = max_len + 2;
    // CTAs per SM the SMEM kernels' grids may occupy (BM2_SMEM_CTAS): fewer leave room for the extension kernels of
    // the other sub-batches in flight (memory-latency-bound search next to ALU-bound DP on the same SM)
    // 8 CTAs/SM for the unsplit batch was faster than 6 or 10 in an A/B (the stage sits on the random-access roofline of HBM: more
    // searches in flight only thrash L2 / the DRAM pages); four sub-batch lanes with 3-4 CTAs/SM each were faster than with 10.
    const int use_tokens = ctx->parent ? env_int("BM2_STAGE_TOKENS", 0, 0, 3) : 0;
    // (with the SMEM token only one lane is in the SMEM stage at a time: it gets the unsplit batch's 8 CTAs per SM)
    const int smem_ctas = env_int("BM2_SMEM_CTAS", (ctx->parent && !(use_tokens & 1)) ? 4 : 8, 1, 16);
    int blocks_a = (n + 127) / 128; int max_blocks_a = ctx->n_sm * smem_ctas;
    {   // per-thread forward scratch = stripe * 32 bytes: keep it under ~8 GB for long reads
        const size_t per_block = (size_t) 128 * stripe * sizeof(FmPrev);
        const size_t fit = ((size_t) 8 << 30) / per_block;
        if ((size_t) max_blocks_a > fit) max_blocks_a = (int) (fit > (size_t) ctx->n_sm ? fit : (size_t) ctx->n_sm);
    }
    if (blocks_a > max_blocks_a) blocks_a = max_blocks_a;
    const size_t thr_a = (size_t) blocks_a * 128;
    if (ctx->ensure(ctx->pipe_d[B_PREV], thr_a * stripe * sizeof(FmPrev))) return 1;
    // capacities grow from the counters when a batch overflows them (then the stage is re-run)
    const double rl = (double) total / n;                                  // mean read length
    unsigned long long cap = (unsigned long long) n * 16 + 4096;
    unsigned long long pool_cap = (unsigned long long) (n * (rl * 1.7 + 64)) + 65536;
    unsigned long long task_cap = (unsigned long long) (n * (rl / 12 + 8)) + 4096;
    unsigned long long rtask_cap = (unsigned long long) n * 8 + 4096;
    const bool q_smem = max_len <= 256;
    const size_t qsm = q_smem ? (size_t) ((max_len + 7) / 8) * 128 * 4 : 0;
    const int blocks_b = ctx->n_sm * smem_ctas;
    // BM2_STAGE_TOKENS: bit 0 = SMEM-stage token, bit 1 = extension-stage token (sub-batch lanes only).  Off by default:
    // slower in an A/B - taking turns in
    // a stage leaves the other lanes' host threads waiting at the token instead of queueing work.
    StageToken tok_smem((use_tokens & 1) ? &ctx->parent->tok_smem : nullptr);
    for (int attempt = 0; attempt < 3; ++attempt) {
        if (ctx->ensure(ctx->pipe_d[B_SMEM_RAW], cap * sizeof(bm2_smem)) || ctx->ensure(ctx->pipe_d[B_POOL], pool_cap * sizeof(FmPrev)) ||
            ctx->ensure(ctx->pipe_d[B_TASKS], task_cap * sizeof(SearchTask)) || ctx->ensure(ctx->pipe_d[B_RTASKS], rtask_cap * sizeof(ReseedTask))) return 1;
        BM2_CUDA_OK(cudaMemsetAsync(d_cnt, 0, sizeof(Counters), st));
        bm2_smem *d_raw = P<bm2_smem>(ctx, B_SMEM_RAW); FmPrev *d_pool = P<FmPrev>(ctx, B_POOL);
        SearchTask *d_tasks = P<SearchTask>(ctx, B_TASKS); ReseedTask *d_rt = P<ReseedTask>(ctx, B_RTASKS);
        // fork: pass 3 on the side stream (it only appends to the SMEM buffer)
        BM2_CUDA_OK(cudaEventRecord(ctx->ev_fork, st));
        BM2_CUDA_OK(cudaStreamWaitEvent(ctx->side_stream, ctx->ev_fork, 0));
        {
            const int p3_ctas = env_int("BM2_SMEM_P3_CTAS", smem_ctas + 2, 1, 16);
            int blocks_p3 = (n + 127) / 128; if (blocks_p3 > ctx->n_sm * p3_ctas) blocks_p3 = ctx->n_sm * p3_ctas;
            if (q_smem) smem_pass3_kernel<true><<<blocks_p3, 128, qsm, ctx->side_stream>>>(pv.fm, pv.sp, d_codes, d_offs, n, d_raw, cap, d_cnt);
            else smem_pass3_kernel<false><<<blocks_p3, 128, 0, ctx->side_stream>>>(pv.fm, pv.sp, d_codes, d_offs, n, d_raw, cap, d_cnt);
            BM2_CUDA_OK(cudaEventRecord(ctx->ev_join, ctx->side_stream));
        }
        // pass 1: forward chains, then one backward task per search (emits SMEMs and re-seed tasks)
        if (q_smem) smem_fwd1_kernel<true><<<blocks_a, 128, qsm, st>>>(pv.fm, d_codes, d_offs, n, stripe, P<FmPrev>(ctx, B_PREV), d_pool, pool_cap, d_tasks, task_cap, d_cnt);
        else smem_fwd1_kernel<false><<<blocks_a, 128, 0, st>>>(pv.fm, d_codes, d_offs, n, stripe, P<FmPrev>(ctx, B_PREV), d_pool, pool_cap, d_tasks, task_cap, d_cnt);
        smem_bwd_kernel<<<blocks_b, 128, 0, st>>>(pv.fm, pv.sp, d_codes, d_offs, 0, d_tasks, task_cap, d_pool, pool_cap, d_raw, cap, d_rt, rtask_cap, d_cnt);
        mark_task1_kernel<<<1, 32, 0, st>>>(d_cnt);
        // pass 2: one forward search per re-seed task, then its backward task
        smem_fwd2_kernel<<<blocks_a, 128, 0, st>>>(pv.fm, d_codes, d_offs, stripe, P<FmPrev>(ctx, B_PREV), d_rt, rtask_cap, d_pool, pool_cap, d_tasks, task_cap, d_cnt);
        smem_bwd_kernel<<<blocks_b, 128, 0, st>>>(pv.fm, pv.sp, d_codes, d_offs, 1, d_tasks, task_cap, d_pool, pool_cap, d_raw, cap, d_rt, rtask_cap, d_cnt);
        BM2_CUDA_OK(cudaStreamWaitEvent(st, ctx->ev_join, 0));          // join
        BM2_CUDA_OK(cudaMemcpyAsync(&h_cnt, d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        if (h_cnt.n_smem <= cap && h_cnt.n_pool <= pool_cap && h_cnt.n_task <= task_cap && h_cnt.n_rtask <= rtask_cap) break;
        if (attempt == 2) { bm2_set_error(ctx, "SMEM stage buffers overflow"); return 1; }
        // an overflow truncates the later phases, so the counters are lower bounds: grow generously
        if (h_cnt.n_smem > cap) cap = h_cnt.n_smem * 2 + 1024;
        if (h_cnt.n_pool > pool_cap) pool_cap = h_cnt.n_pool * 2 + 65536;
        if (h_cnt.n_task > task_cap) task_cap = h_cnt.n_task * 2 + 4096;
        if (h_cnt.n_rtask > rtask_cap) rtask_cap = h_cnt.n_rtask * 2 + 4096;
    }
    tok_smem.release();
    const int64_t n_smem = (int64_t) h_cnt.n_smem;
    bs.n_smem = n_smem;
    ctx->last_n_ext = h_cnt.n_ext;

    // ---- B. order SMEMs -----------------------------------------------------------------------------------
    if (sg.mark("sort")) return 1;
    const int64_t ns1 = n_smem > 0 ? n_smem : 1;
    if (ctx->ensure(ctx->pipe_d[B_KEYS_IN], ns1 * 8) || ctx->ensure(ctx->pipe_d[B_KEYS_OUT], ns1 * 8) || ctx->ensure(ctx->pipe_d[B_VALS_IN], ns1 * 4) ||
        ctx->ensure(ctx->pipe_d[B_VALS_OUT], ns1 * 4) || ctx->ensure(ctx->pipe_d[B_SMEM], (ns1 + 1) * sizeof(bm2_smem)) ||
        ctx->ensure(ctx->pipe_d[B_SLOT_CNT], (ns1 + 1) * 8) || ctx->ensure(ctx->pipe_d[B_SLOT_OFF], (ns1 + 2) * 8) ||
        ctx->ensure(ctx->pipe_d[B_READ_SMEM_OFF], (size_t) (n + 2) * 8)) return 1;
    if (n_smem > 0) {
        const int gb = (int) ((n_smem + 255) / 256);
        smem_keys_kernel<<<gb, 256, 0, st>>>(P<bm2_smem>(ctx, B_SMEM_RAW), n_smem, P<uint64_t>(ctx, B_KEYS_IN), P<uint32_t>(ctx, B_VALS_IN));
        size_t cub_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, P<uint64_t>(ctx, B_KEYS_IN), P<uint64_t>(ctx, B_KEYS_OUT), P<uint32_t>(ctx, B_VALS_IN),
                                        P<uint32_t>(ctx, B_VALS_OUT), (int) n_smem);
        if (ctx->ensure(ctx->pipe_d[B_CUB], cub_bytes)) return 1;
        BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(ctx->pipe_d[B_CUB].p, cub_bytes, P<uint64_t>(ctx, B_KEYS_IN), P<uint64_t>(ctx, B_KEYS_OUT),
                                                    P<uint32_t>(ctx, B_VALS_IN), P<uint32_t>(ctx, B_VALS_OUT), (int) n_smem, 0, 64, st));
        BM2_CUDA_OK(cudaMemsetAsync(P<int64_t>(ctx, B_SLOT_CNT) + n_smem, 0, 8, st));
        smem_gather_kernel<<<gb, 256, 0, st>>>(P<bm2_smem>(ctx, B_SMEM_RAW), P<uint32_t>(ctx, B_VALS_OUT), n_smem, ctx->opt.max_occ,
                                               P<bm2_smem>(ctx, B_SMEM), P<int64_t>(ctx, B_SLOT_CNT));
    } else {
        BM2_CUDA_OK(cudaMemsetAsync(P<int64_t>(ctx, B_SLOT_CNT), 0, 8, st));
    }
    read_smem_off_kernel<<<(n + 1 + 255) / 256, 256, 0, st>>>(P<uint64_t>(ctx, B_KEYS_OUT), n_smem, n, P<int64_t>(ctx, B_READ_SMEM_OFF));
    if (scan64(ctx, P<int64_t>(ctx, B_SLOT_CNT), P<int64_t>(ctx, B_SLOT_OFF), n_smem)) return 1;
    if (upto == UPTO_SMEM) { if (sg.mark("end")) return 1; BM2_CUDA_OK(cudaStreamSynchronize(st)); return 0; }
    int64_t n_slots = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&n_slots, P<int64_t>(ctx, B_SLOT_OFF) + n_smem, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    bs.n_slots = n_slots;
    if (n_slots > (int64_t) 1500000000) { bm2_set_error(ctx, "too many seed occurrences in one batch: use smaller chunks"); return 1; }

    // ---- C. SA lookup -------------------------------------------------------------------------------------
    if (sg.mark("sal")) return 1;
    const size_t sl1 = (size_t) (n_slots > 0 ? n_slots : 1) + 1;
    if (ctx->ensure(ctx->pipe_d[B_SA], sl1 * 8)) return 1;
    if (n_slots > 0) {
        if (ctx->ensure(ctx->pipe_d[B_OWNER], sl1 * 4 * 2)) return 1;
        int32_t *own_in = P<int32_t>(ctx, B_OWNER), *own = own_in + sl1;
        BM2_CUDA_OK(cudaMemsetAsync(own_in, 0, sl1 * 4, st));
        slot_head_kernel<<<(unsigned) ((n_smem + 255) / 256), 256, 0, st>>>(P<int64_t>(ctx, B_SLOT_OFF), n_smem, own_in);
        size_t sbytes = 0;
        cub::DeviceScan::InclusiveScan(nullptr, sbytes, own_in, own, cub::Max(), (int) n_slots);
        if (ctx->ensure(ctx->pipe_d[B_CUB], sbytes)) return 1;
        BM2_CUDA_OK(cub::DeviceScan::InclusiveScan(ctx->pipe_d[B_CUB].p, sbytes, own_in, own, cub::Max(), (int) n_slots, st));
        sa_kernel<<<(unsigned) ((n_slots + 255) / 256), 256, 0, st>>>(pv.fm, P<bm2_smem>(ctx, B_SMEM), P<int64_t>(ctx, B_SLOT_OFF), own, n_slots,
                                                                        ctx->opt.max_occ, P<int64_t>(ctx, B_SA), d_cnt);
    }

    // ---- D. chaining --------------------------------------------------------------------------------------
    if (sg.mark("chain")) return 1;
    if (ctx->ensure(ctx->pipe_d[B_WSEED], sl1 * sizeof(WSeed)) || ctx->ensure(ctx->pipe_d[B_WCHAIN], sl1 * sizeof(WChain)) ||
        ctx->ensure(ctx->pipe_d[B_ORD], sl1 * 4) || ctx->ensure(ctx->pipe_d[B_SRT], sl1 * 4) || ctx->ensure(ctx->pipe_d[B_KV], sl1 * 4) ||
        ctx->ensure(ctx->pipe_d[B_ORDPOS], sl1 * 8) || ctx->ensure(ctx->pipe_d[B_FLT], sl1 * sizeof(FltRec)) ||
        ctx->ensure(ctx->pipe_d[B_FIN_CHAIN], sl1 * sizeof(bm2_chain)) || ctx->ensure(ctx->pipe_d[B_FIN_SEED], sl1 * sizeof(bm2_seed)) ||
        ctx->ensure(ctx->pipe_d[B_PER_READ], al((size_t) (n + 1) * 4) * 5) || ctx->ensure(ctx->pipe_d[B_SCAN], al((size_t) (n + 2) * 8) * 10)) return 1;
    const size_t pr = al((size_t) (n + 1) * 4);
    char *prb = (char *) ctx->pipe_d[B_PER_READ].p;
    int32_t *d_nchain = (int32_t *) prb, *d_nseed = (int32_t *) (prb + pr), *d_nleft = (int32_t *) (prb + 2 * pr),
            *d_nright = (int32_t *) (prb + 3 * pr), *d_nfinal = (int32_t *) (prb + 4 * pr);
    ChainBufs cb = { P<WSeed>(ctx, B_WSEED), P<WChain>(ctx, B_WCHAIN), P<int32_t>(ctx, B_ORD), P<int32_t>(ctx, B_SRT), P<int32_t>(ctx, B_KV),
                     P<int64_t>(ctx, B_ORDPOS), P<FltRec>(ctx, B_FLT),
                     P<bm2_chain>(ctx, B_FIN_CHAIN), P<bm2_seed>(ctx, B_FIN_SEED), d_nchain, d_nseed, d_nleft, d_nright };
    if (ctx->ensure(ctx->pipe_d[B_PERM], al((size_t) n * 4) * 4)) return 1;
    uint32_t *wk_in = (uint32_t *) ctx->pipe_d[B_PERM].p, *wk_out = (uint32_t *) ((char *) ctx->pipe_d[B_PERM].p + al((size_t) n * 4));
    int32_t *wv_in = (int32_t *) ((char *) ctx->pipe_d[B_PERM].p + 2 * al((size_t) n * 4)), *d_perm = (int32_t *) ((char *) ctx->pipe_d[B_PERM].p + 3 * al((size_t) n * 4));
    work_keys_slots_kernel<<<(n + 255) / 256, 256, 0, st>>>(P<int64_t>(ctx, B_READ_SMEM_OFF), P<int64_t>(ctx, B_SLOT_OFF), n, wk_in, wv_in);
    if (sort_work(ctx, wk_in, wk_out, wv_in, d_perm, n, true)) return 1;             // decreasing number of seed slots
    // light reads of the chain and tail kernels in work order instead of input order: no better in an A/B (neighbouring reads share
    // cache lines of the per-read arrays), so off unless BM2_LIGHT_SORTED=1
    const int light_sorted = env_int("BM2_LIGHT_SORTED", 0, 0, 1);
    const int chain_heavy = env_int("BM2_CHAIN_HEAVY", 64, 1, 1 << 30);          // seed occurrences from which a read gets a warp
    const int chain_coop_min = env_int("BM2_CHAIN_COOP_MIN", 1024, 0, 1 << 30);      // seed occurrences from which a warp shares the chaining of a read
    chain_kernel<<<(n + 127) / 128, 128, 0, st>>>(pv.cv, pv.cp, P<bm2_smem>(ctx, B_SMEM), P<int64_t>(ctx, B_READ_SMEM_OFF),
                                                  P<int64_t>(ctx, B_SLOT_OFF), P<int64_t>(ctx, B_SA), d_offs, n, d_perm, cb, pv.sw, ctx->idx.ref, d_codes,
                                                  any_flt ? P<int32_t>(ctx, B_MINHSP) : nullptr, 0, chain_heavy, chain_coop_min, light_sorted);
    {   // heavy reads: one warp each; the sorted list ends the grid early (warps whose read is light return at once)
        int heavy_warps = n < ctx->n_sm * 256 ? n : ctx->n_sm * 256;
        chain_kernel<<<(heavy_warps * 32 + 127) / 128, 128, 0, st>>>(pv.cv, pv.cp, P<bm2_smem>(ctx, B_SMEM), P<int64_t>(ctx, B_READ_SMEM_OFF),
                                                                      P<int64_t>(ctx, B_SLOT_OFF), P<int64_t>(ctx, B_SA), d_offs, n, d_perm, cb, pv.sw,
                                                                      ctx->idx.ref, d_codes, any_flt ? P<int32_t>(ctx, B_MINHSP) : nullptr, 1, chain_heavy, chain_coop_min, 0);
    }

    // ---- E. scans + compaction ------------------------------------------------------------------------------
    if (sg.mark("compact")) return 1;
    const size_t sc = al((size_t) (n + 2) * 8);
    char *scb = (char *) ctx->pipe_d[B_SCAN].p;
    int64_t *w_tmp = (int64_t *) scb, *d_chain_off = (int64_t *) (scb + sc), *d_reg_off = (int64_t *) (scb + 2 * sc),
            *d_left_off = (int64_t *) (scb + 3 * sc), *d_right_off = (int64_t *) (scb + 4 * sc), *d_out_off = (int64_t *) (scb + 5 * sc);
    const int gw = (n + 1 + 255) / 256;
    widen_kernel<<<gw, 256, 0, st>>>(d_nchain, n, w_tmp); if (scan64(ctx, w_tmp, d_chain_off, n)) return 1;
    widen_kernel<<<gw, 256, 0, st>>>(d_nseed, n, w_tmp);  if (scan64(ctx, w_tmp, d_reg_off, n)) return 1;
    widen_kernel<<<gw, 256, 0, st>>>(d_nleft, n, w_tmp);  if (scan64(ctx, w_tmp, d_left_off, n)) return 1;
    widen_kernel<<<gw, 256, 0, st>>>(d_nright, n, w_tmp); if (scan64(ctx, w_tmp, d_right_off, n)) return 1;
    int64_t tot[4];
    BM2_CUDA_OK(cudaMemcpyAsync(&tot[0], d_chain_off + n, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&tot[1], d_reg_off + n, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&tot[2], d_left_off + n, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&tot[3], d_right_off + n, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&h_cnt, d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    ctx->last_n_lf = h_cnt.n_lf;
    const int64_t n_chains = tot[0], n_regs = tot[1], n_left = tot[2], n_right = tot[3];
    bs.n_chains = n_chains; bs.n_regs = n_regs; bs.n_left = n_left; bs.n_right = n_right;
    if (n_regs > 2000000000LL) { bm2_set_error(ctx, "too many seeds in one batch"); return 1; }
    if (ctx->ensure(ctx->pipe_d[B_CHAINS], (size_t) (n_chains + 1) * sizeof(bm2_chain)) || ctx->ensure(ctx->pipe_d[B_SEEDS], (size_t) (n_regs + 1) * sizeof(bm2_seed))) return 1;
    chain_compact_kernel<<<(n + 127) / 128, 128, 0, st>>>(P<int64_t>(ctx, B_READ_SMEM_OFF), P<int64_t>(ctx, B_SLOT_OFF), n, P<bm2_chain>(ctx, B_FIN_CHAIN),
                                                          P<bm2_seed>(ctx, B_FIN_SEED), d_chain_off, d_reg_off, P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS));
    if (upto == UPTO_CHAIN) { if (sg.mark("end")) return 1; BM2_CUDA_OK(cudaStreamSynchronize(st)); return 0; }

    // ---- F. regs + jobs -----------------------------------------------------------------------------------
    if (sg.mark("extbuild")) return 1;
    const size_t nr1 = (size_t) n_regs + 1, nl1 = (size_t) n_left + 1, nrt1 = (size_t) n_right + 1;
    // Lazy extension (BM2_EXT_LAZY, default on): the jobs run in BM2_EXT_WAVES waves (default 2).  Wave 1 extends the first seed of every
    // chain; a post-filter walk (ext_walk_kernel) then decides the seeds after it, up to the first kept seed not extended yet; further
    // speculative waves extend the seeds the walks stopped at; the last wave extends every reg that is neither extended nor proved purged.
    // The seeds proved purged are never extended.  BM2_EXT_LAZY=0: every job in one wave.
    const int lazy = env_int("BM2_EXT_LAZY", 1, 0, 1);
    const int waves = env_int("BM2_EXT_WAVES", 2, 2, 64);
    const size_t aux_bytes = al(nr1 * 4) * 3 + al(nr1 * 8) + al(nl1 * 4) * 2 + al(nrt1 * 4) * 2 + al(nr1 * sizeof(PfBox)) +
                             (lazy ? al(nr1) + al((size_t) n * sizeof(PfCursor)) + al(nl1 * 4) + al(nrt1 * 4) : 0);
    const size_t njmax = nl1 > nrt1 ? nl1 : nrt1;
    if (ctx->ensure(ctx->pipe_d[B_REGS], nr1 * sizeof(bm2_alnreg_t)) || ctx->ensure(ctx->pipe_d[B_REG_AUX], aux_bytes) ||
        ctx->ensure(ctx->pipe_d[B_JOBS], al(nl1 * sizeof(ExtJobRec)) + al(nrt1 * sizeof(ExtJobRec)) + al(njmax * sizeof(ExtJobRec)) + al(njmax * sizeof(BswOut)) +
                                    (lazy ? al(nl1 * sizeof(ExtJobRec)) + al(nrt1 * sizeof(ExtJobRec)) : 0)) ||
        ctx->ensure(ctx->bsw_scratch, bsw_scratch_bytes((int) njmax))) return 1;
    char *ab = (char *) ctx->pipe_d[B_REG_AUX].p;
    int32_t *d_reg_chain = (int32_t *) ab; ab += al(nr1 * 4);
    int32_t *d_reg_seed = (int32_t *) ab; ab += al(nr1 * 4);
    int32_t *d_srt2 = (int32_t *) ab; ab += al(nr1 * 4);
    uint64_t *d_srt = (uint64_t *) ab; ab += al(nr1 * 8);
    int32_t *d_left_reg = (int32_t *) ab; ab += al(nl1 * 4);
    int32_t *d_left_retry = (int32_t *) ab; ab += al(nl1 * 4);
    int32_t *d_right_reg = (int32_t *) ab; ab += al(nrt1 * 4);
    int32_t *d_right_retry = (int32_t *) ab; ab += al(nrt1 * 4);
    PfBox *d_box = (PfBox *) ab; ab += al(nr1 * sizeof(PfBox));
    uint8_t *d_state = nullptr; PfCursor *d_cursor = nullptr; int32_t *d_wleft_reg = nullptr, *d_wright_reg = nullptr;
    if (lazy) {
        d_state = (uint8_t *) ab; ab += al(nr1);
        d_cursor = (PfCursor *) ab; ab += al((size_t) n * sizeof(PfCursor));
        d_wleft_reg = (int32_t *) ab; ab += al(nl1 * 4);
        d_wright_reg = (int32_t *) ab; ab += al(nrt1 * 4);
    }
    char *jb = (char *) ctx->pipe_d[B_JOBS].p;
    ExtJobRec *d_left = (ExtJobRec *) jb; jb += al(nl1 * sizeof(ExtJobRec));
    ExtJobRec *d_right = (ExtJobRec *) jb; jb += al(nrt1 * sizeof(ExtJobRec));
    ExtJobRec *d_retry_jobs = (ExtJobRec *) jb; jb += al(njmax * sizeof(ExtJobRec));
    BswOut *d_outs = (BswOut *) jb; jb += al(njmax * sizeof(BswOut));
    ExtJobRec *d_wleft = nullptr, *d_wright = nullptr;          // the jobs of one wave
    if (lazy) { d_wleft = (ExtJobRec *) jb; jb += al(nl1 * sizeof(ExtJobRec)); d_wright = (ExtJobRec *) jb; }
    bm2_alnreg_t *d_regs = P<bm2_alnreg_t>(ctx, B_REGS);
    ExtBufs eb = { d_regs, d_reg_chain, d_reg_seed, d_srt, d_left, d_right, d_left_reg, d_right_reg, d_state };
    work_keys_off_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_reg_off, n, wk_in, wv_in);       // work ~ regs of the read
    if (sort_work(ctx, wk_in, wk_out, wv_in, d_perm, n)) return 1;
    ext_build_kernel<<<(n + 127) / 128, 128, 0, st>>>(pv.cv, pv.ep, P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS), d_chain_off, d_reg_off,
                                                      d_left_off, d_right_off, d_offs, n, d_perm, eb);
    // from here on d_perm orders the reads by decreasing regs: the walk's and the tail's warp-per-read passes take the heavy reads from it
    work_keys_off_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_reg_off, n, wk_in, wv_in);
    if (sort_work(ctx, wk_in, wk_out, wv_in, d_perm, n, true)) return 1;
    const int heavy_thr = env_int("BM2_TAIL_HEAVY", 24, 1, 1 << 20);            // regs from which a read's post-filter scan gets a warp
    int blocks_i = (n + 127) / 128; const int max_blocks_i = ctx->n_sm * 8; if (blocks_i > max_blocks_i) blocks_i = max_blocks_i;

    // ---- G/H. extension -----------------------------------------------------------------------------------
    auto phase = [&](const char *name, ExtJobRec *jobs, int32_t *job_reg, int32_t *retry, int64_t nj, int is_right) -> int {
        if (sg.mark(name)) return 1;
        if (nj <= 0) return 0;
        StageToken tok_bsw((use_tokens & 2) ? &ctx->parent->tok_bsw : nullptr);
        BswParams bp; bp.a = ctx->opt.a; bp.b = ctx->opt.b; bp.o_del = ctx->opt.o_del; bp.e_del = ctx->opt.e_del; bp.o_ins = ctx->opt.o_ins;
        bp.e_ins = ctx->opt.e_ins; bp.zdrop = ctx->opt.zdrop; bp.end_bonus = is_right ? ctx->opt.pen_clip3 : ctx->opt.pen_clip5; bp.w = ctx->opt.w;
        if (is_right) right_h0_kernel<<<(unsigned) ((nj + 255) / 256), 256, 0, st>>>(jobs, job_reg, (int) nj, d_regs);
        BM2_CUDA_OK(cudaMemsetAsync(&d_cnt->n_retry, 0, 8, st));
        if (bsw_launch_with_scratch(ctx, st, (const BswJob *) jobs, d_outs, (int) nj, ctx->idx.ref, d_codes, bp, &d_cnt->cells, ctx->bsw_scratch.p,
                                    ctx->bsw_scratch.cap, 1)) return 1;
        fold_kernel<<<(unsigned) ((nj + 255) / 256), 256, 0, st>>>(pv.ep, jobs, job_reg, d_outs, nullptr, (int) nj, is_right, bp.w, 0, d_regs, d_reg_chain,
                                                                   P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS), d_offs, retry, d_cnt);
        unsigned long long n_retry = 0;
        BM2_CUDA_OK(cudaMemcpyAsync(&n_retry, &d_cnt->n_retry, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        if (n_retry > 0) {   // MAX_BAND_TRY = 2: re-run the rejected jobs once with the doubled band (src/bwamem.cpp:2472)
            gather_jobs_kernel<<<(unsigned) ((n_retry + 255) / 256), 256, 0, st>>>(jobs, retry, (int) n_retry, d_retry_jobs);
            bp.w = ctx->opt.w << 1;
            if (bsw_launch_with_scratch(ctx, st, (const BswJob *) d_retry_jobs, d_outs, (int) n_retry, ctx->idx.ref, d_codes, bp, &d_cnt->cells,
                                        ctx->bsw_scratch.p, ctx->bsw_scratch.cap, 1)) return 1;
            // `retry` is read as the selection list while the kernel appends nothing new (last_try = 1)
            fold_kernel<<<(unsigned) ((n_retry + 255) / 256), 256, 0, st>>>(pv.ep, jobs, job_reg, d_outs, retry, (int) n_retry, is_right, bp.w, 1, d_regs,
                                                                            d_reg_chain, P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS), d_offs,
                                                                            retry, d_cnt);
        }
        ctx->last_n_retry[is_right] += n_retry;
        return 0;
    };
    ctx->last_n_retry[0] = ctx->last_n_retry[1] = 0;
    ctx->last_jobs_skipped = 0;
    if (!lazy) {
        if (phase("bsw_left", d_left, d_left_reg, d_left_retry, n_left, 0)) return 1;
        if (phase("bsw_right", d_right, d_right_reg, d_right_retry, n_right, 1)) return 1;
    } else {
        int64_t jobs_run = 0;
        for (int wave = 1; wave <= waves; ++wave) {
            const int last = wave == waves;
            if (sg.mark("ext_select")) return 1;
            BM2_CUDA_OK(cudaMemsetAsync(d_cnt->n_sel, 0, sizeof(d_cnt->n_sel), st));
            if (n_left > 0)
                ext_select_kernel<<<(unsigned) ((n_left + 255) / 256), 256, 0, st>>>(d_left, d_left_reg, (int) n_left, d_state, last, d_wleft,
                                                                                     d_wleft_reg, &d_cnt->n_sel[0]);
            if (n_right > 0)
                ext_select_kernel<<<(unsigned) ((n_right + 255) / 256), 256, 0, st>>>(d_right, d_right_reg, (int) n_right, d_state, last, d_wright,
                                                                                      d_wright_reg, &d_cnt->n_sel[1]);
            unsigned long long n_sel[2] = {0, 0};
            BM2_CUDA_OK(cudaMemcpyAsync(n_sel, d_cnt->n_sel, sizeof(n_sel), cudaMemcpyDeviceToHost, st));
            BM2_CUDA_OK(cudaStreamSynchronize(st));
            if (phase("bsw_left", d_wleft, d_wleft_reg, d_left_retry, (int64_t) n_sel[0], 0)) return 1;
            if (phase("bsw_right", d_wright, d_wright_reg, d_right_retry, (int64_t) n_sel[1], 1)) return 1;
            jobs_run += (int64_t) (n_sel[0] + n_sel[1]);
            if (last) break;
            if (sg.mark("ext_walk")) return 1;
            ext_mark_done_kernel<<<(unsigned) ((n_regs + 255) / 256), 256, 0, st>>>(d_state, n_regs);
            ext_walk_kernel<0><<<(n + 127) / 128, 128, 0, st>>>(pv.ep, P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS), d_chain_off, d_reg_off, d_offs,
                                                                n, d_regs, d_reg_seed, d_state, d_srt2, d_box, d_cursor, d_perm, heavy_thr, wave == 1, d_cnt);
            ext_walk_kernel<1><<<blocks_i, 128, 0, st>>>(pv.ep, P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS), d_chain_off, d_reg_off, d_offs,
                                                         n, d_regs, d_reg_seed, d_state, d_srt2, d_box, d_cursor, d_perm, heavy_thr, wave == 1, d_cnt);
        }
        ctx->last_jobs_skipped = (unsigned long long) (n_left + n_right - jobs_run);
    }

    // ---- I. post-filter + tail ----------------------------------------------------------------------------
    if (sg.mark("tail")) return 1;
    const int he_stride = 2 * (max_len + 2);
    if (ctx->ensure(ctx->pipe_d[B_NW], (size_t) blocks_i * 128 * he_stride * 4)) return 1;
    if (getenv("BM2_DEBUG_NREG")) {     // the heaviest reads of the batch (their tail is the critical path of the warp-per-read kernel): stderr
        std::vector<int64_t> ho((size_t) n + 1);
        BM2_CUDA_OK(cudaMemcpyAsync(ho.data(), d_reg_off, (size_t) (n + 1) * 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        std::vector<int64_t> cntv((size_t) n);
        for (int i = 0; i < n; ++i) cntv[i] = ho[i + 1] - ho[i];
        std::sort(cntv.begin(), cntv.end(), [](int64_t a, int64_t b) { return a > b; });
        long long c24 = 0, c256 = 0, c1024 = 0; double sq = 0;
        for (int i = 0; i < n; ++i) { c24 += cntv[i] > 24; c256 += cntv[i] > 256; c1024 += cntv[i] > 1024; if (cntv[i] > 24) sq += (double) cntv[i] * (double) cntv[i]; }
        fprintf(stderr, "[bm2 debug] regs before the tail: reads %d, > 24: %lld, > 256: %lld, > 1024: %lld, sum of squares over the heavy reads %.3g; heaviest:", n, c24, c256, c1024, sq);
        for (int i = 0; i < 8 && i < n; ++i) fprintf(stderr, " %lld", (long long) cntv[i]);
        fprintf(stderr, "\n");
    }
    tail_kernel<0><<<blocks_i, 128, 0, st>>>(pv.cv, pv.ep, ctx->idx.ref, d_codes, d_offs, P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS), d_chain_off,
                                             d_reg_off, n, d_regs, d_reg_seed, d_srt2, P<int32_t>(ctx, B_NW), he_stride, d_perm, d_box, d_nfinal, heavy_thr, light_sorted, 0);
    tail_kernel<1><<<blocks_i, 128, 0, st>>>(pv.cv, pv.ep, ctx->idx.ref, d_codes, d_offs, P<bm2_chain>(ctx, B_CHAINS), P<bm2_seed>(ctx, B_SEEDS), d_chain_off,
                                             d_reg_off, n, d_regs, d_reg_seed, d_srt2, P<int32_t>(ctx, B_NW), he_stride, d_perm, d_box, d_nfinal, heavy_thr, 0, env_int("BM2_TAIL_COOP", 1, 0, 1));

    // ---- J. output ---------------------------------------------------------------------------------------
    if (sg.mark("output")) return 1;
    widen_kernel<<<gw, 256, 0, st>>>(d_nfinal, n, w_tmp); if (scan64(ctx, w_tmp, d_out_off, n)) return 1;
    if (ctx->ensure(ctx->pipe_d[B_OUT], nr1 * sizeof(bm2_alnreg_t))) return 1;
    regs_gather_kernel<<<(n + 127) / 128, 128, 0, st>>>(d_regs, d_reg_off, d_out_off, n, P<bm2_alnreg_t>(ctx, B_OUT));
    if (ctx->ensure_host(ctx->pipe_h[H_OUT_OFF], (size_t) (n + 1) * 8)) return 1;
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->pipe_h[H_OUT_OFF].p, d_out_off, (size_t) (n + 1) * 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&h_cnt, d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    ctx->last_cells = h_cnt.cells;
    ctx->last_walk_done = h_cnt.n_walk_done;
    const int64_t n_out = ((const int64_t *) ctx->pipe_h[H_OUT_OFF].p)[n];
    bs.n_out = n_out;
    if (copy_out && ctx->ensure_host(ctx->pipe_h[H_OUT_REGS], (size_t) (n_out + 1) * sizeof(bm2_alnreg_t))) return 1;
    if (n_out && copy_out) BM2_CUDA_OK(cudaMemcpyAsync(ctx->pipe_h[H_OUT_REGS].p, ctx->pipe_d[B_OUT].p, (size_t) n_out * sizeof(bm2_alnreg_t), cudaMemcpyDeviceToHost, st));
    if (sg.mark("end")) return 1;
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaGetLastError());
    return 0;
}

int finish_stage_times(bm2_ctx *ctx) {
    bm2_ctx *ctx_for_error = ctx;
    ctx->stage_ms.clear();
    size_t n = ctx->stage_names.size();
    // the names vector may be longer than this run's marks when an earlier run went further
    size_t marks = 0;
    for (; marks < n; ++marks) if (strcmp(ctx->stage_names[marks], "end") == 0) { ++marks; break; }
    // a stage marked more than once (the extension stages, once per wave of the lazy extension) is reported once, its times summed
    std::vector<const char *> names;
    for (size_t i = 0; i < marks; ++i) {
        float ms = 0;
        if (i + 1 < marks) BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->events[i], ctx->events[i + 1]));
        size_t j = 0;
        while (j < names.size() && strcmp(names[j], ctx->stage_names[i]) != 0) ++j;
        if (j == names.size()) { names.push_back(ctx->stage_names[i]); ctx->stage_ms.push_back(0.f); }
        ctx->stage_ms[j] += ms;
    }
    ctx->stage_names = names;
    return 0;
}

}  // namespace

// ---- seam 2 entry points -----------------------------------------------------------------------------------
extern "C" int bm2_collect_smems(bm2_ctx *ctx, const bm2_read_batch *reads, bm2_smem_result *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !reads || !out) return 1;
    BatchState bs;
    if (run_pipeline(ctx, reads, UPTO_SMEM, bs)) return 1;
    finish_stage_times(ctx);
    if (ctx->ensure_host(ctx->pipe_h[H_SMEM], (size_t) (bs.n_smem + 1) * sizeof(bm2_smem)) || ctx->ensure_host(ctx->pipe_h[H_OUT_OFF], (size_t) (bs.n + 2) * 8)) return 1;
    if (bs.n_smem) BM2_CUDA_OK(cudaMemcpy(ctx->pipe_h[H_SMEM].p, ctx->pipe_d[B_SMEM].p, (size_t) bs.n_smem * sizeof(bm2_smem), cudaMemcpyDeviceToHost));
    if (bs.n > 0) BM2_CUDA_OK(cudaMemcpy(ctx->pipe_h[H_OUT_OFF].p, ctx->pipe_d[B_READ_SMEM_OFF].p, (size_t) (bs.n + 1) * 8, cudaMemcpyDeviceToHost));
    else ((int64_t *) ctx->pipe_h[H_OUT_OFF].p)[0] = 0;
    out->n = bs.n_smem; out->smems = (const bm2_smem *) ctx->pipe_h[H_SMEM].p; out->read_off = (const int64_t *) ctx->pipe_h[H_OUT_OFF].p;
    return 0;
}

extern "C" int bm2_seed_chain(bm2_ctx *ctx, const bm2_read_batch *reads, bm2_chain_result *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !reads || !out) return 1;
    BatchState bs;
    if (run_pipeline(ctx, reads, UPTO_CHAIN, bs)) return 1;
    finish_stage_times(ctx);
    if (ctx->ensure_host(ctx->pipe_h[H_CHAINS], (size_t) (bs.n_chains + 1) * sizeof(bm2_chain)) ||
        ctx->ensure_host(ctx->pipe_h[H_SEEDS], (size_t) (bs.n_regs + 1) * sizeof(bm2_seed)) || ctx->ensure_host(ctx->pipe_h[H_OUT_OFF], (size_t) (bs.n + 2) * 8)) return 1;
    if (bs.n_chains) BM2_CUDA_OK(cudaMemcpy(ctx->pipe_h[H_CHAINS].p, ctx->pipe_d[B_CHAINS].p, (size_t) bs.n_chains * sizeof(bm2_chain), cudaMemcpyDeviceToHost));
    if (bs.n_regs) BM2_CUDA_OK(cudaMemcpy(ctx->pipe_h[H_SEEDS].p, ctx->pipe_d[B_SEEDS].p, (size_t) bs.n_regs * sizeof(bm2_seed), cudaMemcpyDeviceToHost));
    if (bs.n > 0) {
        const size_t sc = al((size_t) (bs.n + 2) * 8);
        BM2_CUDA_OK(cudaMemcpy(ctx->pipe_h[H_OUT_OFF].p, (char *) ctx->pipe_d[B_SCAN].p + sc, (size_t) (bs.n + 1) * 8, cudaMemcpyDeviceToHost));
    } else ((int64_t *) ctx->pipe_h[H_OUT_OFF].p)[0] = 0;
    out->n_chains = bs.n_chains; out->n_seeds = bs.n_regs; out->chains = (const bm2_chain *) ctx->pipe_h[H_CHAINS].p;
    out->seeds = (const bm2_seed *) ctx->pipe_h[H_SEEDS].p; out->read_off = (const int64_t *) ctx->pipe_h[H_OUT_OFF].p;
    return 0;
}

bm2_ctx *bm2_make_lane(bm2_ctx *parent);   // capi.cu

// mem_kernel1_core + mem_kernel2_core of one batch, as up to n_lanes sub-batches in flight (bm2_set_sub_batches).
// d_codes / d_offs: device-resident inputs (may be null: host inputs are uploaded); results into the context's pinned buffers.
static int run_regs(bm2_ctx *ctx, const bm2_read_batch *rb, const uint8_t *d_codes, const int64_t *d_offs, bool copy_out, bm2_reg_result *out)
{
    bm2_ctx *ctx_for_error = ctx;
    const int n = rb->n_reads;
    int K = ctx->n_lanes;
    if (K > 1 && (int64_t) n < (int64_t) K * ctx->lane_min_reads) K = n / ctx->lane_min_reads;
    if (K <= 1) {
        BatchState bs;
        if (run_pipeline(ctx, rb, UPTO_REGS, bs, d_codes, d_offs, copy_out)) return 1;
        finish_stage_times(ctx);
        if (bs.n <= 0) {
            if (ctx->ensure_host(ctx->pipe_h[H_OUT_OFF], 16) || ctx->ensure_host(ctx->pipe_h[H_OUT_REGS], sizeof(bm2_alnreg_t))) return 1;
            ((int64_t *) ctx->pipe_h[H_OUT_OFF].p)[0] = 0;
        }
        out->n = bs.n_out; out->regs = copy_out ? (const bm2_alnreg_t *) ctx->pipe_h[H_OUT_REGS].p : nullptr; out->read_off = (const int64_t *) ctx->pipe_h[H_OUT_OFF].p;
        return 0;
    }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    while ((int) ctx->lanes.size() < K) {
        bm2_ctx *l = bm2_make_lane(ctx);
        if (!l) return 1;
        ctx->lanes.push_back(l);
    }
    if (!ctx->ev_entry) BM2_CUDA_OK(cudaEventCreateWithFlags(&ctx->ev_entry, cudaEventDisableTiming));
    // the sub-batches start after whatever the caller queued on the context's stream (its inputs, its start event)
    BM2_CUDA_OK(cudaEventRecord(ctx->ev_entry, ctx->stream));
    struct Job { int first = 0, n = 0; std::vector<int64_t> offs; bm2_read_batch rb; BatchState bs; int rc = 0; };
    // (Round 2 also ran every lane over several smaller sub-batches in a row, each sub-batch's regs copied to the host on a copy stream under
    // the kernels of the following ones - the device -> host copies at the end of the step, 387 MB per 1 M reads, are the gap between the
    // resident and the end-to-end number.  Bit-identical and slower end to end in an A/B (2 x 4 and 3 x 4 sub-batches against 4): eight
    // 125 k-read sub-batches lose more in the kernels than the hidden copies give back.)
    std::vector<Job> jobs((size_t) K);
    // cut points (multiples of 512 reads).  BM2_LANE_SKEW = s percent: lane k gets a share proportional to 100 + s * k instead of equal shares,
    // so that the lanes - which start together - leave the SMEM stage at different times (experiment: do unequal lanes overlap unlike stages better?)
    std::vector<int> cut((size_t) K + 1, 0);
    {
        const int skew = env_int("BM2_LANE_SKEW", 0, 0, 400);
        double tot = 0; for (int k = 0; k < K; ++k) tot += 100.0 + (double) skew * k;
        double acc = 0;
        for (int k = 0; k < K; ++k) { cut[k] = (int) ((int64_t) ((double) n * acc / tot) / 512 * 512); acc += 100.0 + (double) skew * k; }
        cut[K] = n;
    }
    for (int k = 0; k < K; ++k) {
        Job &j = jobs[k];
        j.first = cut[k];
        const int next = cut[k + 1];
        j.n = next - j.first;
        bm2_ctx *l = ctx->lanes[k];
        l->opt = ctx->opt;
        BM2_CUDA_OK(cudaStreamWaitEvent(l->stream, ctx->ev_entry, 0));
    }
    auto work = [&](int k) {
        Job &j = jobs[k];
        bm2_ctx *l = ctx->lanes[k];
        const int64_t base = rb->offsets[j.first];
        j.offs.resize((size_t) j.n + 1);
        for (int i = 0; i <= j.n; ++i) j.offs[i] = rb->offsets[j.first + i] - base;
        j.rb.n_reads = j.n; j.rb.codes = rb->codes ? rb->codes + base : nullptr; j.rb.offsets = j.offs.data();
        // (the device offsets of a resident batch mirror the host offsets: the sub-batch's codes start at `base`)
        j.rc = run_pipeline(l, &j.rb, UPTO_REGS, j.bs, d_codes ? d_codes + base : nullptr, nullptr, false);
        if (!j.rc) finish_stage_times(l);
    };
    if (getenv("BM2_SUB_BATCHES_SERIAL")) {        // debugging aid: the same split, one sub-batch after the other
        for (int k = 0; k < K; ++k) work(k);
    } else {
        std::vector<std::thread> th;
        for (int k = 1; k < K; ++k) th.emplace_back(work, k);
        work(0);
        for (auto &t : th) t.join();
    }
    for (int k = 0; k < K; ++k)
        if (jobs[k].rc) { bm2_set_error(ctx, "sub-batch " + std::to_string(k) + ": " + ctx->lanes[k]->err); return 1; }
    // gather: per-read offsets on the host, regs device -> the context's pinned buffer, one copy per lane on its own stream
    int64_t n_out = 0;
    for (int k = 0; k < K; ++k) n_out += jobs[k].bs.n_out;
    if (ctx->ensure_host(ctx->pipe_h[H_OUT_OFF], (size_t) (n + 1) * 8) || ctx->ensure_host(ctx->pipe_h[H_OUT_REGS], (size_t) (n_out + 1) * sizeof(bm2_alnreg_t))) return 1;
    int64_t *off = (int64_t *) ctx->pipe_h[H_OUT_OFF].p;
    bm2_alnreg_t *regs = (bm2_alnreg_t *) ctx->pipe_h[H_OUT_REGS].p;
    int64_t pos = 0;
    for (int k = 0; k < K; ++k) {
        const Job &j = jobs[k];
        bm2_ctx *l = ctx->lanes[k];
        const int64_t *lo = (const int64_t *) l->pipe_h[H_OUT_OFF].p;
        if (copy_out && j.bs.n_out)
            BM2_CUDA_OK(cudaMemcpyAsync(regs + pos, l->pipe_d[B_OUT].p, (size_t) j.bs.n_out * sizeof(bm2_alnreg_t), cudaMemcpyDeviceToHost, l->stream));
        for (int i = 0; i < j.n; ++i) off[j.first + i] = lo[i] + pos;
        pos += j.bs.n_out;
    }
    off[n] = n_out;
    for (int k = 0; k < K; ++k) BM2_CUDA_OK(cudaStreamSynchronize(ctx->lanes[k]->stream));
    // bookkeeping: stage times are summed over the sub-batches (GPU time per stage; the stages of different
    // sub-batches overlap, so they no longer add up to the wall time), counters are totals
    ctx->stage_names = ctx->lanes[0]->stage_names;
    ctx->stage_ms.assign(ctx->lanes[0]->stage_ms.size(), 0.f);
    ctx->last_n_ext = ctx->last_n_lf = ctx->last_cells = 0; ctx->last_n_retry[0] = ctx->last_n_retry[1] = 0;
    ctx->last_jobs_skipped = ctx->last_walk_done = 0;
    for (int k = 0; k < K; ++k) {
        const bm2_ctx *l = ctx->lanes[k];
        for (size_t i = 0; i < ctx->stage_ms.size() && i < l->stage_ms.size(); ++i) ctx->stage_ms[i] += l->stage_ms[i];
        ctx->last_n_ext += l->last_n_ext; ctx->last_n_lf += l->last_n_lf; ctx->last_cells += l->last_cells;
        ctx->last_n_retry[0] += l->last_n_retry[0]; ctx->last_n_retry[1] += l->last_n_retry[1];
        ctx->last_jobs_skipped += l->last_jobs_skipped; ctx->last_walk_done += l->last_walk_done;
    }
    out->n = n_out; out->regs = copy_out ? regs : nullptr; out->read_off = off;
    return 0;
}

extern "C" int bm2_seed_chain_extend(bm2_ctx *ctx, const bm2_read_batch *reads, bm2_reg_result *out) {
    if (!ctx || !reads || !out) return 1;
    return run_regs(ctx, reads, nullptr, nullptr, true, out);
}

extern "C" int bm2_seed_chain_extend_resident(bm2_ctx *ctx, const bm2_read_batch *reads, const uint8_t *d_codes, const int64_t *d_offsets,
                                              int copy_out, bm2_reg_result *out) {
    if (!ctx || !reads || !out || !d_codes || !d_offsets) return 1;
    return run_regs(ctx, reads, d_codes, d_offsets, copy_out != 0, out);
}

extern "C" int bm2_last_stage_ms(const bm2_ctx *ctx, const char *const **names, const float **ms, int *n) {
    if (!ctx) return 1;
    *names = ctx->stage_names.data(); *ms = ctx->stage_ms.data();
    *n = (int) (ctx->stage_ms.size() < ctx->stage_names.size() ? ctx->stage_ms.size() : ctx->stage_names.size());
    return 0;
}

extern "C" int bm2_last_counters(const bm2_ctx *ctx, unsigned long long *v, int n) {
    if (!ctx || n < 5) return 1;
    v[0] = ctx->last_n_ext; v[1] = ctx->last_n_lf; v[2] = ctx->last_cells; v[3] = ctx->last_n_retry[0]; v[4] = ctx->last_n_retry[1];
    if (n >= 7) { v[5] = ctx->last_jobs_skipped; v[6] = ctx->last_walk_done; }
    return 0;
}

// markdup.cu — duplicate marking on the GPU (bm2_mem --markdup); the per-template and per-group logic is markdup_device.cuh's.
//   bm2_dup_signatures   one warp per template: its primaries found by a ballot over its records, then per primary the CIGAR's reference
//                        length (inline or CG:B,I) and the qualities >= 15 summed across the warp; lane 0 writes the template's entries into
//                        fixed slots (one pair slot, two fragment-space slots), which cub::DeviceSelect compacts in template order
//   bm2_dup_resolve      entries sorted by (k1, k2, score descending, tid): an ordinal array through one stable cub::DeviceRadixSort pass per
//                        field, least significant first, each over the bits that field uses (their OR, from one reduction kernel); then
//                        (resolve) group heads, an inclusive scan into group numbers, per group whether it holds a pair-end entry and its first
//                        other entry (atomics), and cub::DeviceSelect::Flagged of the duplicates' template ids
//   bm2_dup_set          the duplicate bitset, kept on the context for bm2_bam_sort_compress_ex (bam_sort.cu)
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "markdup_device.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <vector>

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;

template <class T> __device__ __forceinline__ T warp_sum(T v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

__global__ void dup_sig_kernel(const uint8_t *__restrict__ in, const int64_t *__restrict__ starts, const int64_t *__restrict__ tfirst,
                               const int64_t *__restrict__ tids, int64_t n_tmpl, bm2_dup_entry *pair, bm2_dup_entry *frag) {
    const int64_t t = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (t >= n_tmpl) return;
    const int64_t r0 = tfirst[t], r1 = tfirst[t + 1];
    int n_prim = 0;
    int64_t prim[2] = { 0, 0 };
    for (int64_t b = r0; b < r1 && n_prim <= 2; b += 32) {
        const int64_t i = b + lane;
        unsigned m = __ballot_sync(kFull, i < r1 && dup_is_primary((int32_t) bam_le16(in + starts[i] + 18)));
        for (; m && n_prim <= 2; m &= m - 1, ++n_prim) if (n_prim < 2) prim[n_prim] = b + __ffs(m) - 1;
    }
    int mapped[2] = { 0, 0 };
    uint64_t end[2] = { 0, 0 };
    int32_t score[2] = { 0, 0 };
    for (int k = 0; k < n_prim && k < 2; ++k) {
        const uint8_t *r = in + starts[prim[k]];
        mapped[k] = !(bam_le16(r + 18) & 4);
        score[k] = dup_read_score(warp_sum(dup_qual_part(r, lane, 32)));
        if (mapped[k]) {
            const DupCigar c = dup_cigar(r);
            end[k] = dup_read_end(r, c, warp_sum(dup_ref_len_part(c, lane, 32)));
        }
    }
    if (lane) return;
    bm2_dup_entry pe, fe[2];
    int has_pair = 0, n_frag = 0;
    dup_template_entries(n_prim, mapped, end, score, tids[t], &pe, &has_pair, fe, &n_frag);
    pe.kind = has_pair ? pe.kind : -1;
    pair[t] = pe;
    for (int k = 0; k < 2; ++k) { if (k >= n_frag) fe[k].kind = -1; frag[2 * t + k] = fe[k]; }
}

struct IsEntry { __device__ __forceinline__ bool operator()(const bm2_dup_entry &e) const { return e.kind >= 0; } };

__global__ void dup_or_kernel(const bm2_dup_entry *__restrict__ e, int64_t n, unsigned long long *ors) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long a = 0, b = 0, c = 0;
    if (i < n) { a = e[i].k1; b = e[i].k2; c = (unsigned long long) e[i].tid; }
    for (int o = 16; o; o >>= 1) { a |= __shfl_xor_sync(kFull, a, o); b |= __shfl_xor_sync(kFull, b, o); c |= __shfl_xor_sync(kFull, c, o); }
    if ((threadIdx.x & 31) == 0) { atomicOr(ors, a); atomicOr(ors + 1, b); atomicOr(ors + 2, c); }
}

__global__ void dup_iota_kernel(uint32_t *ord, int64_t n) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ord[i] = (uint32_t) i;
}

// field 0: tid, 1: descending score, 2: k2, 3: k1 - of the entry at each place of the current order
__global__ void dup_field_kernel(const bm2_dup_entry *__restrict__ e, const uint32_t *__restrict__ ord, int64_t n, int field, uint64_t *keys) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bm2_dup_entry &x = e[ord[i]];
    keys[i] = field == 0 ? (uint64_t) x.tid : field == 1 ? dup_score_key(x.score) : field == 2 ? x.k2 : x.k1;
}

__global__ void dup_permute_kernel(const bm2_dup_entry *__restrict__ e, const uint32_t *__restrict__ ord, int64_t n, bm2_dup_entry *s) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) s[i] = e[ord[i]];
}

__global__ void dup_head_kernel(const bm2_dup_entry *__restrict__ s, int64_t n, int32_t *head) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) head[i] = (i == 0 || !dup_same_key(s[i], s[i - 1])) ? 1 : 0;
}

// seg: 1-based group numbers; per group whether it holds a pair-end entry, and its first entry that is not one
__global__ void dup_group_kernel(const bm2_dup_entry *__restrict__ s, const int32_t *__restrict__ seg, int64_t n, int32_t *has_pe, uint32_t *first) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t g = seg[i] - 1;
    if (s[i].kind == DUP_KIND_PAIR_END) atomicOr(has_pe + g, 1);
    else atomicMin(first + g, (uint32_t) i);
}

__global__ void dup_mark_kernel(const bm2_dup_entry *__restrict__ s, const int32_t *__restrict__ seg, const int32_t *__restrict__ has_pe,
                                const uint32_t *__restrict__ first, int64_t n, uint8_t *flag, int64_t *tid) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t g = seg[i] - 1;
    flag[i] = dup_is_duplicate(s[i].kind, has_pe[g], (int64_t) first[g], i) ? 1 : 0;
    tid[i] = s[i].tid;
}

enum { DD_IN, DD_STARTS, DD_TFIRST, DD_TID, DD_PAIR, DD_FRAG, DD_OUT, DD_CNT, DD_TEMP, DD_KEYS0, DD_KEYS1, DD_ORD0, DD_ORD1, DD_SORTED, DD_END };
static_assert(DD_END == std::extent<decltype(bm2_ctx::dup_d)>::value, "bm2_ctx::dup_d: one buffer per slot");
// bm2_dup_resolve reuses the signature slots: entries in DD_PAIR, group numbers / flags / ids in DD_IN / DD_STARTS / DD_TFIRST / DD_TID / DD_FRAG

int bits_of(uint64_t v) { int b = 0; while (b < 64 && (v >> b)) ++b; return b; }

int ensure_events(bm2_ctx *ctx) {
    bm2_ctx *ctx_for_error = ctx;
    for (cudaEvent_t &ev : ctx->dup_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    return 0;
}

}  // namespace

extern "C" int bm2_dup_signatures(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tmpl_first,
                                  const int64_t *tmpl_id, int64_t n_tmpl, const bm2_dup_entry **pairs, int64_t *n_pairs, const bm2_dup_entry **frags,
                                  int64_t *n_frags) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts) || n_tmpl < 0 || !tmpl_first || (n_tmpl && !tmpl_id) || !pairs ||
        !n_pairs || !frags || !n_frags) {
        if (ctx) bm2_set_error(ctx, "bm2_dup_signatures: bad arguments");
        return 1;
    }
    if (n_tmpl >= (1LL << 30)) { bm2_set_error(ctx, "bm2_dup_signatures: 2^30 templates or more in one call"); return 1; }
    if (tmpl_first[0] != 0 || tmpl_first[n_tmpl] != n_recs) { bm2_set_error(ctx, "bm2_dup_signatures: the templates do not cover the records"); return 1; }
    for (int64_t t = 0; t < n_tmpl; ++t)
        if (tmpl_first[t + 1] < tmpl_first[t]) { bm2_set_error(ctx, "bm2_dup_signatures: template " + std::to_string(t) + " ends before it starts"); return 1; }
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t s = starts[i];
        if (s < 0 || s + 36 > n || s + 4 + (int64_t) bam_le32(recs + s) > n || (i && s < starts[i - 1] + 4 + (int64_t) bam_le32(recs + starts[i - 1]))) {
            bm2_set_error(ctx, "bm2_dup_signatures: record " + std::to_string(i) + " does not lie within the buffer after the one before");
            return 1;
        }
    }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->dup_d;
    size_t temp = 0;
    BM2_CUDA_OK(cub::DeviceSelect::If(nullptr, temp, (bm2_dup_entry *) nullptr, (bm2_dup_entry *) nullptr, (int64_t *) nullptr,
                                      (int) bm2_max<int64_t>(2 * n_tmpl, 1), IsEntry(), st));
    if (ctx->ensure(b[DD_IN], (size_t) n + 16) || ctx->ensure(b[DD_STARTS], (size_t) n_recs * 8 + 8) ||
        ctx->ensure(b[DD_TFIRST], (size_t) (n_tmpl + 1) * 8) || ctx->ensure(b[DD_TID], (size_t) n_tmpl * 8 + 8) ||
        ctx->ensure(b[DD_PAIR], (size_t) n_tmpl * sizeof(bm2_dup_entry) + 8) || ctx->ensure(b[DD_FRAG], (size_t) 2 * n_tmpl * sizeof(bm2_dup_entry) + 8) ||
        ctx->ensure(b[DD_OUT], (size_t) 2 * n_tmpl * sizeof(bm2_dup_entry) + 8) || ctx->ensure(b[DD_CNT], 16) || ctx->ensure(b[DD_TEMP], temp + 16) ||
        ensure_events(ctx)) return 1;
    int64_t cnt[2] = { 0, 0 };
    ctx->dup_sig_ms = 0;
    if (n_tmpl) {
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_IN].p, recs, (size_t) n, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_TFIRST].p, tmpl_first, (size_t) (n_tmpl + 1) * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_TID].p, tmpl_id, (size_t) n_tmpl * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[0], st));
        dup_sig_kernel<<<(unsigned) ((n_tmpl * 32 + 255) / 256), 256, 0, st>>>((const uint8_t *) b[DD_IN].p, (const int64_t *) b[DD_STARTS].p,
                                                                              (const int64_t *) b[DD_TFIRST].p, (const int64_t *) b[DD_TID].p, n_tmpl,
                                                                              (bm2_dup_entry *) b[DD_PAIR].p, (bm2_dup_entry *) b[DD_FRAG].p);
        BM2_CUDA_OK(cudaGetLastError());
        bm2_dup_entry *outp = (bm2_dup_entry *) b[DD_OUT].p;
        size_t tb = b[DD_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceSelect::If(b[DD_TEMP].p, tb, (const bm2_dup_entry *) b[DD_PAIR].p, outp, (int64_t *) b[DD_CNT].p, (int) n_tmpl, IsEntry(), st));
        BM2_CUDA_OK(cudaMemcpyAsync(&cnt[0], b[DD_CNT].p, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        ctx->dup_pairs.resize((size_t) cnt[0]);
        if (cnt[0]) BM2_CUDA_OK(cudaMemcpyAsync(ctx->dup_pairs.data(), outp, (size_t) cnt[0] * sizeof(bm2_dup_entry), cudaMemcpyDeviceToHost, st));
        tb = b[DD_TEMP].cap;
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        BM2_CUDA_OK(cub::DeviceSelect::If(b[DD_TEMP].p, tb, (const bm2_dup_entry *) b[DD_FRAG].p, outp, (int64_t *) b[DD_CNT].p, (int) (2 * n_tmpl),
                                          IsEntry(), st));
        BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[1], st));
        BM2_CUDA_OK(cudaMemcpyAsync(&cnt[1], b[DD_CNT].p, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        ctx->dup_frags.resize((size_t) cnt[1]);
        if (cnt[1]) BM2_CUDA_OK(cudaMemcpy(ctx->dup_frags.data(), outp, (size_t) cnt[1] * sizeof(bm2_dup_entry), cudaMemcpyDeviceToHost));
        float ms = 0;
        BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->dup_ev[0], ctx->dup_ev[1]));
        ctx->dup_sig_ms = ms;
    } else { ctx->dup_pairs.clear(); ctx->dup_frags.clear(); }
    *pairs = ctx->dup_pairs.data(); *n_pairs = cnt[0];
    *frags = ctx->dup_frags.data(); *n_frags = cnt[1];
    return 0;
}

extern "C" int bm2_dup_resolve(bm2_ctx *ctx, const bm2_dup_entry *entries, int64_t n, int resolve, const bm2_dup_entry **sorted, const int64_t **dups,
                               int64_t *n_dups) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n < 0 || (n && !entries) || (!resolve && !sorted) || (resolve && (!dups || !n_dups))) {
        if (ctx) bm2_set_error(ctx, "bm2_dup_resolve: bad arguments");
        return 1;
    }
    if (n >= (1LL << 31) - 1) { bm2_set_error(ctx, "bm2_dup_resolve: 2^31-1 entries or more in one call"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->dup_d;
    const int ni = (int) bm2_max<int64_t>(n, 1);
    size_t temp = 0, t2 = 0;
    {
        cub::DoubleBuffer<uint64_t> k((uint64_t *) nullptr, nullptr); cub::DoubleBuffer<uint32_t> v((uint32_t *) nullptr, nullptr);
        BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, ni, 0, 64, st));
        BM2_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, t2, (const int32_t *) nullptr, (int32_t *) nullptr, ni, st));
        temp = bm2_max(temp, t2);
        BM2_CUDA_OK(cub::DeviceSelect::Flagged(nullptr, t2, (const int64_t *) nullptr, (const uint8_t *) nullptr, (int64_t *) nullptr, (int64_t *) nullptr,
                                               ni, st));
        temp = bm2_max(temp, t2);
    }
    const size_t ne = (size_t) n * sizeof(bm2_dup_entry) + 8;
    if (ctx->ensure(b[DD_PAIR], ne) || ctx->ensure(b[DD_SORTED], ne) || ctx->ensure(b[DD_KEYS0], (size_t) n * 8 + 8) ||
        ctx->ensure(b[DD_KEYS1], (size_t) n * 8 + 8) || ctx->ensure(b[DD_ORD0], (size_t) n * 4 + 8) || ctx->ensure(b[DD_ORD1], (size_t) n * 4 + 8) ||
        ctx->ensure(b[DD_CNT], 32) || ctx->ensure(b[DD_TEMP], temp + 16) || ensure_events(ctx)) return 1;
    if (resolve && (ctx->ensure(b[DD_IN], (size_t) n * 4 + 8) || ctx->ensure(b[DD_STARTS], (size_t) n * 4 + 8) ||
                    ctx->ensure(b[DD_TFIRST], (size_t) n * 4 + 8) || ctx->ensure(b[DD_TID], (size_t) n * 4 + 8) ||
                    ctx->ensure(b[DD_FRAG], (size_t) n * 9 + 32) || ctx->ensure(b[DD_OUT], (size_t) n * 8 + 8))) return 1;
    ctx->dup_resolve_ms = 0;
    ctx->dup_sorted.clear(); ctx->dup_ids.clear();
    if (n == 0) {
        if (sorted) *sorted = ctx->dup_sorted.data();
        if (resolve) { *dups = ctx->dup_ids.data(); *n_dups = 0; }
        return 0;
    }
    const unsigned g = (unsigned) ((n + 255) / 256);
    bm2_dup_entry *E = (bm2_dup_entry *) b[DD_PAIR].p, *S = (bm2_dup_entry *) b[DD_SORTED].p;
    BM2_CUDA_OK(cudaMemcpyAsync(E, entries, (size_t) n * sizeof(bm2_dup_entry), cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemsetAsync(b[DD_CNT].p, 0, 24, st));
    BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[0], st));
    dup_or_kernel<<<g, 256, 0, st>>>(E, n, (unsigned long long *) b[DD_CNT].p);
    BM2_CUDA_OK(cudaGetLastError());
    dup_iota_kernel<<<g, 256, 0, st>>>((uint32_t *) b[DD_ORD0].p, n);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[1], st));
    uint64_t ors[3] = { 0, 0, 0 };
    BM2_CUDA_OK(cudaMemcpyAsync(ors, b[DD_CNT].p, 24, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[2], st));
    // least significant field first: tid, descending score, k2, k1; each pass stable, over the bits that field uses
    const int bits[4] = { bits_of(ors[2]), 15, bits_of(ors[1]), bits_of(ors[0]) };
    cub::DoubleBuffer<uint64_t> kb((uint64_t *) b[DD_KEYS0].p, (uint64_t *) b[DD_KEYS1].p);
    cub::DoubleBuffer<uint32_t> vb((uint32_t *) b[DD_ORD0].p, (uint32_t *) b[DD_ORD1].p);
    for (int f = 0; f < 4; ++f) {
        if (!bits[f]) continue;
        dup_field_kernel<<<g, 256, 0, st>>>(E, vb.Current(), n, f, kb.Current());
        BM2_CUDA_OK(cudaGetLastError());
        size_t tb = b[DD_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(b[DD_TEMP].p, tb, kb, vb, (int) n, 0, bits[f], st));
    }
    dup_permute_kernel<<<g, 256, 0, st>>>(E, vb.Current(), n, S);
    BM2_CUDA_OK(cudaGetLastError());
    int64_t nd = 0;
    if (!resolve) {
        BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[3], st));
        ctx->dup_sorted.resize((size_t) n);
        BM2_CUDA_OK(cudaMemcpyAsync(ctx->dup_sorted.data(), S, (size_t) n * sizeof(bm2_dup_entry), cudaMemcpyDeviceToHost, st));
    } else {
        int32_t *head = (int32_t *) b[DD_IN].p, *seg = (int32_t *) b[DD_STARTS].p, *has_pe = (int32_t *) b[DD_TFIRST].p;
        uint32_t *first = (uint32_t *) b[DD_TID].p;
        uint8_t *flag = (uint8_t *) b[DD_FRAG].p;
        int64_t *tid = (int64_t *) ((uint8_t *) b[DD_FRAG].p + (((size_t) n + 15) & ~(size_t) 7));
        dup_head_kernel<<<g, 256, 0, st>>>(S, n, head);
        BM2_CUDA_OK(cudaGetLastError());
        size_t tb = b[DD_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceScan::InclusiveSum(b[DD_TEMP].p, tb, (const int32_t *) head, seg, (int) n, st));
        BM2_CUDA_OK(cudaMemsetAsync(has_pe, 0, (size_t) n * 4, st));
        BM2_CUDA_OK(cudaMemsetAsync(first, 0xFF, (size_t) n * 4, st));
        dup_group_kernel<<<g, 256, 0, st>>>(S, seg, n, has_pe, first);
        BM2_CUDA_OK(cudaGetLastError());
        dup_mark_kernel<<<g, 256, 0, st>>>(S, seg, has_pe, first, n, flag, tid);
        BM2_CUDA_OK(cudaGetLastError());
        tb = b[DD_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceSelect::Flagged(b[DD_TEMP].p, tb, (const int64_t *) tid, (const uint8_t *) flag, (int64_t *) b[DD_OUT].p,
                                               (int64_t *) b[DD_CNT].p, (int) n, st));
        BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[3], st));
        BM2_CUDA_OK(cudaMemcpyAsync(&nd, b[DD_CNT].p, 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        ctx->dup_ids.resize((size_t) nd);
        if (nd) BM2_CUDA_OK(cudaMemcpyAsync(ctx->dup_ids.data(), b[DD_OUT].p, (size_t) nd * 8, cudaMemcpyDeviceToHost, st));
    }
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms[2] = { 0, 0 };
    BM2_CUDA_OK(cudaEventElapsedTime(&ms[0], ctx->dup_ev[0], ctx->dup_ev[1]));
    BM2_CUDA_OK(cudaEventElapsedTime(&ms[1], ctx->dup_ev[2], ctx->dup_ev[3]));
    ctx->dup_resolve_ms = (double) ms[0] + ms[1];
    if (sorted) *sorted = ctx->dup_sorted.data();
    if (resolve) { *dups = ctx->dup_ids.data(); *n_dups = nd; }
    return 0;
}

extern "C" int bm2_last_dup_stats(const bm2_ctx *ctx, double *signatures_ms, double *resolve_ms) {
    if (!ctx) return 1;
    if (signatures_ms) *signatures_ms = ctx->dup_sig_ms;
    if (resolve_ms) *resolve_ms = ctx->dup_resolve_ms;
    return 0;
}

extern "C" int bm2_dup_set(bm2_ctx *ctx, const uint64_t *bits, int64_t n_bits) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n_bits < 0 || (n_bits && !bits)) { if (ctx) bm2_set_error(ctx, "bm2_dup_set: bad arguments"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    const size_t bytes = (size_t) ((n_bits + 63) / 64) * 8;
    if (bytes > ctx->dup_bits.cap) {
        size_t fr = 0, tot = 0;
        BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
        if (bytes > fr) {
            bm2_set_error(ctx, "bm2_dup_set: the duplicate bitset needs " + std::to_string(bytes) + " bytes of device memory, " + std::to_string(fr) +
                               " bytes free");
            return 1;
        }
    }
    if (ctx->ensure(ctx->dup_bits, bytes + 8)) return 1;
    if (bytes) BM2_CUDA_OK(cudaMemcpy(ctx->dup_bits.p, bits, bytes, cudaMemcpyHostToDevice));
    ctx->dup_n_bits = n_bits;
    return 0;
}

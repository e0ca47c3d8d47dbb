// wgs.cu — the per-base coverage of bm2_wgsmetrics on the GPU (wgs_device.cuh's rule).
//   bm2_wgs_set     one uint32 counter per reference base and the no-call bitset (1 bit per base, from the N / n / . holes); zeroes the counters
//   bm2_wgs_add     one window of records in file order: check, count, overlap pass (below)
//   bm2_wgs_finish  one streaming pass over every locus: the depth histogram and the capped bases
// Each window is uploaded after the carried records (the records of earlier windows a later record may still overlap), as one buffer.
//   check    one warp per record: the lanes sum the CIGAR (aligned, reference and query lengths), lane 0 applies the filters and writes the
//            record's placement and its sort key; a read error takes the first record by index (atomicMin).  Nothing is counted before the
//            host has seen that no record of the window is an error.
//   count    one warp per new record, grid-stride: the aligned bases of a filtered record go to its counter; the lanes walk a passing record's
//            CIGAR on consecutive bases, test the no-call bit, count EXC_BASEQ and atomicAdd each high-quality base's counter.  The exclusion
//            counts are summed over the warp and added once per warp.
//   overlap  the candidates (carried records and the window's passing ones) sorted by (name hash, file order) with cub; a warp takes each
//            run of two or more equal hashes.  For each new member and each of its high-quality loci, when an earlier member of the same name
//            (compared byte for byte) also has a high-quality base there, the locus's counter loses 1 and EXC_OVERLAP gains 1.  A carried
//            member was settled in its own window.  The lanes take consecutive loci of the new member; each lane finds the earlier
//            member's base at its locus by walking that member's CIGAR.
//   carry    after the window, the candidates on the last record's contig whose span ends past its start are kept (bytes, on the host)
//   finish   a grid-stride pass over the counters, four loci per thread: no-call loci are skipped, min(d, cap) is binned in a per-block
//            shared-memory histogram (one atomic per group of lanes with the same depth, __match_any_sync), flushed to 64-bit bins, and
//            max(0, d - cap) is summed.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "wgs_device.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kRecBytes = 300;              // a short read's record, for bm2_wgs_memory's estimate

__global__ void wgs_nocall_kernel(uint32_t *bits, int64_t n_words, const int64_t *ranges, int64_t n) {
    for (int64_t w = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t) gridDim.x * blockDim.x)
        bits[w] = wgs_range_word(ranges, n, w);
}

__global__ void __launch_bounds__(kWarps * 32) wgs_check_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                                int64_t n_carry, const int64_t *__restrict__ off, const int32_t *__restrict__ len,
                                                                int32_t n_contigs, bm2_wgs_params_t p, WgsInfo *info, uint64_t *keys, uint32_t *vals,
                                                                unsigned long long *err, int64_t first) {
    const int lane = threadIdx.x & 31;
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const uint8_t *r = base + starts[w];
        const DupCigar c = dup_cigar(r);
        const bool inside = wgs_cigar_inside(r, c);
        int64_t s[3] = {0, 0, 0};
        if (inside) wgs_cigar_part(c, lane, 32, s);
        for (int k = 0; k < 3; ++k)
            for (int o = 16; o; o >>= 1) s[k] += __shfl_xor_sync(kFull, s[k], o);
        if (lane == 0) {
            WgsInfo in;
            const int st = wgs_status(r, s, inside, off, len, n_contigs, p, in);
            info[w] = in;
            keys[w] = wgs_key(r, in);
            vals[w] = (uint32_t) w;
            if (st >= WGS_ERR_NOQUAL && w >= n_carry) atomicMin(err, (unsigned long long) (first + w - n_carry) << 4 | (unsigned) (st - WGS_ERR_NOQUAL + 1));
        }
    }
}

__global__ void __launch_bounds__(kWarps * 32) wgs_count_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                                int64_t n_carry, const WgsInfo *__restrict__ info, const uint32_t *__restrict__ nocall,
                                                                int min_baseq, uint32_t *pile, unsigned long long *exc) {
    const int lane = threadIdx.x & 31;
    unsigned long long c0 = 0, c1 = 0, c2 = 0, c3 = 0;                   // EXC_MAPQ, EXC_DUPE, EXC_UNPAIRED, EXC_BASEQ (registers, not an array)
    for (int64_t w = n_carry + (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const WgsInfo in = info[w];
        if (in.status <= WGS_FILT_UNPAIRED) {
            const unsigned long long a = lane == 0 ? (unsigned long long) in.aligned : 0;
            c0 += in.status == WGS_FILT_MAPQ ? a : 0; c1 += in.status == WGS_FILT_DUPE ? a : 0; c2 += in.status == WGS_FILT_UNPAIRED ? a : 0;
            continue;
        }
        if (in.status != WGS_PASS) continue;
        const uint8_t *r = base + starts[w];
        const DupCigar c = dup_cigar(r);
        const WgsSeq sq = wgs_seq(r);
        int64_t k = 0, g = in.g0;
        for (int64_t i = 0; i < c.n; ++i) {
            const uint32_t op = dup_op(c, i), ln = op >> 4;
            if (wgs_aligned_op(op))
                for (uint32_t b = lane; b < ln; b += 32) {
                    if (wgs_nocall(nocall, g + b)) continue;
                    if (wgs_hq(sq, k + b, min_baseq)) atomicAdd(&pile[g + b], 1u);
                    else ++c3;
                }
            if (dup_consumes_ref(op)) g += ln;
            if (wgs_query_op(op)) k += ln;
        }
    }
    for (int o = 16; o; o >>= 1) {
        c0 += __shfl_xor_sync(kFull, c0, o); c1 += __shfl_xor_sync(kFull, c1, o);
        c2 += __shfl_xor_sync(kFull, c2, o); c3 += __shfl_xor_sync(kFull, c3, o);
    }
    if (lane == 0) {
        if (c0) atomicAdd(&exc[WGS_EXC_MAPQ], c0);
        if (c1) atomicAdd(&exc[WGS_EXC_DUPE], c1);
        if (c2) atomicAdd(&exc[WGS_EXC_UNPAIRED], c2);
        if (c3) atomicAdd(&exc[WGS_EXC_BASEQ], c3);
    }
}

__global__ void __launch_bounds__(kWarps * 32) wgs_overlap_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                                  int64_t n_carry, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ vals,
                                                                  const WgsInfo *__restrict__ info, const uint32_t *__restrict__ nocall, int min_baseq,
                                                                  uint32_t *pile, unsigned long long *exc) {
    const int lane = threadIdx.x & 31;
    unsigned long long ov = 0;
    for (int64_t i = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); i < n; i += (int64_t) gridDim.x * kWarps) {
        const uint64_t key = keys[i];
        if ((key & WGS_NOT_CANDIDATE) || (i > 0 && keys[i - 1] == key)) continue;   // not a run's first member
        int64_t e = i + 1;
        while (e < n && keys[e] == key) ++e;
        for (int64_t j = i + 1; j < e; ++j) {
            const int64_t x = vals[j];
            if (x < n_carry) continue;                                   // settled in its own window
            const WgsInfo in = info[x];
            const uint8_t *r = base + starts[x];
            const DupCigar c = dup_cigar(r);
            const WgsSeq sq = wgs_seq(r);
            int64_t k = 0, g = in.g0;
            for (int64_t op_i = 0; op_i < c.n; ++op_i) {
                const uint32_t op = dup_op(c, op_i), ln = op >> 4;
                if (wgs_aligned_op(op))
                    for (uint32_t b0 = 0; b0 < ln; b0 += 32) {
                        const uint32_t b = b0 + lane;
                        const int64_t gg = g + b;
                        const bool hq = b < ln && !wgs_nocall(nocall, gg) && wgs_hq(sq, k + b, min_baseq);
                        if (!__any_sync(kFull, hq)) continue;
                        bool cov = false;
                        for (int64_t m = i; m < j; ++m) {                // the earlier members of the run
                            const int64_t y = vals[m];
                            const WgsInfo im = info[y];
                            if (!wgs_spans_overlap(im, in)) continue;
                            const uint8_t *rm = base + starts[y];
                            if (!wgs_same_name(rm, r)) continue;
                            if (hq && !cov) cov = wgs_hq_at(rm, dup_cigar(rm), im.g0, gg, min_baseq);
                        }
                        if (cov) { atomicSub(&pile[gg], 1u); ++ov; }
                    }
                if (dup_consumes_ref(op)) g += ln;
                if (wgs_query_op(op)) k += ln;
            }
        }
    }
    for (int o = 16; o; o >>= 1) ov += __shfl_xor_sync(kFull, ov, o);
    if (lane == 0 && ov) atomicAdd(&exc[WGS_EXC_OVERLAP], ov);
}

__global__ void __launch_bounds__(256) wgs_finish_kernel(const uint32_t *__restrict__ pile, const uint32_t *__restrict__ nocall, int64_t l_pac, int cap,
                                                         unsigned long long *hist, unsigned long long *exc) {
    extern __shared__ uint32_t s_bins[];
    for (int d = threadIdx.x; d <= cap; d += blockDim.x) s_bins[d] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    unsigned long long capped = 0;
    const int64_t n4 = (l_pac + 3) / 4;
    const uint4 *p4 = (const uint4 *) pile;
    const int64_t stride = (int64_t) gridDim.x * blockDim.x;
    for (int64_t t0 = (int64_t) blockIdx.x * blockDim.x; t0 < n4; t0 += stride) {   // warp-uniform trip count: the whole warp takes part
        const int64_t t = t0 + threadIdx.x;
        uint4 v = make_uint4(0, 0, 0, 0);
        uint32_t skip = 0xF;
        if (t < n4) {
            v = __ldcs(p4 + t);
            const int64_t g = 4 * t;
            skip = (nocall[g >> 5] >> (g & 31)) & 0xF;
            if (g + 4 > l_pac) skip |= 0xFu << (l_pac - g) & 0xF;
        }
        const uint32_t d[4] = {v.x, v.y, v.z, v.w};
        for (int q = 0; q < 4; ++q) {
            const bool on = !((skip >> q) & 1);
            if (on && d[q] > (uint32_t) cap) capped += d[q] - (uint32_t) cap;
            const int bin = on ? (int) bm2_min<uint32_t>(d[q], (uint32_t) cap) : -1;
            const unsigned grp = __match_any_sync(kFull, bin);
            if (bin >= 0 && lane == __ffs(grp) - 1) atomicAdd(&s_bins[bin], (uint32_t) __popc(grp));
        }
    }
    for (int o = 16; o; o >>= 1) capped += __shfl_xor_sync(kFull, capped, o);
    if (lane == 0 && capped) atomicAdd(&exc[WGS_EXC_CAPPED], capped);
    __syncthreads();
    for (int d = threadIdx.x; d <= cap; d += blockDim.x) if (s_bins[d]) atomicAdd(&hist[d], (unsigned long long) s_bins[d]);
}

enum { WG_PILE, WG_NOCALL, WG_RANGES, WG_OFF, WG_LEN, WG_EXC, WG_HIST, WG_ERR, WG_RECS, WG_STARTS, WG_INFO, WG_KEYS, WG_VALS, WG_KEYS2, WG_VALS2,
       WG_TEMP, WG_END };
static_assert(WG_END == std::extent<decltype(bm2_ctx::wgs_d)>::value, "bm2_ctx::wgs_d: one buffer per slot");

const char *const kErrText[3] = {"has no base qualities (l_seq 0 or QUAL '*')", "does not lie inside a contig of the reference",
                                 "has a CIGAR that does not match its record"};

// exactly `bytes` (the counters are too large for bm2_ctx::ensure's 25% headroom)
int ensure_exact(bm2_ctx *ctx, DevBuf &b, size_t bytes) {
    bm2_ctx *ctx_for_error = ctx;
    if (b.cap >= bytes) return 0;
    if (b.p) BM2_CUDA_OK(cudaFree(b.p));
    b.p = nullptr; b.cap = 0;
    BM2_CUDA_OK(cudaMalloc(&b.p, bytes));
    b.cap = bytes;
    return 0;
}

size_t pile_bytes(int64_t l_pac) { return (size_t) ((l_pac + 3) / 4) * 16; }
size_t nocall_bytes(int64_t l_pac) { return (size_t) ((l_pac + 127) / 128) * 16; }

}  // namespace

extern "C" int bm2_wgs_set(bm2_ctx *ctx, const int64_t *contig_off, const int32_t *contig_len, int32_t n_contigs, int64_t l_pac, const int64_t *nocall,
                           int64_t n_nocall, const bm2_wgs_params_t *params) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n_contigs < 0 || (n_contigs && (!contig_off || !contig_len)) || l_pac < 1 || n_nocall < 0 || (n_nocall && !nocall) || !params ||
        params->min_mapq < 0 || params->min_baseq < 0 || params->coverage_cap < 1 || params->coverage_cap > BM2_WGS_MAX_CAP) {
        if (ctx) bm2_set_error(ctx, "bm2_wgs_set: bad arguments");
        return 1;
    }
    for (int32_t k = 0; k < n_contigs; ++k)
        if (contig_off[k] < 0 || contig_len[k] < 0 || contig_off[k] + contig_len[k] > l_pac) {
            bm2_set_error(ctx, "bm2_wgs_set: contig " + std::to_string(k) + " does not lie inside the reference"); return 1;
        }
    for (int64_t h = 0; h < n_nocall; ++h)
        if (nocall[2 * h] < 0 || nocall[2 * h + 1] < nocall[2 * h] || nocall[2 * h + 1] > l_pac || (h && nocall[2 * h] < nocall[2 * h - 1])) {
            bm2_set_error(ctx, "bm2_wgs_set: the no-call ranges must be sorted [beg, end) ranges inside the reference"); return 1;
        }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->wgs_d;
    const size_t pb = pile_bytes(l_pac), nb = nocall_bytes(l_pac);
    if (b[WG_PILE].cap < pb || b[WG_NOCALL].cap < nb) {
        size_t fr = 0, tot = 0;
        BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
        fr += b[WG_PILE].cap + b[WG_NOCALL].cap;
        if (pb + nb > fr) {
            bm2_set_error(ctx, "bm2_wgs_set: the coverage counters need " + std::to_string(pb + nb) + " bytes of device memory, " + std::to_string(fr) +
                               " bytes free");
            return 1;
        }
        for (int s : {WG_PILE, WG_NOCALL}) { if (b[s].p) BM2_CUDA_OK(cudaFree(b[s].p)); b[s].p = nullptr; b[s].cap = 0; }
    }
    if (ensure_exact(ctx, b[WG_PILE], pb) || ensure_exact(ctx, b[WG_NOCALL], nb) || ctx->ensure(b[WG_RANGES], (size_t) n_nocall * 16 + 16) ||
        ctx->ensure(b[WG_OFF], (size_t) n_contigs * 8 + 8) || ctx->ensure(b[WG_LEN], (size_t) n_contigs * 4 + 8) ||
        ctx->ensure(b[WG_EXC], WGS_NEXC * 8) || ctx->ensure(b[WG_HIST], (size_t) (params->coverage_cap + 1) * 8) || ctx->ensure(b[WG_ERR], 8)) return 1;
    cudaStream_t st = ctx->stream;
    BM2_CUDA_OK(cudaMemsetAsync(b[WG_PILE].p, 0, pb, st));
    if (n_nocall) BM2_CUDA_OK(cudaMemcpyAsync(b[WG_RANGES].p, nocall, (size_t) n_nocall * 16, cudaMemcpyHostToDevice, st));
    if (n_contigs) {
        BM2_CUDA_OK(cudaMemcpyAsync(b[WG_OFF].p, contig_off, (size_t) n_contigs * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[WG_LEN].p, contig_len, (size_t) n_contigs * 4, cudaMemcpyHostToDevice, st));
    }
    const int64_t n_words = (int64_t) nb / 4;
    wgs_nocall_kernel<<<(unsigned) bm2_min<int64_t>((n_words + 255) / 256, (int64_t) ctx->n_sm * 16), 256, 0, st>>>(
        (uint32_t *) b[WG_NOCALL].p, n_words, (const int64_t *) b[WG_RANGES].p, n_nocall);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaMemsetAsync(b[WG_EXC].p, 0, WGS_NEXC * 8, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    ctx->wgs_params = *params; ctx->wgs_l_pac = l_pac; ctx->wgs_n_contigs = n_contigs;
    ctx->wgs_contig_off.assign(contig_off, contig_off + n_contigs);
    ctx->wgs_seen = 0; ctx->wgs_counted = 0; ctx->wgs_carried_max = 0; ctx->wgs_add_ms = 0; ctx->wgs_finish_ms = 0;
    ctx->wgs_carry.clear(); ctx->wgs_carry_starts.clear();
    ctx->wgs_set = true;
    return 0;
}

extern "C" int bm2_wgs_memory(const bm2_ctx *ctx, int64_t l_pac, int64_t window_bytes, int64_t *needed, int64_t *free_bytes) {
    if (!ctx || l_pac < 0 || window_bytes < 0 || !needed || !free_bytes) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // the counters and the bitset exactly; the window with room for as many carried bytes again, and per record its start, placement, two
    // key / value pairs and the sort's scratch, rounded up by 1.25 as bm2_ctx::ensure allocates
    const double w = 2.0 * (double) window_bytes, recs = w / kRecBytes + 1;
    const double bytes = (double) pile_bytes(l_pac) + (double) nocall_bytes(l_pac) + 1.25 * (w + recs * (8 + sizeof(WgsInfo) + 2 * 12 + 32)) +
                         64.0 * (1 << 20);
    size_t fr = 0, tot = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
    *needed = (int64_t) bytes; *free_bytes = (int64_t) fr + (int64_t) (ctx->wgs_d[WG_PILE].cap + ctx->wgs_d[WG_NOCALL].cap);
    return 0;
}

extern "C" int bm2_wgs_add(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts)) { if (ctx) bm2_set_error(ctx, "bm2_wgs_add: bad arguments"); return 1; }
    if (!ctx->wgs_set) { bm2_set_error(ctx, "bm2_wgs_add: no counters on this context (bm2_wgs_set)"); return 1; }
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t s = starts[i];
        if (s < 0 || s + 36 > n) { bm2_set_error(ctx, "bm2_wgs_add: record " + std::to_string(i) + " is not inside the buffer"); return 1; }
        const BamFixed f = bam_fixed(recs + s);
        const int32_t l_seq = bam_le32(recs + s + 20);
        if (f.block_size < 32 || s + 4 + (int64_t) f.block_size > n || l_seq < 0 || f.l_read_name < 1 ||
            32 + (int64_t) f.l_read_name + 4 * (int64_t) f.n_cigar + (l_seq + 1) / 2 + (int64_t) l_seq > (int64_t) f.block_size) {
            bm2_set_error(ctx, "bm2_wgs_add: record " + std::to_string(i) + " is malformed");
            return 1;
        }
    }
    if (!n_recs) return 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->wgs_d;
    const int64_t n_carry = (int64_t) ctx->wgs_carry_starts.size(), carry_len = (int64_t) ctx->wgs_carry.size(), n_all = n_carry + n_recs;
    if (n_all >= ((int64_t) 1 << 32)) { bm2_set_error(ctx, "bm2_wgs_add: more than 2^32 - 1 records in one window"); return 1; }
    std::vector<int64_t> all_starts(ctx->wgs_carry_starts);
    for (int64_t i = 0; i < n_recs; ++i) all_starts.push_back(carry_len + starts[i]);
    size_t temp = 0;
    {
        cub::DoubleBuffer<uint64_t> k((uint64_t *) nullptr, nullptr); cub::DoubleBuffer<uint32_t> v((uint32_t *) nullptr, nullptr);
        BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int) n_all, 0, 64, st));
    }
    const size_t na = (size_t) n_all;
    if (ctx->ensure(b[WG_RECS], (size_t) (carry_len + n) + 16) || ctx->ensure(b[WG_STARTS], na * 8 + 8) || ctx->ensure(b[WG_INFO], na * sizeof(WgsInfo) + 8) ||
        ctx->ensure(b[WG_KEYS], na * 8 + 8) || ctx->ensure(b[WG_VALS], na * 4 + 8) || ctx->ensure(b[WG_KEYS2], na * 8 + 8) ||
        ctx->ensure(b[WG_VALS2], na * 4 + 8) || ctx->ensure(b[WG_TEMP], temp + 16)) return 1;
    for (cudaEvent_t &ev : ctx->wgs_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    uint8_t *d_recs = (uint8_t *) b[WG_RECS].p;
    const int64_t *d_starts = (const int64_t *) b[WG_STARTS].p;
    WgsInfo *d_info = (WgsInfo *) b[WG_INFO].p;
    const uint32_t *d_nocall = (const uint32_t *) b[WG_NOCALL].p;
    uint32_t *d_pile = (uint32_t *) b[WG_PILE].p;
    unsigned long long *d_exc = (unsigned long long *) b[WG_EXC].p;
    if (carry_len) BM2_CUDA_OK(cudaMemcpyAsync(d_recs, ctx->wgs_carry.data(), (size_t) carry_len, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(d_recs + carry_len, recs, (size_t) n, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(b[WG_STARTS].p, all_starts.data(), na * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemsetAsync(b[WG_ERR].p, 0xff, 8, st));
    const unsigned g = (unsigned) bm2_min<int64_t>((n_all + kWarps - 1) / kWarps, (int64_t) ctx->n_sm * 8);
    BM2_CUDA_OK(cudaEventRecord(ctx->wgs_ev[0], st));
    wgs_check_kernel<<<g, kWarps * 32, 0, st>>>(d_recs, d_starts, n_all, n_carry, (const int64_t *) b[WG_OFF].p, (const int32_t *) b[WG_LEN].p,
                                                ctx->wgs_n_contigs, ctx->wgs_params, d_info, (uint64_t *) b[WG_KEYS].p, (uint32_t *) b[WG_VALS].p,
                                                (unsigned long long *) b[WG_ERR].p, ctx->wgs_seen);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->wgs_ev[1], st));
    unsigned long long err = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&err, b[WG_ERR].p, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->wgs_ev[0], ctx->wgs_ev[1]));
    ctx->wgs_add_ms += ms;
    if (err != ~0ULL) {                                                  // a read error: nothing of this window is counted
        const int64_t idx = (int64_t) (err >> 4), i = idx - ctx->wgs_seen;
        const uint8_t *r = recs + starts[i];
        bm2_set_error(ctx, "bm2_wgs_add: read " + std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0) + " (record " + std::to_string(idx) + ") " +
                               kErrText[(err & 15) - 1]);
        return 2;
    }
    BM2_CUDA_OK(cudaEventRecord(ctx->wgs_ev[0], st));
    wgs_count_kernel<<<g, kWarps * 32, 0, st>>>(d_recs, d_starts, n_all, n_carry, d_info, d_nocall, ctx->wgs_params.min_baseq, d_pile, d_exc);
    BM2_CUDA_OK(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> kb((uint64_t *) b[WG_KEYS].p, (uint64_t *) b[WG_KEYS2].p);
    cub::DoubleBuffer<uint32_t> vb((uint32_t *) b[WG_VALS].p, (uint32_t *) b[WG_VALS2].p);
    BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(b[WG_TEMP].p, temp, kb, vb, (int) n_all, 0, 64, st));
    wgs_overlap_kernel<<<g, kWarps * 32, 0, st>>>(d_recs, d_starts, n_all, n_carry, kb.Current(), vb.Current(), d_info, d_nocall,
                                                  ctx->wgs_params.min_baseq, d_pile, d_exc);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->wgs_ev[1], st));
    std::vector<WgsInfo> info(na);
    BM2_CUDA_OK(cudaMemcpyAsync(info.data(), d_info, na * sizeof(WgsInfo), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->wgs_ev[0], ctx->wgs_ev[1]));
    ctx->wgs_add_ms += ms;
    for (int64_t i = n_carry; i < n_all; ++i) ctx->wgs_counted += info[(size_t) i].status == WGS_PASS;
    // the carry: candidates a later record may still overlap, in file order
    const BamFixed lf = bam_fixed(recs + starts[n_recs - 1]);
    const int64_t last_g = lf.rid >= 0 && lf.rid < ctx->wgs_n_contigs ? ctx->wgs_contig_off[(size_t) lf.rid] + lf.pos : 0;
    std::vector<uint8_t> carry;
    std::vector<int64_t> cst;
    for (int64_t i = 0; i < n_all; ++i) {
        if (!wgs_carried(info[(size_t) i], lf.rid, last_g)) continue;
        const uint8_t *r = i < n_carry ? ctx->wgs_carry.data() + all_starts[(size_t) i] : recs + starts[i - n_carry];
        cst.push_back((int64_t) carry.size());
        carry.insert(carry.end(), r, r + 4 + bam_le32(r));
    }
    ctx->wgs_carry.swap(carry); ctx->wgs_carry_starts.swap(cst);
    ctx->wgs_carried_max = bm2_max<int64_t>(ctx->wgs_carried_max, (int64_t) ctx->wgs_carry_starts.size());
    ctx->wgs_seen += n_recs;
    return 0;
}

extern "C" int bm2_wgs_finish(bm2_ctx *ctx, bm2_wgs_result_t *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out) { if (ctx) bm2_set_error(ctx, "bm2_wgs_finish: bad arguments"); return 1; }
    if (!ctx->wgs_set) { bm2_set_error(ctx, "bm2_wgs_finish: no counters on this context (bm2_wgs_set)"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->wgs_d;
    const int cap = ctx->wgs_params.coverage_cap;
    for (cudaEvent_t &ev : ctx->wgs_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    BM2_CUDA_OK(cudaMemsetAsync(b[WG_HIST].p, 0, (size_t) (cap + 1) * 8, st));
    BM2_CUDA_OK(cudaMemsetAsync((unsigned long long *) b[WG_EXC].p + WGS_EXC_CAPPED, 0, 8, st));
    // enough blocks that no block's 32-bit bins see 2^31 loci
    const int64_t n4 = (ctx->wgs_l_pac + 3) / 4;
    const int64_t grid = bm2_max<int64_t>(bm2_min<int64_t>((n4 + 255) / 256, (int64_t) ctx->n_sm * 4), (ctx->wgs_l_pac >> 31) + 1);
    BM2_CUDA_OK(cudaEventRecord(ctx->wgs_ev[0], st));
    wgs_finish_kernel<<<(unsigned) grid, 256, (size_t) (cap + 1) * 4, st>>>((const uint32_t *) b[WG_PILE].p, (const uint32_t *) b[WG_NOCALL].p,
                                                                           ctx->wgs_l_pac, cap, (unsigned long long *) b[WG_HIST].p,
                                                                           (unsigned long long *) b[WG_EXC].p);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->wgs_ev[1], st));
    ctx->wgs_hist.assign((size_t) cap + 1, 0);
    int64_t exc[WGS_NEXC];
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->wgs_hist.data(), b[WG_HIST].p, (size_t) (cap + 1) * 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(exc, b[WG_EXC].p, sizeof exc, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->wgs_ev[0], ctx->wgs_ev[1]));
    ctx->wgs_finish_ms = ms;
    out->hist = ctx->wgs_hist.data(); out->cap = cap;
    for (int k = 0; k < WGS_NEXC; ++k) out->exc[k] = exc[k];
    out->records = ctx->wgs_seen; out->counted_records = ctx->wgs_counted; out->carried_max = ctx->wgs_carried_max;
    out->add_ms = ctx->wgs_add_ms; out->finish_ms = ctx->wgs_finish_ms;
    return 0;
}

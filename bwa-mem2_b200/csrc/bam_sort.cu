// bam_sort.cu — coordinate sort of BAM records on the GPU, compressed as they leave (bm2_bam_sort_compress): one buffer of records (a
// sorted run of bm2_mem --sort, or a merge window) in, BGZF members of carry + the sorted records out, with every record's index data.
//   upload      the records and their starts (host)
//   keys        one thread per record: its fixed fields, end and bin (bam_sort_device.cuh), its length, and the largest refID and pos + 1
//   pack        the coordinate key squeezed into the bits the refIDs and positions use (refID -1 ranked after the largest refID), the
//               ordinal as the value; then cub::DeviceRadixSort::SortPairs over those bits only: LSD radix sort is stable, so ties keep
//               input order
//   scan        the lengths in sorted order, an exclusive scan: each record's place after the carry
//   gather      one warp per record, 16-byte copies when source and destination agree modulo 16
//   BGZF        the blocks are cut on the host (bam_sort_layout) from the scan, and bm2_bgzf_compress's kernels compress them straight from the
//               sorted device buffer; the unfinished last block goes back as the carry (bam_compress_stream, which bm2_bqsr_apply shares)
// bm2_bam_qname_sort_compress (bm2_sort -n) is the same code with only the keys and sort stages changed:
//   keys        the same key kernel (the index data and lengths), then one thread per record writes its 8-byte entry: the offset of its QNAME in
//               the uploaded buffer and its flag & 0xc0 (bam_qname_entry); the names are not copied
//   sort        cub::DeviceMergeSort::SortKeys over the 32-bit ordinals with bam_qname_cmp (bam_sort_device.cuh) as the comparison: names,
//               then flag bits, then ordinal, a total order, so ties keep input order
// bm2_bam_sort_compress_ex is the same code with one template id per record carried through the permutation; with a duplicate bitset on the
// context (bm2_dup_set, markdup.cu) the key kernel sets 0x400 in the index data of the records of duplicate templates and the gather writes it
// into the copied record.  With counting armed (bm2_bqsr_sites, bqsr.cu), the sorted records are counted for the recalibration tables after
// the gather, where they carry their duplicate flags, and before BGZF.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "bam_sort_device.cuh"
#include "markdup_device.cuh"
#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <vector>

namespace {

constexpr int kRecBytes = 300;      // a short read's record, for bm2_bam_sort_memory's estimate

// tids / dup_bits (bm2_bam_sort_compress_ex with a bitset): a record of a duplicate template that lacks 0x4 gets 0x400 in its info's flag
__global__ void sort_key_kernel(const uint8_t *__restrict__ in, const int64_t *__restrict__ starts, int64_t n, bm2_sort_rec *info,
                                int64_t *len, unsigned *maxes, const int64_t *__restrict__ tids, const uint64_t *__restrict__ dup_bits, int64_t n_bits) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    unsigned mr = 0, mp = 0;
    if (i < n) {
        const uint8_t *r = in + starts[i];
        bm2_sort_rec s = bam_sort_rec(r);
        if (dup_bits) s.flag = dup_marked_flag(s.flag, tids[i], dup_bits, n_bits);
        info[i] = s;
        len[i] = 4 + (int64_t) bam_le32(r);
        mr = s.rid >= 0 ? (unsigned) s.rid + 1 : 0;
        mp = (unsigned) (s.pos + 1);
    }
    for (int o = 16; o; o >>= 1) { mr = max(mr, __shfl_xor_sync(0xFFFFFFFFu, mr, o)); mp = max(mp, __shfl_xor_sync(0xFFFFFFFFu, mp, o)); }
    if ((threadIdx.x & 31) == 0) { atomicMax(maxes, mr); atomicMax(maxes + 1, mp); }
}

// rank(refID) << (pos_bits + 1) | (pos + 1) << 1 | reverse: the order of samtools' key, in rank_bits + pos_bits + 1 bits
__global__ void sort_pack_kernel(const bm2_sort_rec *__restrict__ info, int64_t n, unsigned unplaced_rank, int pos_bits, uint64_t *keys,
                                 uint32_t *vals) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bm2_sort_rec s = info[i];
    const uint64_t rank = s.rid >= 0 ? (uint64_t) s.rid : unplaced_rank;
    keys[i] = rank << (pos_bits + 1) | (uint64_t) (uint32_t) (s.pos + 1) << 1 | (uint64_t) ((s.flag & 16) ? 1 : 0);
    vals[i] = (uint32_t) i;
}

__global__ void sort_permute_kernel(const uint32_t *__restrict__ ord, int64_t n, const int64_t *__restrict__ len, const bm2_sort_rec *__restrict__ info,
                                    int64_t *len_sorted, bm2_sort_rec *info_sorted, const int64_t *__restrict__ tids, int64_t *tids_sorted) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { len_sorted[n] = 0; return; }
    const uint32_t k = ord[i];
    len_sorted[i] = len[k]; info_sorted[i] = info[k];
    if (tids) tids_sorted[i] = tids[k];
}

// one warp per record: in + starts[ord[i]] -> out + base + offs[i]; with info_sorted (marking), a flag with 0x400 replaces the copied one
__global__ void sort_gather_kernel(const uint8_t *__restrict__ in, const int64_t *__restrict__ starts, const uint32_t *__restrict__ ord,
                                   const int64_t *__restrict__ offs, const int64_t *__restrict__ len, int64_t n, int64_t base, uint8_t *out,
                                   const bm2_sort_rec *__restrict__ info_sorted) {
    const int64_t w = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n) return;
    const uint8_t *s = in + starts[ord[w]];
    uint8_t *d = out + base + offs[w];
    const int64_t m = len[w];
    int64_t head = 0, body = 0;
    if ((((uintptr_t) s ^ (uintptr_t) d) & 15) == 0) {
        head = bm2_min<int64_t>(m, (16 - ((uintptr_t) d & 15)) & 15);
        body = (m - head) & ~(int64_t) 15;
    }
    for (int64_t k = lane; k < head; k += 32) d[k] = s[k];
    const uint4 *s4 = (const uint4 *) (s + head);
    uint4 *d4 = (uint4 *) (d + head);
    for (int64_t k = lane; k < body / 16; k += 32) d4[k] = s4[k];
    for (int64_t k = head + body + lane; k < m; k += 32) d[k] = s[k];
    if (info_sorted) {
        const uint16_t f = info_sorted[w].flag;
        __syncwarp();
        if (lane == 0 && (f & 0x400)) { d[18] = (uint8_t) f; d[19] = (uint8_t) (f >> 8); }
    }
}

// name order: one thread per record, its entry and its ordinal
__global__ void qname_key_kernel(const uint8_t *__restrict__ in, const int64_t *__restrict__ starts, int64_t n, uint64_t *ent, uint32_t *ord) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ent[i] = bam_qname_entry(in + starts[i], starts[i]);
    ord[i] = (uint32_t) i;
}

// the name order of two ordinals, through their entries into the uploaded records
struct QnameLess {
    const uint8_t *in; const uint64_t *ent;
    __device__ bool operator()(uint32_t a, uint32_t b) const {
        const uint64_t x = ent[a], y = ent[b];
        return bam_qname_cmp(in + (x >> 8), (uint32_t) (x & 0xc0), a, in + (y >> 8), (uint32_t) (y & 0xc0), b) < 0;
    }
};

size_t qname_sort_temp(int64_t n, cudaStream_t st, cudaError_t *e) {
    size_t t = 0;
    *e = cub::DeviceMergeSort::SortKeys(nullptr, t, (uint32_t *) nullptr, n, QnameLess{nullptr, nullptr}, st);
    return t;
}

enum { SD_IN, SD_STARTS, SD_INFO, SD_LEN, SD_KEYS0, SD_KEYS1, SD_VALS0, SD_VALS1, SD_LENS, SD_OFFS, SD_TEMP, SD_OUT, SD_SINFO, SD_MAX, SD_TIDS,
       SD_STIDS, SD_END };
enum { SH_OFFS, SH_INFO, SH_END };
static_assert(SD_END == std::extent<decltype(bm2_ctx::sort_d)>::value, "bm2_ctx::sort_d: one buffer per slot");
static_assert(SH_END == std::extent<decltype(bm2_ctx::sort_h)>::value, "bm2_ctx::sort_h: one buffer per slot");

int bits_of(uint64_t v) { int b = 0; while (v >> b) ++b; return b; }

}  // namespace

// bm2_bam_sort_compress and bm2_bam_sort_compress_ex: tids (may be NULL) carried into ctx->sort_tids; marking when tids and a bitset are there.
// by_name: bm2_bam_qname_sort_compress (no tids)
static int sort_compress(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tids, const uint8_t *carry,
                         int64_t carry_len, int last, bm2_sort_out *out, bool by_name = false) {
    bm2_ctx *ctx_for_error = ctx;
    const std::string what = by_name ? "bm2_bam_qname_sort_compress" : "bm2_bam_sort_compress";
    if (!ctx || !out || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts) || carry_len < 0 || carry_len >= BGZF_BLOCK ||
        (carry_len && !carry)) {
        if (ctx) bm2_set_error(ctx, what + ": bad arguments");
        return 1;
    }
    const bool mark = tids && ctx->dup_n_bits > 0;
    if (n_recs >= (1LL << 31) - 1) { bm2_set_error(ctx, what + ": 2^31-1 records or more in one call"); return 1; }
    for (int64_t i = 0; i < n_recs; ++i) {                       // each record whole inside the buffer, in order, not overlapping the next
        const int64_t s = starts[i];
        if (s < 0 || s + 36 > n || (i && s < starts[i - 1] + 4 + (int64_t) bam_le32(recs + starts[i - 1]))) {
            bm2_set_error(ctx, what + ": record " + std::to_string(i) + " does not lie within the buffer after the one before");
            return 1;
        }
        const int64_t m = 4 + (int64_t) bam_le32(recs + s);
        const int32_t rid = bam_le32(recs + s + 4);
        if (m < 36 || s + m > n || rid < -1) { bm2_set_error(ctx, what + ": record " + std::to_string(i) + " is malformed"); return 1; }
    }
    memset(out, 0, sizeof *out);
    for (double &x : ctx->sort_ms) x = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->sort_d;
    const int64_t nr = n_recs;
    size_t temp = 0;
    if (by_name) {
        cudaError_t e;
        temp = qname_sort_temp(bm2_max<int64_t>(nr, 1), st, &e);
        BM2_CUDA_OK(e);
    } else {
        cub::DoubleBuffer<uint64_t> k((uint64_t *) nullptr, nullptr); cub::DoubleBuffer<uint32_t> v((uint32_t *) nullptr, nullptr);
        BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, (int) bm2_max<int64_t>(nr, 1), 0, 64, st));
    }
    {
        size_t t2 = 0;
        BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, t2, (int64_t *) nullptr, (int64_t *) nullptr, (int) nr + 1, st));
        temp = bm2_max(temp, t2);
    }
    if (ctx->ensure(b[SD_IN], (size_t) n + 16) || ctx->ensure(b[SD_STARTS], (size_t) nr * 8 + 8) ||
        ctx->ensure(b[SD_INFO], (size_t) nr * sizeof(bm2_sort_rec) + 8) || ctx->ensure(b[SD_LEN], (size_t) nr * 8 + 8) ||
        ctx->ensure(b[SD_KEYS0], (size_t) nr * 8 + 8) || ctx->ensure(b[SD_KEYS1], (size_t) nr * 8 + 8) ||
        ctx->ensure(b[SD_VALS0], (size_t) nr * 4 + 8) || ctx->ensure(b[SD_VALS1], (size_t) nr * 4 + 8) ||
        ctx->ensure(b[SD_LENS], (size_t) nr * 8 + 8) || ctx->ensure(b[SD_OFFS], (size_t) nr * 8 + 8) || ctx->ensure(b[SD_TEMP], temp + 16) ||
        ctx->ensure(b[SD_OUT], (size_t) (carry_len + n) + 16) || ctx->ensure(b[SD_SINFO], (size_t) nr * sizeof(bm2_sort_rec) + 8) ||
        ctx->ensure(b[SD_MAX], 16) || ctx->ensure_host(ctx->sort_h[SH_OFFS], (size_t) nr * 8 + 16) ||
        ctx->ensure_host(ctx->sort_h[SH_INFO], (size_t) nr * sizeof(bm2_sort_rec) + 16)) return 1;
    if (tids && (ctx->ensure(b[SD_TIDS], (size_t) nr * 8 + 8) || ctx->ensure(b[SD_STIDS], (size_t) nr * 8 + 8))) return 1;
    int64_t *d_tids = tids ? (int64_t *) b[SD_TIDS].p : nullptr, *d_stids = tids ? (int64_t *) b[SD_STIDS].p : nullptr;
    ctx->sort_tids.resize(tids ? (size_t) nr : 0);
    for (cudaEvent_t &ev : ctx->sort_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    if (carry_len) BM2_CUDA_OK(cudaMemcpy(b[SD_OUT].p, carry, (size_t) carry_len, cudaMemcpyHostToDevice));   // carry may be this context's last carry
    int64_t *h_offs = (int64_t *) ctx->sort_h[SH_OFFS].p;
    bm2_sort_rec *h_info = (bm2_sort_rec *) ctx->sort_h[SH_INFO].p;
    const uint32_t *ord = (const uint32_t *) b[SD_VALS0].p;
    if (nr) {
        BM2_CUDA_OK(cudaMemcpyAsync(b[SD_IN].p, recs, (size_t) n, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[SD_STARTS].p, starts, (size_t) nr * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemsetAsync(b[SD_MAX].p, 0, 8, st));
        if (tids) BM2_CUDA_OK(cudaMemcpyAsync(d_tids, tids, (size_t) nr * 8, cudaMemcpyHostToDevice, st));
        const unsigned g = (unsigned) ((nr + 255) / 256), g1 = (unsigned) ((nr + 256) / 256);
        BM2_CUDA_OK(cudaEventRecord(ctx->sort_ev[0], st));
        sort_key_kernel<<<g, 256, 0, st>>>((const uint8_t *) b[SD_IN].p, (const int64_t *) b[SD_STARTS].p, nr, (bm2_sort_rec *) b[SD_INFO].p,
                                           (int64_t *) b[SD_LEN].p, (unsigned *) b[SD_MAX].p, d_tids,
                                           mark ? (const uint64_t *) ctx->dup_bits.p : nullptr, ctx->dup_n_bits);
        BM2_CUDA_OK(cudaGetLastError());
        if (by_name) {                                          // the entries in the key buffer, the ordinals in the value buffer
            qname_key_kernel<<<g, 256, 0, st>>>((const uint8_t *) b[SD_IN].p, (const int64_t *) b[SD_STARTS].p, nr, (uint64_t *) b[SD_KEYS0].p,
                                                (uint32_t *) b[SD_VALS0].p);
            BM2_CUDA_OK(cudaGetLastError());
        }
        BM2_CUDA_OK(cudaEventRecord(ctx->sort_ev[1], st));
        size_t tb = b[SD_TEMP].cap;
        if (by_name) {
            BM2_CUDA_OK(cub::DeviceMergeSort::SortKeys(b[SD_TEMP].p, tb, (uint32_t *) b[SD_VALS0].p, nr,
                                                       QnameLess{(const uint8_t *) b[SD_IN].p, (const uint64_t *) b[SD_KEYS0].p}, st));
        } else {
            unsigned mx[2] = { 0, 0 };
            BM2_CUDA_OK(cudaMemcpyAsync(mx, b[SD_MAX].p, 8, cudaMemcpyDeviceToHost, st));
            BM2_CUDA_OK(cudaStreamSynchronize(st));
            const int pos_bits = bits_of(mx[1]), end_bit = bm2_max(1, bits_of(mx[0]) + pos_bits + 1);   // ranks 0..mx[0] (mx[0]: refID -1)
            sort_pack_kernel<<<g, 256, 0, st>>>((const bm2_sort_rec *) b[SD_INFO].p, nr, mx[0], pos_bits, (uint64_t *) b[SD_KEYS0].p,
                                                (uint32_t *) b[SD_VALS0].p);
            BM2_CUDA_OK(cudaGetLastError());
            cub::DoubleBuffer<uint64_t> kb((uint64_t *) b[SD_KEYS0].p, (uint64_t *) b[SD_KEYS1].p);
            cub::DoubleBuffer<uint32_t> vb((uint32_t *) b[SD_VALS0].p, (uint32_t *) b[SD_VALS1].p);
            BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(b[SD_TEMP].p, tb, kb, vb, (int) nr, 0, end_bit, st));
            ord = vb.Current();
        }
        BM2_CUDA_OK(cudaEventRecord(ctx->sort_ev[2], st));
        sort_permute_kernel<<<g1, 256, 0, st>>>(ord, nr, (const int64_t *) b[SD_LEN].p, (const bm2_sort_rec *) b[SD_INFO].p, (int64_t *) b[SD_LENS].p,
                                                (bm2_sort_rec *) b[SD_SINFO].p, d_tids, d_stids);
        BM2_CUDA_OK(cudaGetLastError());
        tb = b[SD_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceScan::ExclusiveSum(b[SD_TEMP].p, tb, (const int64_t *) b[SD_LENS].p, (int64_t *) b[SD_OFFS].p, (int) nr + 1, st));
        sort_gather_kernel<<<(unsigned) ((nr * 32 + 255) / 256), 256, 0, st>>>((const uint8_t *) b[SD_IN].p, (const int64_t *) b[SD_STARTS].p, ord,
                                                                               (const int64_t *) b[SD_OFFS].p, (const int64_t *) b[SD_LENS].p, nr,
                                                                               carry_len, (uint8_t *) b[SD_OUT].p,
                                                                               mark ? (const bm2_sort_rec *) b[SD_SINFO].p : nullptr);
        BM2_CUDA_OK(cudaGetLastError());
        BM2_CUDA_OK(cudaEventRecord(ctx->sort_ev[3], st));
        if (ctx->bqsr_armed && bqsr_count_device(ctx, (const uint8_t *) b[SD_OUT].p + carry_len, (const int64_t *) b[SD_OFFS].p, nr, st)) return 1;
        BM2_CUDA_OK(cudaMemcpyAsync(h_offs, b[SD_OFFS].p, (size_t) (nr + 1) * 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaMemcpyAsync(h_info, b[SD_SINFO].p, (size_t) nr * sizeof(bm2_sort_rec), cudaMemcpyDeviceToHost, st));
        if (tids) BM2_CUDA_OK(cudaMemcpyAsync(ctx->sort_tids.data(), d_stids, (size_t) nr * 8, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        float ms[3] = { 0, 0, 0 };
        for (int k = 0; k < 3; ++k) BM2_CUDA_OK(cudaEventElapsedTime(&ms[k], ctx->sort_ev[k], ctx->sort_ev[k + 1]));
        for (int k = 0; k < 3; ++k) ctx->sort_ms[k] = ms[k];
        if (ctx->bqsr_armed && bqsr_count_done(ctx, (const uint8_t *) b[SD_OUT].p + carry_len, h_offs, nr)) return 1;
    } else h_offs[0] = 0;
    // the members: the sorted buffer is free after the gather, so the compressed bytes are gathered into the records' input buffer
    if (bam_compress_stream(ctx, (const uint8_t *) b[SD_OUT].p, carry_len, h_offs, nr, h_offs[nr], last, h_info, &b[SD_IN], ctx->sort_carry,
                            ctx->sort_recs, out)) return 1;
    ctx->sort_ms[3] = ctx->bgzf_ms;
    return 0;
}

int bam_compress_stream(bm2_ctx *ctx, const uint8_t *d_stream, int64_t carry_len, const int64_t *offs, int64_t n_recs, int64_t total, int last,
                        bm2_sort_rec *recs, DevBuf *gather, std::vector<uint8_t> &carry_v, std::vector<bm2_sort_rec> &recs_v, bm2_sort_out *out) {
    bm2_ctx *ctx_for_error = ctx;
    std::vector<int64_t> cut;
    SortLayout L;
    bam_sort_layout(carry_len, offs, n_recs, total, last != 0, cut, L, recs);
    const uint8_t *z = nullptr; int64_t zl = 0;
    if (bgzf_compress_device(ctx, d_stream, L.starts.data(), L.n_full, &z, &zl, gather)) return 1;
    const int64_t c0 = L.starts[(size_t) L.n_full], c1 = carry_len + total;
    carry_v.resize((size_t) (c1 - c0));
    if (c1 > c0) BM2_CUDA_OK(cudaMemcpy(carry_v.data(), d_stream + c0, (size_t) (c1 - c0), cudaMemcpyDeviceToHost));
    recs_v.assign(recs, recs + n_recs);
    out->z = z; out->z_len = zl;
    out->member_size = ctx->bgzf_sizes.data(); out->n_members = L.n_full;
    out->carry = carry_v.data(); out->carry_len = c1 - c0;
    out->recs = recs_v.data(); out->n_recs = n_recs;
    return 0;
}

extern "C" int bm2_bam_sort_compress(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry,
                                     int64_t carry_len, int last, bm2_sort_out *out) {
    return sort_compress(ctx, recs, n, starts, n_recs, nullptr, carry, carry_len, last, out);
}

extern "C" int bm2_bam_sort_compress_ex(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tids,
                                        const uint8_t *carry, int64_t carry_len, int last, bm2_sort_out *out, const int64_t **tids_out) {
    if (sort_compress(ctx, recs, n, starts, n_recs, tids, carry, carry_len, last, out)) return 1;
    if (tids_out) *tids_out = tids ? ctx->sort_tids.data() : nullptr;
    return 0;
}

extern "C" int bm2_bam_qname_sort_compress(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry,
                                           int64_t carry_len, int last, bm2_sort_out *out) {
    return sort_compress(ctx, recs, n, starts, n_recs, nullptr, carry, carry_len, last, out, true);
}

extern "C" int bm2_last_sort_stats(const bm2_ctx *ctx, double ms[4]) {
    if (!ctx || !ms) return 1;
    for (int k = 0; k < 4; ++k) ms[k] = ctx->sort_ms[k];
    return 0;
}

extern "C" int bm2_bam_sort_memory(const bm2_ctx *ctx, int64_t run_bytes, int64_t *needed, int64_t *free_bytes) {
    return bm2_bam_sort_memory_ex(ctx, run_bytes, 0, needed, free_bytes);
}

extern "C" int bm2_bam_sort_memory_ex(const bm2_ctx *ctx, int64_t run_bytes, int with_tids, int64_t *needed, int64_t *free_bytes) {
    if (!ctx || run_bytes < 0 || !needed || !free_bytes) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // what the buffers of one call ask for, each rounded up by 1.25 as bm2_ctx::ensure allocates: records in (reused for the compressed
    // members), the sorted stream, the BGZF slots (one 64 KiB slot per 65280-byte block), and 120 bytes per record of keys, ordinals, lengths,
    // offsets and index data (twice for the radix sort's double buffers)
    const double r = (double) run_bytes, recs = r / kRecBytes + 1;
    const double bytes = 1.25 * (r + (r + BGZF_BLOCK) + (r / BGZF_BLOCK + 2) * BGZF_MAX_MEMBER + (with_tids ? 136 : 120) * recs) + 64.0 * (1 << 20);
    size_t fr = 0, tot = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
    *needed = (int64_t) bytes; *free_bytes = (int64_t) fr;
    return 0;
}

extern "C" int bm2_bam_qname_sort_memory(const bm2_ctx *ctx, int64_t run_bytes, int64_t *needed, int64_t *free_bytes) {
    if (bm2_bam_sort_memory(ctx, run_bytes, needed, free_bytes)) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // bm2_bam_sort_memory's buffers (the 8-byte entries in its key buffer, the 4-byte ordinals in its value buffer) plus cub's merge-sort
    // temporary storage for as many records, rounded up by 1.25 as bm2_ctx::ensure allocates
    cudaError_t e;
    const size_t t = qname_sort_temp((int64_t) ((double) run_bytes / kRecBytes) + 1, nullptr, &e);
    BM2_CUDA_OK(e);
    *needed += (int64_t) (1.25 * (double) t);
    return 0;
}

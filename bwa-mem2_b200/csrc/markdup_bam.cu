// markdup_bam.cu — the GPU half of bm2_markdup: Picard MarkDuplicates over coordinate-sorted BAM files (markdup_device.cuh's rule; the host
// half, the merge, pairing, resolve and metrics, is markdup_bam.h).
//   bm2_markdup_set      the merged header's read groups (each @RG ID and its library index) to the context, the per-library counters zeroed
//   bm2_markdup_records  one merged window: one warp per record.  Lane 0 finds the RG:Z value and the lanes compare it against 32 IDs of the
//                        shared-memory map at a time (bqsr_rg_lookup, as bqsr_apply.cu does).  Secondary / supplementary records and unmapped primaries are
//                        counted per library (one atomic per record).  A mapped primary gets its end and score from the warp's sums
//                        (dup_ref_len_part, dup_qual_part: markdup.cu's helpers) and, when it is half of a pair, its location from a ballot
//                        per 32 bytes of its QNAME (the colon finder of bm2_dup_signatures_ex).
//   bm2_markdup_pair     the halves of a window and those carried before it: a stable cub radix sort of their indices by read group, then
//                        by name hash; then one thread per run of equal (hash, read group), which joins its halves by their names byte for
//                        byte (dup_pair_run, markdup_device.cuh).  Runs are one or two halves but for hash collisions.
//   bm2_markdup_mark     one window of the second pass: one thread per record sets or clears 0x400 from the bitset of bm2_dup_set, by the
//                        record's ordinal in the merged stream, and writes its bm2_sort_rec; the stream carry + records is then compressed by
//                        bam_compress_stream (bam_sort.cu), as bm2_bqsr_apply does, so SortedWriter and BaiBuilder take the result.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "bam_sort_device.cuh"
#include "bqsr_device.cuh"
#include "markdup_device.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int64_t kMapMax = 32768;          // bytes of the read-group map (in shared memory)
constexpr int kRecBytes = 300;              // a short read's record, for bm2_markdup_memory's estimate

template <class T> __device__ __forceinline__ T warp_sum(T v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// map: n_ids int4 {offset of the ID's bytes from the map's start, length, library index, 0}, then the bytes.  cnt: per library, records with
// 0x100 / 0x800 at [2 lib] and unmapped primaries at [2 lib + 1].
__global__ void __launch_bounds__(kWarps * 32) mdb_record_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                                 const int4 *__restrict__ map, int map_bytes, int n_ids, int unknown_lib,
                                                                 bm2_markdup_rec *out, unsigned long long *cnt) {
    extern __shared__ int4 s_map[];
    for (int i = threadIdx.x; i < map_bytes / 16; i += blockDim.x) s_map[i] = map[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const uint8_t *rec = base + starts[w];
        const int32_t flag = (int32_t) bam_le16(rec + 18);
        int32_t len = 0, at = -1;
        if (lane == 0) at = bqsr_aux_rg(rec, &len);
        at = __shfl_sync(kFull, at, 0); len = __shfl_sync(kFull, len, 0);
        int rg = n_ids, lib = unknown_lib;                               // no tag: the shared read group n_ids
        if (at >= 0) {
            rg = bqsr_rg_lookup((const BqsrRgEntry *) s_map, n_ids, rec, at, len);   // -1: a value that is no @RG ID
            if (rg >= 0) lib = s_map[rg].z;
        }
        bm2_markdup_rec o{};
        o.rg = rg; o.lib = lib; o.kind = BM2_MDB_NONE;
        if (!dup_is_primary(flag)) {
            if (lane == 0) atomicAdd(cnt + 2 * lib, 1ULL);
        } else if (flag & 4) {
            if (lane == 0) atomicAdd(cnt + 2 * lib + 1, 1ULL);
            if ((flag & 1) && !(flag & 8)) o.kind = BM2_MDB_UNMAPPED_HALF;
        } else {
            o.kind = (flag & 1) && !(flag & 8) ? BM2_MDB_HALF : BM2_MDB_FRAG;
            o.score = dup_read_score(warp_sum(dup_qual_part(rec, lane, 32)));
            const DupCigar c = dup_cigar(rec);
            o.end = dup_read_end(rec, c, warp_sum(dup_ref_len_part(c, lane, 32)));
            if (o.kind == BM2_MDB_HALF) {                                // the QNAME split on ':' by a ballot per 32 bytes
                int nc = 0, c1 = -1, c2 = -1, c3 = -1;
                const uint8_t *name = rec + 36;
                const int ln = bm2_max<int>((int) rec[12] - 1, 0);
                for (int b = 0; b < ln; b += 32) {
                    const int i = b + lane;
                    for (unsigned m = __ballot_sync(kFull, i < ln && name[i] == ':'); m; m &= m - 1) { c1 = c2; c2 = c3; c3 = b + __ffs(m) - 1; ++nc; }
                }
                o.loc = dup_location_from_colons(name, ln, nc, c1, c2, c3, &o.tile, &o.x, &o.y);
            }
        }
        if (o.kind == BM2_MDB_HALF || o.kind == BM2_MDB_UNMAPPED_HALF) {
            if (lane == 0) o.hash = dup_name_hash(rec + 36, bm2_max<int>((int) rec[12] - 1, 0));
        }
        if (lane == 0) out[w] = o;
    }
}

// the pairing's sort keys: field 0 the read group, 1 the hash, of the half at each place of the current order
__global__ void mdb_pair_key_kernel(const bm2_markdup_half *__restrict__ h, const uint32_t *__restrict__ ord, int64_t n, int field, uint64_t *keys) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bm2_markdup_half &x = h[ord[i]];
    keys[i] = field == 0 ? (uint64_t) (uint32_t) x.rg : x.hash;
}

__global__ void mdb_iota_kernel(uint32_t *ord, int64_t n) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ord[i] = (uint32_t) i;
}

// one thread per sorted place that starts a run of equal (hash, read group): the run's halves joined by name
__global__ void mdb_pair_run_kernel(const bm2_markdup_half *__restrict__ h, const uint32_t *__restrict__ ord, int64_t n, const uint8_t *__restrict__ names,
                                    int32_t *partner) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    auto same = [&](int64_t a, int64_t b) { return h[ord[a]].hash == h[ord[b]].hash && h[ord[a]].rg == h[ord[b]].rg; };
    if (i > 0 && same(i, i - 1)) return;
    int64_t e = i + 1;
    while (e < n && same(e, i)) ++e;
    dup_pair_run(h, ord, i, e, names, partner);
}

// the second pass: 0x400 from bit (first + i) of bits, cleared everywhere else, and each record's index data
__global__ void mdb_mark_kernel(uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n, int64_t first, const uint64_t *__restrict__ bits,
                                int64_t n_bits, bm2_sort_rec *info) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t *r = base + starts[i];
    const int64_t o = first + i;
    const bool dup = o < n_bits && ((bits[o >> 6] >> (o & 63)) & 1);
    const uint32_t f = (bam_le16(r + 18) & ~0x400u) | (dup ? 0x400u : 0u);
    r[18] = (uint8_t) f; r[19] = (uint8_t) (f >> 8);
    info[i] = bam_sort_rec(r);
}

enum { MB_MAP, MB_STREAM, MB_STARTS, MB_OUT, MB_INFO, MB_CNT,
       MB_HALF, MB_NAMES, MB_KEY0, MB_KEY1, MB_ORD0, MB_ORD1, MB_PART, MB_TEMP,   // bm2_markdup_pair
       MB_END };
enum { MH_INFO, MH_END };
static_assert(MB_END == std::extent<decltype(bm2_ctx::mdb_d)>::value, "bm2_ctx::mdb_d: one buffer per slot");
static_assert(MH_END == std::extent<decltype(bm2_ctx::mdb_h)>::value, "bm2_ctx::mdb_h: one buffer per slot");
static_assert(sizeof(bm2_markdup_rec) == 48 && sizeof(bm2_markdup_half) == 24, "bm2_markdup_rec, bm2_markdup_half: no padding, as the Python bindings read them");

}  // namespace

// the records at starts are whole, each where the one before ends, the last ending at n
int bam_check_records(bm2_ctx *ctx, const char *fn, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs) {
    for (int64_t i = 0, at = 0; i <= n_recs; ++i) {
        if (i == n_recs) { if (at != n) { bm2_set_error(ctx, std::string(fn) + ": the records do not end where the buffer ends"); return 1; } break; }
        const int64_t s = starts[i];
        if (s != at || s + 36 > n) { bm2_set_error(ctx, std::string(fn) + ": record " + std::to_string(i) + " does not start where the one before ends"); return 1; }
        const BamFixed f = bam_fixed(recs + s);
        const int32_t l_seq = bam_le32(recs + s + 20);
        if (f.block_size < 32 || s + 4 + (int64_t) f.block_size > n || l_seq < 0 || f.l_read_name < 1 ||
            32 + (int64_t) f.l_read_name + 4 * (int64_t) f.n_cigar + (l_seq + 1) / 2 + (int64_t) l_seq > (int64_t) f.block_size) {
            bm2_set_error(ctx, std::string(fn) + ": record " + std::to_string(i) + " is malformed");
            return 1;
        }
        at = s + 4 + f.block_size;
    }
    return 0;
}

extern "C" int bm2_markdup_set(bm2_ctx *ctx, int32_t n_ids, const char *const *ids, const int32_t *libs, int32_t n_lib, int32_t unknown_lib) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n_ids < 0 || (n_ids && (!ids || !libs)) || n_lib < 1 || unknown_lib < 0 || unknown_lib >= n_lib) {
        if (ctx) bm2_set_error(ctx, "bm2_markdup_set: bad arguments");
        return 1;
    }
    std::vector<int4> map((size_t) n_ids);
    std::string bytes;
    for (int32_t i = 0; i < n_ids; ++i) {
        if (!ids[i] || libs[i] < 0 || libs[i] >= n_lib) { bm2_set_error(ctx, "bm2_markdup_set: a bad read-group entry"); return 1; }
        map[(size_t) i] = int4{(int) bytes.size(), (int) strlen(ids[i]), libs[i], 0};
        bytes += ids[i];
    }
    const int64_t total = ((16 * (int64_t) n_ids + (int64_t) bytes.size()) + 15) / 16 * 16;
    if (total > kMapMax) {
        bm2_set_error(ctx, "bm2_markdup_set: the header's read-group IDs take " + std::to_string(total) + " bytes, more than " + std::to_string(kMapMax));
        return 1;
    }
    for (int4 &e : map) e.x += 16 * n_ids;
    std::vector<uint8_t> blob((size_t) total + 16, 0);
    if (n_ids) memcpy(blob.data(), map.data(), map.size() * 16);
    memcpy(blob.data() + 16 * n_ids, bytes.data(), bytes.size());
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->mdb_d;
    if (ctx->ensure(b[MB_MAP], blob.size()) || ctx->ensure(b[MB_CNT], (size_t) (2 * n_lib) * 8)) return 1;
    BM2_CUDA_OK(cudaMemcpy(b[MB_MAP].p, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    BM2_CUDA_OK(cudaMemset(b[MB_CNT].p, 0, (size_t) (2 * n_lib) * 8));
    ctx->mdb_map_bytes = total; ctx->mdb_n_ids = n_ids; ctx->mdb_n_lib = n_lib; ctx->mdb_unknown_lib = unknown_lib;
    ctx->mdb_records_ms = 0; ctx->mdb_pair_ms = 0; ctx->mdb_mark_ms = 0; ctx->mdb_bgzf_ms = 0;
    ctx->mdb_set = true;
    return 0;
}

extern "C" int bm2_markdup_records(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const bm2_markdup_rec **out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts)) {
        if (ctx) bm2_set_error(ctx, "bm2_markdup_records: bad arguments");
        return 1;
    }
    if (!ctx->mdb_set) { bm2_set_error(ctx, "bm2_markdup_records: no read groups on this context (bm2_markdup_set)"); return 1; }
    if (bam_check_records(ctx, "bm2_markdup_records", recs, n, starts, n_recs)) return 1;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->mdb_d;
    if (ctx->ensure(b[MB_STREAM], (size_t) n + 16) || ctx->ensure(b[MB_STARTS], (size_t) n_recs * 8 + 8) ||
        ctx->ensure(b[MB_OUT], (size_t) n_recs * sizeof(bm2_markdup_rec) + 8)) return 1;
    for (cudaEvent_t &ev : ctx->mdb_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    ctx->mdb_recs.resize((size_t) n_recs);
    *out = ctx->mdb_recs.data();
    if (!n_recs) return 0;
    BM2_CUDA_OK(cudaMemcpyAsync(b[MB_STREAM].p, recs, (size_t) n, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(b[MB_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
    const int smem = (int) ctx->mdb_map_bytes;
    const int64_t g = bm2_min<int64_t>((n_recs + kWarps - 1) / kWarps, (int64_t) ctx->n_sm * 8);
    BM2_CUDA_OK(cudaEventRecord(ctx->mdb_ev[0], st));
    mdb_record_kernel<<<(unsigned) g, kWarps * 32, smem, st>>>((const uint8_t *) b[MB_STREAM].p, (const int64_t *) b[MB_STARTS].p, n_recs,
                                                               (const int4 *) b[MB_MAP].p, smem, ctx->mdb_n_ids, ctx->mdb_unknown_lib,
                                                               (bm2_markdup_rec *) b[MB_OUT].p, (unsigned long long *) b[MB_CNT].p);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->mdb_ev[1], st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->mdb_recs.data(), b[MB_OUT].p, (size_t) n_recs * sizeof(bm2_markdup_rec), cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->mdb_ev[0], ctx->mdb_ev[1]));
    ctx->mdb_records_ms += ms;
    return 0;
}

extern "C" int bm2_markdup_pair(bm2_ctx *ctx, const bm2_markdup_half *halves, int64_t n, const uint8_t *names, int64_t names_len, const int32_t **partner) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !partner || n < 0 || (n && !halves) || names_len < 0 || (names_len && !names)) {
        if (ctx) bm2_set_error(ctx, "bm2_markdup_pair: bad arguments");
        return 1;
    }
    if (n >= ((int64_t) 1 << 31)) { bm2_set_error(ctx, "bm2_markdup_pair: 2^31 halves or more in one call"); return 1; }
    for (int64_t i = 0; i < n; ++i)
        if (halves[i].name_len < 0 || halves[i].name_off < 0 || halves[i].name_off + halves[i].name_len > names_len) {
            bm2_set_error(ctx, "bm2_markdup_pair: half " + std::to_string(i) + "'s name lies outside the names");
            return 1;
        }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->mdb_d;
    const int ni = (int) bm2_max<int64_t>(n, 1);
    size_t temp = 0;
    {
        cub::DoubleBuffer<uint64_t> k((uint64_t *) nullptr, nullptr); cub::DoubleBuffer<uint32_t> v((uint32_t *) nullptr, nullptr);
        BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, temp, k, v, ni, 0, 64, st));
    }
    if (ctx->ensure(b[MB_HALF], (size_t) n * sizeof(bm2_markdup_half) + 8) || ctx->ensure(b[MB_NAMES], (size_t) names_len + 8) ||
        ctx->ensure(b[MB_KEY0], (size_t) n * 8 + 8) || ctx->ensure(b[MB_KEY1], (size_t) n * 8 + 8) || ctx->ensure(b[MB_ORD0], (size_t) n * 4 + 8) ||
        ctx->ensure(b[MB_ORD1], (size_t) n * 4 + 8) || ctx->ensure(b[MB_PART], (size_t) n * 4 + 8) || ctx->ensure(b[MB_TEMP], temp + 16)) return 1;
    for (cudaEvent_t &ev : ctx->mdb_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    ctx->mdb_partner.resize((size_t) n);
    *partner = ctx->mdb_partner.data();
    if (!n) return 0;
    const unsigned g = (unsigned) ((n + 255) / 256);
    const bm2_markdup_half *H = (const bm2_markdup_half *) b[MB_HALF].p;
    BM2_CUDA_OK(cudaMemcpyAsync(b[MB_HALF].p, halves, (size_t) n * sizeof(bm2_markdup_half), cudaMemcpyHostToDevice, st));
    if (names_len) BM2_CUDA_OK(cudaMemcpyAsync(b[MB_NAMES].p, names, (size_t) names_len, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaEventRecord(ctx->mdb_ev[0], st));
    mdb_iota_kernel<<<g, 256, 0, st>>>((uint32_t *) b[MB_ORD0].p, n);
    BM2_CUDA_OK(cudaGetLastError());
    cub::DoubleBuffer<uint64_t> kb((uint64_t *) b[MB_KEY0].p, (uint64_t *) b[MB_KEY1].p);
    cub::DoubleBuffer<uint32_t> vb((uint32_t *) b[MB_ORD0].p, (uint32_t *) b[MB_ORD1].p);
    for (int f = 0; f < 2; ++f) {                              // read group, then hash: each pass stable, so ties keep the index order
        mdb_pair_key_kernel<<<g, 256, 0, st>>>(H, vb.Current(), n, f, kb.Current());
        BM2_CUDA_OK(cudaGetLastError());
        size_t tb = b[MB_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(b[MB_TEMP].p, tb, kb, vb, (int) n, 0, f ? 64 : 32, st));
    }
    mdb_pair_run_kernel<<<g, 256, 0, st>>>(H, vb.Current(), n, (const uint8_t *) b[MB_NAMES].p, (int32_t *) b[MB_PART].p);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->mdb_ev[1], st));
    BM2_CUDA_OK(cudaMemcpyAsync(ctx->mdb_partner.data(), b[MB_PART].p, (size_t) n * 4, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->mdb_ev[0], ctx->mdb_ev[1]));
    ctx->mdb_pair_ms += ms;
    return 0;
}

extern "C" int bm2_markdup_counts(bm2_ctx *ctx, int64_t *counts) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !counts) { if (ctx) bm2_set_error(ctx, "bm2_markdup_counts: bad arguments"); return 1; }
    if (!ctx->mdb_set) { bm2_set_error(ctx, "bm2_markdup_counts: no read groups on this context (bm2_markdup_set)"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    std::vector<unsigned long long> c((size_t) 2 * ctx->mdb_n_lib);
    BM2_CUDA_OK(cudaMemcpy(c.data(), ctx->mdb_d[MB_CNT].p, c.size() * 8, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < c.size(); ++i) counts[i] = (int64_t) c[i];
    return 0;
}

extern "C" int bm2_markdup_mark(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, int64_t first, const uint8_t *carry,
                                int64_t carry_len, int last, bm2_sort_out *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts) || first < 0 || carry_len < 0 || carry_len >= BGZF_BLOCK ||
        (carry_len && !carry)) {
        if (ctx) bm2_set_error(ctx, "bm2_markdup_mark: bad arguments");
        return 1;
    }
    if (!ctx->mdb_set) { bm2_set_error(ctx, "bm2_markdup_mark: no read groups on this context (bm2_markdup_set)"); return 1; }
    if (bam_check_records(ctx, "bm2_markdup_mark", recs, n, starts, n_recs)) return 1;
    memset(out, 0, sizeof *out);
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->mdb_d;
    if (ctx->ensure(b[MB_STREAM], (size_t) (carry_len + n) + 16) || ctx->ensure(b[MB_STARTS], (size_t) n_recs * 8 + 8) ||
        ctx->ensure(b[MB_INFO], (size_t) n_recs * sizeof(bm2_sort_rec) + 8) ||
        ctx->ensure_host(ctx->mdb_h[MH_INFO], (size_t) n_recs * sizeof(bm2_sort_rec) + 16)) return 1;
    for (cudaEvent_t &ev : ctx->mdb_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    uint8_t *d_stream = (uint8_t *) b[MB_STREAM].p;
    bm2_sort_rec *h_info = (bm2_sort_rec *) ctx->mdb_h[MH_INFO].p;
    if (carry_len) BM2_CUDA_OK(cudaMemcpy(d_stream, carry, (size_t) carry_len, cudaMemcpyHostToDevice));   // carry may be this context's last carry
    if (n_recs) {
        BM2_CUDA_OK(cudaMemcpyAsync(d_stream + carry_len, recs, (size_t) n, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[MB_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaEventRecord(ctx->mdb_ev[0], st));
        mdb_mark_kernel<<<(unsigned) ((n_recs + 255) / 256), 256, 0, st>>>(d_stream + carry_len, (const int64_t *) b[MB_STARTS].p, n_recs, first,
                                                                           (const uint64_t *) ctx->dup_bits.p, ctx->dup_n_bits,
                                                                           (bm2_sort_rec *) b[MB_INFO].p);
        BM2_CUDA_OK(cudaGetLastError());
        BM2_CUDA_OK(cudaEventRecord(ctx->mdb_ev[1], st));
        BM2_CUDA_OK(cudaMemcpyAsync(h_info, b[MB_INFO].p, (size_t) n_recs * sizeof(bm2_sort_rec), cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        float ms = 0;
        BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->mdb_ev[0], ctx->mdb_ev[1]));
        ctx->mdb_mark_ms += ms;
    }
    if (bam_compress_stream(ctx, d_stream, carry_len, starts, n_recs, n, last, h_info, nullptr, ctx->mdb_carry, ctx->mdb_srecs, out)) return 1;
    ctx->mdb_bgzf_ms += ctx->bgzf_ms;
    return 0;
}

extern "C" int bm2_last_markdup_stats(const bm2_ctx *ctx, bm2_markdup_stats_t *out) {
    if (!ctx || !out) return 1;
    out->records_ms = ctx->mdb_records_ms; out->pair_ms = ctx->mdb_pair_ms; out->mark_ms = ctx->mdb_mark_ms; out->bgzf_ms = ctx->mdb_bgzf_ms;
    return 0;
}

extern "C" int bm2_markdup_memory(const bm2_ctx *ctx, int64_t window_bytes, int64_t *needed, int64_t *free_bytes) {
    if (!ctx || window_bytes < 0 || !needed || !free_bytes) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // each rounded up by 1.25 as bm2_ctx::ensure allocates: the stream (carry + window), the BGZF slots (one 64 KiB slot per 65280-byte block)
    // and the gathered members, per record 8 bytes of starts, 16 of index data and one bm2_markdup_rec, and for the pairing (every record a
    // half at most) 24 bytes of half, 16 of sort keys, 8 of order, 4 of partner and about 60 of name and sort scratch; the read-group map.
    // The duplicate bitset (bm2_dup_set) and bm2_dup_resolve_ex's buffers come on top.
    const double w = (double) window_bytes, slots = (w / BGZF_BLOCK + 2) * BGZF_MAX_MEMBER;
    const double bytes = 1.25 * ((w + BGZF_BLOCK) + 2 * slots + (24.0 + sizeof(bm2_markdup_rec) + 112.0) * (w / kRecBytes + 1) + kMapMax) + 64.0 * (1 << 20);
    size_t fr = 0, tot = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
    *needed = (int64_t) bytes; *free_bytes = (int64_t) fr;
    return 0;
}

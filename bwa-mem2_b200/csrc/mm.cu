// mm.cu — the alignment summary and insert size counts of bm2_multiplemetrics on the GPU (mm_device.cuh's rule).
//   bm2_mm_set     the packed reference (2 bits per base), a hole bitset (1 bit per base, built here from the sorted hole ranges) and the
//                  ranges with their letters for a binary search at hole loci; zeroes the counters
//   bm2_mm_add     one window of records in any order, in two kernels (below); no record is carried between windows
//   bm2_mm_finish  copies back the counters, the histograms up to their largest keys, and sorts the large insert sizes on the host
//   check   one warp per record: the lanes sum the CIGAR (aligned, reference, query lengths, clipped bases, indel operations), lane 0
//           classifies the record (mm_classify) and writes its MmInfo; a read error takes the first record by index (atomicMin).  Nothing is
//           counted before the host has seen that no record of the window is an error.
//   count   one warp per record, grid-stride: the lanes take consecutive bases for the no-calls by cycle (global atomics: they are rare) and,
//           for an aligned record, consecutive aligned bases (nibble, quality, 2-bit reference code, hole bit) for the mismatches and Q20
//           bases, reduced over the warp.  Lane 0 adds the record's counters to per-block shared counters and its read length and mismatch
//           count to per-block shared bins below kHot (global atomics above), and its insert size to dense per-orientation bins below 2^20
//           or to an append list.  Each block flushes once with 64-bit atomics and raises the running maxima (atomicMax).
// Only integer atomics: the sums commute, so the counts do not depend on the windows or the order of the records.
//
// GC bias (bm2_mm_gc_set, bm2_mm_gc_finish; the rule is mm_device.cuh's, the text mm_gcbias.h's):
//   scan    the reference windows, once per bm2_mm_gc_set: each block takes tiles of kScanTile window starts; one thread per 32-locus word
//           builds the tile's GC and N bitsets (kScanTile + W loci) from the packed bases and the hole bitset, the hole letters found by a
//           binary search of the holes where a word has a hole bit (mm_gc_word), and a block scan of their popcounts gives prefix counts,
//           so a window's counts are two prefix lookups and two masked popcounts each.  The tile walks the contigs it overlaps, clipped to
//           their counted starts; bins go to a per-block shared histogram (one atomic per __match_any_sync group), flushed once.
//   add     the check and count kernels instantiated with GC on: the check applies the aligned checks to every placed record and writes its
//           MmGc (window locus, I and D lengths); the count warp classifies the 100 letters of the window with ballots and popcounts and
//           adds the read start, bases and errors to per-block shared bins.  The instantiations with GC off are the kernels above unchanged.
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "mm_metrics.h"
#include <algorithm>
#include <cub/block/block_scan.cuh>
#include <vector>

namespace {

constexpr int kWarps = 8;
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kRecBytes = 300;              // a short read's record, for bm2_mm_memory's estimate
constexpr int kHot = 256;                   // read lengths and mismatch counts below this are binned per block in shared memory
constexpr size_t kLenBins = (size_t) MM_MAX_LSEQ + 1, kInsBins = (size_t) MM_DENSE_INSERT;
constexpr int kScanThreads = 256, kScanTile = 32 * (kScanThreads - 4);   // a tile's words (one per thread) cover its starts and W - 1 more loci
// the GC bias counters: read starts, bases and errors per bin, then TOTAL_CLUSTERS and ALIGNED_READS
enum { GC_READS = 0, GC_BASES = MM_GC_BINS, GC_ERRORS = 2 * MM_GC_BINS, GC_CLUSTERS = 3 * MM_GC_BINS, GC_ALIGNED, GC_NCOUNT };

__constant__ char c_kmers[MM_N_ADAPTER_KMERS][MM_ADAPTER_LEN];

// the scalars of the device: the first error, the count of large insert sizes, the longest read, the largest dense insert size
enum { SC_ERR, SC_BIG_N, SC_MAX_LEN, SC_MAX_INS, SC_END };

__global__ void mm_holes_kernel(uint32_t *bits, int64_t n_words, const int64_t *ranges, int64_t n) {
    for (int64_t w = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t) gridDim.x * blockDim.x)
        bits[w] = wgs_range_word(ranges, n, w);
}

template <bool GC>
__global__ void __launch_bounds__(kWarps * 32) mm_check_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                               const int64_t *__restrict__ off, const int32_t *__restrict__ len, int32_t n_contigs,
                                                               MmInfo *info, unsigned long long *sc, int64_t first, MmGc *gc) {
    const int lane = threadIdx.x & 31;
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const uint8_t *r = base + starts[w];
        const DupCigar c = dup_cigar(r);
        const bool inside = wgs_cigar_inside(r, c);
        int64_t s[3] = {0, 0, 0}, t[3] = {0, 0, 0};
        if (inside) { wgs_cigar_part(c, lane, 32, s); mm_clip_part(c, lane, 32, t); }
        for (int k = 0; k < 3; ++k)
            for (int o = 16; o; o >>= 1) { s[k] += __shfl_xor_sync(kFull, s[k], o); t[k] += __shfl_xor_sync(kFull, t[k], o); }
        int64_t idlen = 0;
        if constexpr (GC) {
            if (inside) idlen = mm_gc_idlen_part(c, lane, 32);
            for (int o = 16; o; o >>= 1) idlen += __shfl_xor_sync(kFull, idlen, o);
        }
        if (lane == 0) {
            MmInfo in;
            mm_classify(r, s, t, inside, off, len, n_contigs, c_kmers, in, GC);
            info[w] = in;
            if (in.err) atomicMin(&sc[SC_ERR], (unsigned long long) (first + w) << 4 | (unsigned) in.err);
            if constexpr (GC) gc[w] = MmGc{(in.bits & MMB_PLACED) ? mm_gc_window(r, s[1], off, len) : -1, idlen};
        }
    }
}

template <bool GC>
__global__ void __launch_bounds__(kWarps * 32) mm_count_kernel(const uint8_t *__restrict__ base, const int64_t *__restrict__ starts, int64_t n,
                                                               const MmInfo *__restrict__ info, const uint8_t *__restrict__ pac,
                                                               const uint32_t *__restrict__ hole_bits, const int64_t *__restrict__ holes,
                                                               const char *__restrict__ hole_char, int64_t n_holes, unsigned long long *cnt,
                                                               unsigned long long *len_hist, unsigned long long *mism_hist,
                                                               unsigned long long *nocall, unsigned long long *ins, uint64_t *big,
                                                               unsigned long long *sc, const MmGc *__restrict__ gc, unsigned long long *gc_cnt) {
    __shared__ unsigned long long s_cnt[MM_NCAT * MM_NCOUNT];
    __shared__ unsigned long long s_gc[GC ? GC_NCOUNT : 1];
    if constexpr (GC) for (int k = threadIdx.x; k < GC_NCOUNT; k += blockDim.x) s_gc[k] = 0;
    __shared__ uint32_t s_len[MM_NCAT][kHot], s_mis[MM_NCAT][kHot];
    __shared__ uint32_t s_max_len, s_max_ins;
    for (int k = threadIdx.x; k < MM_NCAT * MM_NCOUNT; k += blockDim.x) s_cnt[k] = 0;
    for (int k = threadIdx.x; k < MM_NCAT * kHot; k += blockDim.x) { s_len[k / kHot][k % kHot] = 0; s_mis[k / kHot][k % kHot] = 0; }
    if (threadIdx.x == 0) { s_max_len = 0; s_max_ins = 0; }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int64_t w = (int64_t) blockIdx.x * kWarps + (threadIdx.x >> 5); w < n; w += (int64_t) gridDim.x * kWarps) {
        const MmInfo in = info[w];
        if (!(in.bits & MMB_COUNTED)) continue;
        const uint8_t *r = base + starts[w];
        const WgsSeq sq = wgs_seq(r);
        const size_t row = (size_t) in.cat * kLenBins;
        for (int32_t k = lane; k < in.l_seq; k += 32)
            if (mm_nibble(sq.seq, k) == 15)
                atomicAdd(&nocall[row + (size_t) ((in.bits & MMB_REV) ? in.l_seq - 1 - k : k)], 1ull);
        uint32_t mism = 0, q20 = 0;
        if (in.bits & (GC ? MMB_PLACED : MMB_ALIGNED)) {
            const DupCigar c = dup_cigar(r);
            const bool noqual = in.bits & MMB_NOQUAL;
            int64_t k = 0, g = in.g0;
            for (int64_t i = 0; i < c.n; ++i) {
                const uint32_t op = dup_op(c, i), ln = op >> 4;
                if (wgs_aligned_op(op))
                    for (uint32_t b = lane; b < ln; b += 32) mm_base(sq, noqual, k + b, g + b, pac, hole_bits, holes, hole_char, n_holes, mism, q20);
                if (dup_consumes_ref(op)) g += ln;
                if (wgs_query_op(op)) k += ln;
            }
            mism = __reduce_add_sync(kFull, mism);
            q20 = __reduce_add_sync(kFull, q20);
        }
        if constexpr (GC) {
            const MmGc gi = gc[w];
            int bin = -1;
            if (gi.gw >= 0) {                                            // the window's letters, 32 at a time
                int n_gc = 0, n_n = 0;
                for (int j = 0; j < MM_GC_W; j += 32) {
                    const int cls = j + lane < MM_GC_W ? mm_gc_class(mm_ref_letter(pac, hole_bits, holes, hole_char, n_holes, gi.gw + j + lane)) : 0;
                    n_gc += __popc(__ballot_sync(kFull, cls == 1));
                    n_n += __popc(__ballot_sync(kFull, cls == 2));
                }
                bin = mm_gc_bin(n_gc, n_n);
            }
            if (lane == 0) {
                if (in.cat != MM_SECOND) atomicAdd(&s_gc[GC_CLUSTERS], 1ull);
                if (in.bits & MMB_PLACED) atomicAdd(&s_gc[GC_ALIGNED], 1ull);
                if (bin >= 0) {
                    atomicAdd(&s_gc[GC_READS + bin], 1ull);
                    atomicAdd(&s_gc[GC_BASES + bin], (unsigned long long) in.l_seq);
                    atomicAdd(&s_gc[GC_ERRORS + bin], (unsigned long long) mism + (unsigned long long) gi.idlen);
                }
            }
        }
        if (lane == 0) {
            int64_t v[MM_NCOUNT];
            mm_record_counts(in, mism, q20, v);
            for (int k = 0; k < MM_NCOUNT; ++k) if (v[k]) atomicAdd(&s_cnt[in.cat * MM_NCOUNT + k], (unsigned long long) v[k]);
            if (in.l_seq < kHot) atomicAdd(&s_len[in.cat][in.l_seq], 1u);
            else atomicAdd(&len_hist[row + (size_t) in.l_seq], 1ull);
            atomicMax(&s_max_len, (uint32_t) in.l_seq);
            if (in.bits & MMB_HQ) {
                if (mism < (uint32_t) kHot) atomicAdd(&s_mis[in.cat][mism], 1u);
                else atomicAdd(&mism_hist[row + mism], 1ull);
            }
            if (in.bits & MMB_INSERT) {
                if (in.insert < MM_DENSE_INSERT) {
                    atomicAdd(&ins[(size_t) in.orient * kInsBins + (size_t) in.insert], 1ull);
                    atomicMax(&s_max_ins, (uint32_t) in.insert);
                } else {
                    const unsigned long long at = atomicAdd(&sc[SC_BIG_N], 1ull);
                    big[at] = (uint64_t) in.orient << 32 | (uint64_t) in.insert;
                }
            }
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < MM_NCAT * MM_NCOUNT; k += blockDim.x) if (s_cnt[k]) atomicAdd(&cnt[k], s_cnt[k]);
    for (int k = threadIdx.x; k < MM_NCAT * kHot; k += blockDim.x) {
        const int c = k / kHot, b = k % kHot;
        if (s_len[c][b]) atomicAdd(&len_hist[(size_t) c * kLenBins + b], (unsigned long long) s_len[c][b]);
        if (s_mis[c][b]) atomicAdd(&mism_hist[(size_t) c * kLenBins + b], (unsigned long long) s_mis[c][b]);
    }
    if (threadIdx.x == 0) {
        if (s_max_len) atomicMax(&sc[SC_MAX_LEN], (unsigned long long) s_max_len);
        if (s_max_ins) atomicMax(&sc[SC_MAX_INS], (unsigned long long) s_max_ins);
    }
    if constexpr (GC) for (int k = threadIdx.x; k < GC_NCOUNT; k += blockDim.x) if (s_gc[k]) atomicAdd(&gc_cnt[k], s_gc[k]);
}

// the reference windows by GC bin (mm_device.cuh's rule): tiles of kScanTile window starts, grid-stride; contigs sorted and disjoint
__global__ void __launch_bounds__(kScanThreads) mm_gc_scan_kernel(const uint8_t *__restrict__ pac, const uint32_t *__restrict__ hole_bits,
                                                                  const int64_t *__restrict__ holes, const char *__restrict__ hole_char, int64_t n_holes,
                                                                  int64_t l_pac, const int64_t *__restrict__ off, const int32_t *__restrict__ len,
                                                                  int32_t n_contigs, int64_t n_tiles, unsigned long long *windows) {
    using Scan = cub::BlockScan<uint32_t, kScanThreads>;
    __shared__ typename Scan::TempStorage s_scan;
    __shared__ uint32_t s_gcw[kScanThreads], s_nw[kScanThreads], s_pre[kScanThreads], s_hist[MM_GC_BINS];
    for (int k = threadIdx.x; k < MM_GC_BINS; k += blockDim.x) s_hist[k] = 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int64_t b = t * kScanTile;                                 // a multiple of 32: word k of the tile is locus word b / 32 + k
        uint32_t gcm, nm;
        mm_gc_word(pac, hole_bits, holes, hole_char, n_holes, l_pac, b / 32 + threadIdx.x, gcm, nm);
        uint32_t pre;
        __syncthreads();                                                 // the last tile's readers are done
        Scan(s_scan).ExclusiveSum((uint32_t) __popc(gcm) << 16 | (uint32_t) __popc(nm), pre);   // at most 8192 each
        s_gcw[threadIdx.x] = gcm; s_nw[threadIdx.x] = nm; s_pre[threadIdx.x] = pre;
        __syncthreads();
        // GC letters and Ns before tile locus x: packed (GC << 16 | N)
        auto before = [&](int x) {
            const uint32_t m = (1u << (x & 31)) - 1;
            return s_pre[x >> 5] + ((uint32_t) __popc(s_gcw[x >> 5] & m) << 16) + (uint32_t) __popc(s_nw[x >> 5] & m);
        };
        int32_t lo = 0, hi = n_contigs;                                  // the first contig ending after b
        while (lo < hi) { const int32_t m = (lo + hi) / 2; if (off[m] + len[m] <= b) lo = m + 1; else hi = m; }
        const int64_t e = bm2_min<int64_t>(b + kScanTile, l_pac);
        for (int32_t c = lo; c < n_contigs && off[c] < e; ++c) {
            const int64_t g0 = bm2_max<int64_t>(b, off[c] + 1), g1 = bm2_min<int64_t>(e, off[c] + len[c] - MM_GC_W);
            for (int64_t k = g0 + warp * 32; k < g1; k += kScanThreads) {   // warp-uniform trips
                int bin = -1;
                if (k + lane < g1) {
                    const int x = (int) (k + lane - b);
                    const uint32_t d = before(x + MM_GC_W) - before(x);
                    bin = mm_gc_bin((int) (d >> 16), (int) (d & 0xFFFF));
                }
                const unsigned peers = __match_any_sync(kFull, bin);
                if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_hist[bin], (uint32_t) __popc(peers));
            }
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < MM_GC_BINS; k += blockDim.x) if (s_hist[k]) atomicAdd(&windows[k], (unsigned long long) s_hist[k]);
}

enum { MD_PAC, MD_HOLEBITS, MD_HOLES, MD_HOLECHAR, MD_OFF, MD_LEN, MD_CNT, MD_LENH, MD_MISH, MD_NOCALL, MD_INS, MD_SC, MD_BIG, MD_RECS,
       MD_STARTS, MD_INFO, MD_GC_WIN, MD_GC_CNT, MD_GC_INFO, MD_END };
static_assert(MD_END == std::extent<decltype(bm2_ctx::mm_d)>::value, "bm2_ctx::mm_d: one buffer per slot");
static_assert(MM_GC_BINS == BM2_MM_GC_BINS, "bm2_mm_gc_result_t's bins");

const char *const kErrText[3] = {"has l_seq 0 or above 1048576", "does not lie inside a contig of the reference",
                                 "has a CIGAR that does not match its record"};

size_t pac_bytes(int64_t l_pac) { return (size_t) ((l_pac + 3) / 4); }
size_t bits_bytes(int64_t l_pac) { return (size_t) ((l_pac + 127) / 128) * 16; }
// the per-category length arrays (three of them), the dense insert bins and the counters
size_t hist_bytes() { return 3 * (size_t) MM_NCAT * kLenBins * 8 + (size_t) MM_NORIENT * kInsBins * 8 + (size_t) MM_NCAT * MM_NCOUNT * 8; }

// exactly `bytes` (the reference is too large for bm2_ctx::ensure's 25% headroom)
int ensure_exact(bm2_ctx *ctx, DevBuf &b, size_t bytes) {
    bm2_ctx *ctx_for_error = ctx;
    if (b.cap >= bytes) return 0;
    if (b.p) BM2_CUDA_OK(cudaFree(b.p));
    b.p = nullptr; b.cap = 0;
    BM2_CUDA_OK(cudaMalloc(&b.p, bytes));
    b.cap = bytes;
    return 0;
}

}  // namespace

extern "C" int bm2_mm_set(bm2_ctx *ctx, const int64_t *contig_off, const int32_t *contig_len, int32_t n_contigs, int64_t l_pac, const uint8_t *pac,
                          const int64_t *holes, const char *hole_char, int64_t n_holes) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n_contigs < 0 || (n_contigs && (!contig_off || !contig_len)) || l_pac < 1 || !pac || n_holes < 0 || (n_holes && (!holes || !hole_char))) {
        if (ctx) bm2_set_error(ctx, "bm2_mm_set: bad arguments");
        return 1;
    }
    for (int32_t k = 0; k < n_contigs; ++k)
        if (contig_off[k] < 0 || contig_len[k] < 0 || contig_off[k] + contig_len[k] > l_pac) {
            bm2_set_error(ctx, "bm2_mm_set: contig " + std::to_string(k) + " does not lie inside the reference"); return 1;
        }
    for (int64_t h = 0; h < n_holes; ++h)
        if (holes[2 * h] < 0 || holes[2 * h + 1] < holes[2 * h] || holes[2 * h + 1] > l_pac || (h && holes[2 * h] < holes[2 * h - 1])) {
            bm2_set_error(ctx, "bm2_mm_set: the holes must be sorted, disjoint [beg, end) ranges inside the reference"); return 1;
        }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    DevBuf *b = ctx->mm_d;
    const size_t pb = pac_bytes(l_pac), bb = bits_bytes(l_pac);
    if (b[MD_PAC].cap < pb || b[MD_HOLEBITS].cap < bb) {
        size_t fr = 0, tot = 0;
        BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
        fr += b[MD_PAC].cap + b[MD_HOLEBITS].cap;
        if (pb + bb > fr) {
            bm2_set_error(ctx, "bm2_mm_set: the reference needs " + std::to_string(pb + bb) + " bytes of device memory, " + std::to_string(fr) + " bytes free");
            return 1;
        }
        for (int s : {MD_PAC, MD_HOLEBITS}) { if (b[s].p) BM2_CUDA_OK(cudaFree(b[s].p)); b[s].p = nullptr; b[s].cap = 0; }
    }
    const size_t L = (size_t) MM_NCAT * kLenBins * 8, I = (size_t) MM_NORIENT * kInsBins * 8, C = (size_t) MM_NCAT * MM_NCOUNT * 8;
    if (ensure_exact(ctx, b[MD_PAC], pb) || ensure_exact(ctx, b[MD_HOLEBITS], bb) || ctx->ensure(b[MD_HOLES], (size_t) n_holes * 16 + 16) ||
        ctx->ensure(b[MD_HOLECHAR], (size_t) n_holes + 16) || ctx->ensure(b[MD_OFF], (size_t) n_contigs * 8 + 8) ||
        ctx->ensure(b[MD_LEN], (size_t) n_contigs * 4 + 8) || ensure_exact(ctx, b[MD_CNT], C) || ensure_exact(ctx, b[MD_LENH], L) ||
        ensure_exact(ctx, b[MD_MISH], L) || ensure_exact(ctx, b[MD_NOCALL], L) || ensure_exact(ctx, b[MD_INS], I) ||
        ctx->ensure(b[MD_SC], SC_END * 8)) return 1;
    cudaStream_t st = ctx->stream;
    char kmers[MM_N_ADAPTER_KMERS][MM_ADAPTER_LEN];
    mm_adapter_kmers(kmers);
    BM2_CUDA_OK(cudaMemcpyToSymbolAsync(c_kmers, kmers, sizeof kmers, 0, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(b[MD_PAC].p, pac, pb, cudaMemcpyHostToDevice, st));
    if (n_holes) {
        BM2_CUDA_OK(cudaMemcpyAsync(b[MD_HOLES].p, holes, (size_t) n_holes * 16, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[MD_HOLECHAR].p, hole_char, (size_t) n_holes, cudaMemcpyHostToDevice, st));
    }
    if (n_contigs) {
        BM2_CUDA_OK(cudaMemcpyAsync(b[MD_OFF].p, contig_off, (size_t) n_contigs * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[MD_LEN].p, contig_len, (size_t) n_contigs * 4, cudaMemcpyHostToDevice, st));
    }
    const int64_t n_words = (int64_t) bb / 4;
    mm_holes_kernel<<<(unsigned) bm2_min<int64_t>((n_words + 255) / 256, (int64_t) ctx->n_sm * 16), 256, 0, st>>>(
        (uint32_t *) b[MD_HOLEBITS].p, n_words, (const int64_t *) b[MD_HOLES].p, n_holes);
    BM2_CUDA_OK(cudaGetLastError());
    for (int s : {MD_CNT, MD_LENH, MD_MISH, MD_NOCALL, MD_INS}) BM2_CUDA_OK(cudaMemsetAsync(b[s].p, 0, b[s].cap, st));
    BM2_CUDA_OK(cudaMemsetAsync(b[MD_SC].p, 0, SC_END * 8, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    ctx->mm_l_pac = l_pac; ctx->mm_n_holes = n_holes; ctx->mm_n_contigs = n_contigs;
    ctx->mm_seen = 0; ctx->mm_big.clear(); ctx->mm_add_ms = 0; ctx->mm_finish_ms = 0;
    ctx->mm_set = true; ctx->mm_gc = false;
    return 0;
}

extern "C" int bm2_mm_memory(const bm2_ctx *ctx, int64_t l_pac, int64_t window_bytes, int64_t *needed, int64_t *free_bytes) {
    if (!ctx || l_pac < 0 || window_bytes < 0 || !needed || !free_bytes) return 1;
    bm2_ctx *ctx_for_error = (bm2_ctx *) ctx;
    // the reference, its bitset and the histograms exactly; the window, and per record its start, its MmInfo and a large insert size,
    // rounded up by 1.25 as bm2_ctx::ensure allocates
    const double w = (double) window_bytes, recs = w / kRecBytes + 1;
    const double bytes = (double) pac_bytes(l_pac) + (double) bits_bytes(l_pac) + (double) hist_bytes() +
                         1.25 * (w + recs * (8 + sizeof(MmInfo) + 8)) + 64.0 * (1 << 20);
    size_t fr = 0, tot = 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
    int64_t held = 0;
    for (int s : {MD_PAC, MD_HOLEBITS, MD_CNT, MD_LENH, MD_MISH, MD_NOCALL, MD_INS}) held += (int64_t) ctx->mm_d[s].cap;
    *needed = (int64_t) bytes; *free_bytes = (int64_t) fr + held;
    return 0;
}

extern "C" int bm2_mm_add(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts)) { if (ctx) bm2_set_error(ctx, "bm2_mm_add: bad arguments"); return 1; }
    if (!ctx->mm_set) { bm2_set_error(ctx, "bm2_mm_add: no reference on this context (bm2_mm_set)"); return 1; }
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t s = starts[i];
        if (s < 0 || s + 36 > n) { bm2_set_error(ctx, "bm2_mm_add: record " + std::to_string(i) + " is not inside the buffer"); return 1; }
        const BamFixed f = bam_fixed(recs + s);
        const int32_t l_seq = bam_le32(recs + s + 20);
        if (f.block_size < 32 || s + 4 + (int64_t) f.block_size > n || l_seq < 0 || f.l_read_name < 1 ||
            32 + (int64_t) f.l_read_name + 4 * (int64_t) f.n_cigar + (l_seq + 1) / 2 + (int64_t) l_seq > (int64_t) f.block_size) {
            bm2_set_error(ctx, "bm2_mm_add: record " + std::to_string(i) + " is malformed");
            return 1;
        }
    }
    if (!n_recs) return 0;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->mm_d;
    const size_t nr = (size_t) n_recs;
    const bool gc = ctx->mm_gc;
    if (ctx->ensure(b[MD_RECS], (size_t) n + 16) || ctx->ensure(b[MD_STARTS], nr * 8 + 8) || ctx->ensure(b[MD_INFO], nr * sizeof(MmInfo) + 8) ||
        ctx->ensure(b[MD_BIG], nr * 8 + 8) || (gc && ctx->ensure(b[MD_GC_INFO], nr * sizeof(MmGc) + 8))) return 1;
    MmGc *d_gc = (MmGc *) b[MD_GC_INFO].p;
    for (cudaEvent_t &ev : ctx->mm_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    uint8_t *d_recs = (uint8_t *) b[MD_RECS].p;
    const int64_t *d_starts = (const int64_t *) b[MD_STARTS].p;
    MmInfo *d_info = (MmInfo *) b[MD_INFO].p;
    unsigned long long *d_sc = (unsigned long long *) b[MD_SC].p;
    BM2_CUDA_OK(cudaMemcpyAsync(d_recs, recs, (size_t) n, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemcpyAsync(b[MD_STARTS].p, starts, nr * 8, cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemsetAsync(d_sc + SC_ERR, 0xff, 8, st));
    BM2_CUDA_OK(cudaMemsetAsync(d_sc + SC_BIG_N, 0, 8, st));
    const unsigned g = (unsigned) bm2_min<int64_t>((n_recs + kWarps - 1) / kWarps, (int64_t) ctx->n_sm * 8);
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[0], st));
    if (gc)
        mm_check_kernel<true><<<g, kWarps * 32, 0, st>>>(d_recs, d_starts, n_recs, (const int64_t *) b[MD_OFF].p, (const int32_t *) b[MD_LEN].p,
                                                         ctx->mm_n_contigs, d_info, d_sc, ctx->mm_seen, d_gc);
    else
        mm_check_kernel<false><<<g, kWarps * 32, 0, st>>>(d_recs, d_starts, n_recs, (const int64_t *) b[MD_OFF].p, (const int32_t *) b[MD_LEN].p,
                                                          ctx->mm_n_contigs, d_info, d_sc, ctx->mm_seen, nullptr);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[1], st));
    unsigned long long err = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&err, d_sc + SC_ERR, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->mm_ev[0], ctx->mm_ev[1]));
    ctx->mm_add_ms += ms;
    if (gc) ctx->mm_gc_add_ms += ms;
    if (err != ~0ULL) {                                                  // a read error: nothing of this window is counted
        const int64_t idx = (int64_t) (err >> 4), i = idx - ctx->mm_seen;
        const uint8_t *r = recs + starts[i];
        bm2_set_error(ctx, "bm2_mm_add: read " + std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0) + " (record " + std::to_string(idx) + ") " +
                               kErrText[(err & 15) - 1]);
        return 2;
    }
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[0], st));
    if (gc)
        mm_count_kernel<true><<<g, kWarps * 32, 0, st>>>(d_recs, d_starts, n_recs, d_info, (const uint8_t *) b[MD_PAC].p,
                                                         (const uint32_t *) b[MD_HOLEBITS].p, (const int64_t *) b[MD_HOLES].p,
                                                         (const char *) b[MD_HOLECHAR].p, ctx->mm_n_holes, (unsigned long long *) b[MD_CNT].p,
                                                         (unsigned long long *) b[MD_LENH].p, (unsigned long long *) b[MD_MISH].p,
                                                         (unsigned long long *) b[MD_NOCALL].p, (unsigned long long *) b[MD_INS].p,
                                                         (uint64_t *) b[MD_BIG].p, d_sc, d_gc, (unsigned long long *) b[MD_GC_CNT].p);
    else
        mm_count_kernel<false><<<g, kWarps * 32, 0, st>>>(d_recs, d_starts, n_recs, d_info, (const uint8_t *) b[MD_PAC].p,
                                                          (const uint32_t *) b[MD_HOLEBITS].p, (const int64_t *) b[MD_HOLES].p,
                                                          (const char *) b[MD_HOLECHAR].p, ctx->mm_n_holes, (unsigned long long *) b[MD_CNT].p,
                                                          (unsigned long long *) b[MD_LENH].p, (unsigned long long *) b[MD_MISH].p,
                                                          (unsigned long long *) b[MD_NOCALL].p, (unsigned long long *) b[MD_INS].p,
                                                          (uint64_t *) b[MD_BIG].p, d_sc, nullptr, nullptr);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[1], st));
    unsigned long long n_big = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&n_big, d_sc + SC_BIG_N, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->mm_ev[0], ctx->mm_ev[1]));
    ctx->mm_add_ms += ms;
    if (gc) ctx->mm_gc_add_ms += ms;
    if (n_big) {                                                         // the window's large insert sizes, kept on the host until the finish
        const size_t at = ctx->mm_big.size();
        ctx->mm_big.resize(at + (size_t) n_big);
        BM2_CUDA_OK(cudaMemcpy(ctx->mm_big.data() + at, b[MD_BIG].p, (size_t) n_big * 8, cudaMemcpyDeviceToHost));
    }
    ctx->mm_seen += n_recs;
    return 0;
}

extern "C" int bm2_mm_finish(bm2_ctx *ctx, bm2_mm_result_t *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out) { if (ctx) bm2_set_error(ctx, "bm2_mm_finish: bad arguments"); return 1; }
    if (!ctx->mm_set) { bm2_set_error(ctx, "bm2_mm_finish: no reference on this context (bm2_mm_set)"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->mm_d;
    for (cudaEvent_t &ev : ctx->mm_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    unsigned long long sc[SC_END];
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[0], st));
    BM2_CUDA_OK(cudaMemcpyAsync(sc, b[MD_SC].p, sizeof sc, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(out->counts, b[MD_CNT].p, sizeof out->counts, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    const size_t L = (size_t) sc[SC_MAX_LEN] + 1, I = (size_t) sc[SC_MAX_INS] + 1;
    ctx->mm_hist.assign(3 * MM_NCAT * L + MM_NORIENT * I, 0);
    int64_t *h = ctx->mm_hist.data();
    for (int a = 0; a < 3; ++a)                                          // len_hist, mism_hist, nocall: rows of max_len + 1
        BM2_CUDA_OK(cudaMemcpy2DAsync(h + (size_t) a * MM_NCAT * L, L * 8, (const int64_t *) b[MD_LENH + a].p, kLenBins * 8, L * 8, MM_NCAT,
                                      cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpy2DAsync(h + 3 * MM_NCAT * L, I * 8, b[MD_INS].p, kInsBins * 8, I * 8, MM_NORIENT, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[1], st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->mm_ev[0], ctx->mm_ev[1]));
    ctx->mm_finish_ms = ms;
    std::sort(ctx->mm_big.begin(), ctx->mm_big.end());
    out->max_len = (int32_t) sc[SC_MAX_LEN];
    out->len_hist = h; out->mism_hist = h + MM_NCAT * L; out->nocall = h + 2 * MM_NCAT * L;
    out->max_insert = (int32_t) sc[SC_MAX_INS];
    out->insert_hist = h + 3 * MM_NCAT * L;
    out->insert_big = ctx->mm_big.data(); out->n_big = (int64_t) ctx->mm_big.size();
    out->records = ctx->mm_seen;
    out->add_ms = ctx->mm_add_ms; out->finish_ms = ctx->mm_finish_ms;
    return 0;
}

extern "C" int bm2_mm_gc_memory(const bm2_ctx *ctx, int64_t window_bytes, int64_t *needed) {
    if (!ctx || window_bytes < 0 || !needed) return 1;
    // the bins exactly; per record its MmGc, rounded up by 1.25 as bm2_ctx::ensure allocates.  The scan needs nothing more: it reads the hole
    // letters from the hole list bm2_mm_set uploaded.
    const double recs = (double) window_bytes / kRecBytes + 1;
    *needed = (int64_t) ((double) (MM_GC_BINS + GC_NCOUNT) * 8 + 1.25 * recs * sizeof(MmGc));
    return 0;
}

extern "C" int bm2_mm_gc_set(bm2_ctx *ctx) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx) return 1;
    if (!ctx->mm_set) { bm2_set_error(ctx, "bm2_mm_gc_set: no reference on this context (bm2_mm_set)"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->mm_d;
    const int32_t nc = ctx->mm_n_contigs;
    std::vector<int64_t> off((size_t) nc);
    std::vector<int32_t> len((size_t) nc);
    if (nc) {
        BM2_CUDA_OK(cudaMemcpy(off.data(), b[MD_OFF].p, (size_t) nc * 8, cudaMemcpyDeviceToHost));
        BM2_CUDA_OK(cudaMemcpy(len.data(), b[MD_LEN].p, (size_t) nc * 4, cudaMemcpyDeviceToHost));
    }
    for (int32_t k = 1; k < nc; ++k)
        if (off[k] < off[k - 1] + len[k - 1]) { bm2_set_error(ctx, "bm2_mm_gc_set: the contigs must be sorted and disjoint"); return 1; }
    const size_t win = (size_t) MM_GC_BINS * 8, cnt = (size_t) GC_NCOUNT * 8;
    if (b[MD_GC_WIN].cap < win || b[MD_GC_CNT].cap < cnt) {
        size_t fr = 0, tot = 0;
        BM2_CUDA_OK(cudaMemGetInfo(&fr, &tot));
        if (win + cnt > fr) {
            bm2_set_error(ctx, "bm2_mm_gc_set: GC bias needs " + std::to_string(win + cnt) + " bytes of device memory, " + std::to_string(fr) + " bytes free");
            return 1;
        }
    }
    if (ensure_exact(ctx, b[MD_GC_WIN], win) || ensure_exact(ctx, b[MD_GC_CNT], cnt)) return 1;
    for (cudaEvent_t &ev : ctx->mm_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    BM2_CUDA_OK(cudaMemsetAsync(b[MD_GC_WIN].p, 0, win, st));
    BM2_CUDA_OK(cudaMemsetAsync(b[MD_GC_CNT].p, 0, cnt, st));
    const int64_t n_tiles = (ctx->mm_l_pac + kScanTile - 1) / kScanTile;
    // at least one block per 4096 tiles, so that a block's 32-bit shared bins hold its windows (4096 * kScanTile < 2^32)
    const int64_t grid = bm2_min<int64_t>(n_tiles, bm2_max<int64_t>((int64_t) ctx->n_sm * 8, (n_tiles + 4095) / 4096));
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[0], st));
    mm_gc_scan_kernel<<<(unsigned) grid, kScanThreads, 0, st>>>((const uint8_t *) b[MD_PAC].p, (const uint32_t *) b[MD_HOLEBITS].p,
                                                                 (const int64_t *) b[MD_HOLES].p, (const char *) b[MD_HOLECHAR].p, ctx->mm_n_holes,
                                                                 ctx->mm_l_pac, (const int64_t *) b[MD_OFF].p, (const int32_t *) b[MD_LEN].p, nc, n_tiles,
                                                                 (unsigned long long *) b[MD_GC_WIN].p);
    BM2_CUDA_OK(cudaGetLastError());
    BM2_CUDA_OK(cudaEventRecord(ctx->mm_ev[1], st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    BM2_CUDA_OK(cudaEventElapsedTime(&ms, ctx->mm_ev[0], ctx->mm_ev[1]));
    ctx->mm_gc_scan_ms = ms; ctx->mm_gc_add_ms = 0;
    ctx->mm_gc = true;
    return 0;
}

extern "C" int bm2_mm_gc_finish(bm2_ctx *ctx, bm2_mm_gc_result_t *out) {
    bm2_ctx *ctx_for_error = ctx;
    if (!ctx || !out) { if (ctx) bm2_set_error(ctx, "bm2_mm_gc_finish: bad arguments"); return 1; }
    if (!ctx->mm_set || !ctx->mm_gc) { bm2_set_error(ctx, "bm2_mm_gc_finish: GC bias is not on for this context (bm2_mm_gc_set)"); return 1; }
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    unsigned long long c[GC_NCOUNT];
    BM2_CUDA_OK(cudaMemcpy(out->windows, ctx->mm_d[MD_GC_WIN].p, sizeof out->windows, cudaMemcpyDeviceToHost));
    BM2_CUDA_OK(cudaMemcpy(c, ctx->mm_d[MD_GC_CNT].p, sizeof c, cudaMemcpyDeviceToHost));
    for (int k = 0; k < MM_GC_BINS; ++k) {
        out->reads[k] = (int64_t) c[GC_READS + k]; out->bases[k] = (int64_t) c[GC_BASES + k]; out->errors[k] = (int64_t) c[GC_ERRORS + k];
    }
    out->total_clusters = (int64_t) c[GC_CLUSTERS]; out->aligned_reads = (int64_t) c[GC_ALIGNED];
    out->scan_ms = ctx->mm_gc_scan_ms; out->add_ms = ctx->mm_gc_add_ms;
    return 0;
}

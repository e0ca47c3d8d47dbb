// bsw.cu — banded affine-gap seed-extension (BSW) kernels for sm_90a.
//
// Replaces BandedPairWiseSW::{getScores8,getScores16,scalarBandedSWAWrapper}
// (reference src/bandedSWA.cpp:1970, :2664, :242).  Semantics = ksw_extend2 / scalarBandedSWA
// (src/bandedSWA.cpp:116-237) with the band derived as the SIMD wrappers derive it
// (src/bandedSWA.cpp:2905-2926).
//
// Kernel "thread-per-job" (short queries, the 2x151 bp workload): the DP of one job is
// row-sequential with data-dependent band / early exit, so parallelism is taken ACROSS jobs, one
// job per thread, exactly the inter-sequence scheme of the reference's SIMD kernels but 32-wide
// SIMT with independent control per lane.  The per-column state {H(i-1,j-1), E(i,j)} is packed
// 16+16 bit in one shared-memory word laid out [column][thread] (bank == lane: conflict-free for
// any per-thread column), the query is packed 4 bit/base in the same layout.  Jobs are radix-sorted
// by (query-length class, target length) so that the 32 lanes of a warp run similar trip counts.
// Integer-ALU bound; HBM traffic is ~(qlen+tlen+56) B per job.
#include "bm2_common.cuh"
#include "bsw_pair.cuh"
#include "bsw_col2.cuh"
#include <cstdlib>
#include <mutex>
#include <cub/device/device_radix_sort.cuh>

#define BSW_THREADS 128
#define BSW_NBOUND 12
#define BSW_NCLASS 24          // class = 2 * bound index + (needs 16-bit state); class 24 = wide (warp / global-state kernels)
#define BSW_NPAIR 5            // pair classes 25..29: two jobs per thread in packed 16-bit halves (bsw_pair.cuh), bounds 32..96
#define BSW_PAIR0 (BSW_NCLASS + 1)
#define BSW_NALL (BSW_PAIR0 + BSW_NPAIR)
// Upper query-length bound of each class (state words = bound + 2).  The shared memory of a launch is sized by its bound and decides how many
// CTAs (4 warps each) an SM holds - the column-pair kernel needs 6 B per column pair and thread - so every bound up to 256 is the LARGEST query
// length that still fits k CTAs of 128 threads into 227 KB: k = 16, 11, 8, 7, 6, 5, 4, 3, 2.  (Round 2: with the bounds 32, 64, ... 160 the right
// extensions of 129..132 columns of a 151 bp read ran in the 160-column class at 3 CTAs per SM and took as long as the whole 128-column class.)
__constant__ int c_class_bound[BSW_NBOUND] = {32, 48, 70, 80, 96, 116, 146, 196, 256, 384, 512, 1024};
static const int h_class_bound[BSW_NBOUND] = {32, 48, 70, 80, 96, 116, 146, 196, 256, 384, 512, 1024};

struct BswSortScratch {
    uint32_t *keys_in, *keys_out;
    int32_t *idx_in, *idx_out;
    int32_t *class_cnt;      // BSW_NCLASS + 2 counters (last = "global-state" class)
    int32_t *class_off;      // BSW_NCLASS + 3 offsets
    void *cub_tmp;
    size_t cub_bytes;
};

__device__ __forceinline__ int bsw_class_of(int qlen, int tlen, int h0, int a) {
    // scores must fit 15 bits for the packed state (same rule as the reference's int16 class,
    // src/bwamem.cpp:2307); anything else goes to the wide / global-state kernel.
    int minlen = qlen < tlen ? qlen : tlen;
    long long maxsc = (long long) h0 + (long long) minlen * a;
    if (maxsc >= 32768 || qlen > c_class_bound[BSW_NBOUND - 1]) return BSW_NCLASS;
    const int wide16 = maxsc > 255 ? 1 : 0;
#pragma unroll
    for (int c = 0; c < BSW_NBOUND; ++c)
        if (qlen <= c_class_bound[c]) return 2 * c + wide16;
    return BSW_NCLASS;
}

__global__ void bsw_keys_kernel(const BswJob *jobs, int n, int a, int pair_ok, const uint8_t *__restrict__ qbase, uint32_t *keys, int32_t *idx,
                                int32_t *class_cnt) {
    __shared__ int hist[BSW_NALL];
    if (threadIdx.x < BSW_NALL) hist[threadIdx.x] = 0;
    __syncthreads();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        BswJob j = jobs[i];
        int c = bsw_class_of(j.qlen, j.tlen, j.h0, a);
        // 8-bit-score jobs with a short N-free query run two per thread (bsw_pair_kernel)
        if (pair_ok && !(c & 1) && c < 2 * BSW_NPAIR) {
            const uint8_t *qp = qbase + j.qoff;
            bool has_n = false;
            for (int k = 0; k < j.qlen && !has_n; ++k) has_n = qp[(long long) k * j.qstride] > 3;
            if (!has_n) c = BSW_PAIR0 + (c >> 1);
        }
        // ascending sort => class ascending, then query length descending (long jobs first: the persistent CTAs take them first),
        // then h0 descending, then target length: query length and h0 shape the band of every row, so the 32 jobs of a warp run rows of
        // similar width (row-lockstep model on the reference's jobs, scripts/study_bsw_order.py: efficiency 0.92 against 0.85 for
        // round 1's (target length, query length) key)
        const int q = j.qlen > 0x3FF ? 0x3FF : j.qlen;
        const int h = j.h0 < 0 ? 0 : (j.h0 > 0x3FF ? 0x3FF : j.h0);
        const int t = (j.tlen >> 3) > 0x7F ? 0x7F : (j.tlen >> 3);
        keys[i] = ((uint32_t) c << 27) | ((uint32_t) (0x3FF - q) << 17) | ((uint32_t) (0x3FF - h) << 7) | (uint32_t) (0x7F - t);   // c <= 29: 5 bits
        idx[i] = i;
        atomicAdd(&hist[c], 1);
    }
    __syncthreads();
    if (threadIdx.x < BSW_NALL && hist[threadIdx.x]) atomicAdd(&class_cnt[threadIdx.x], hist[threadIdx.x]);
}

__global__ void bsw_class_off_kernel(const int32_t *class_cnt, int32_t *class_off) {
    if (threadIdx.x == 0) {
        int s = 0;
        for (int c = 0; c < BSW_NALL; ++c) { class_off[c] = s; s += class_cnt[c]; }
        class_off[BSW_NALL] = s;
    }
}

// ---------------------------------------------------------------------------------------------
// The extension DP of one job (one thread).  `St` abstracts the per-column state storage.
// ---------------------------------------------------------------------------------------------
// (Measured: splitting H and E into separate narrow arrays - 2 LDS + 2 STS per cell instead of pack/unpack ALU
// ops - made the kernel slower in an A/B; the packed word stays.)
// The kernel is bound by the integer-ALU pipe (LOP3/SHF/VIMNMX/SEL/PRMT); the FMA pipe (IMAD) idles.  Field
// extraction and packing are therefore written as multiply-adds so that they issue on the FMA pipe:
//   x >> s == umulhi(x, 2^(32-s)),  x & (2^s-1) == x - (x >> s) * 2^s,  (a << s) | b == a * 2^s + b  (b < 2^s).
__device__ __forceinline__ uint32_t fma_shr(uint32_t x, uint32_t two_pow_32_minus_s) { return __umulhi(x, two_pow_32_minus_s); }
__device__ __forceinline__ int fma_mad(int a, int b, int c) { int d; asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }

struct SmemPacked {            // H | E<<16 in shared memory, [column][thread]; explicit shared-space accesses
    unsigned base;             // shared-window address of &sh[threadIdx.x]
    unsigned stride;           // blockDim.x * 4 bytes
    __device__ __forceinline__ uint32_t ldw(int j) const {
        uint32_t w; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(base + (unsigned) j * stride)); return w;
    }
    __device__ __forceinline__ void stw(int j, uint32_t w) const {
        asm volatile("st.shared.u32 [%0], %1;" :: "r"(base + (unsigned) j * stride), "r"(w) : "memory");
    }
    __device__ __forceinline__ void get(int j, int &h, int &e) const { uint32_t w = ldw(j); e = (int) fma_shr(w, 1u << 16); h = fma_mad(e, -65536, (int) w); }
    __device__ __forceinline__ void put(int j, int h, int e) const { stw(j, (uint32_t) fma_mad(e, 65536, h)); }
    __device__ __forceinline__ bool zero(int j) const { return ldw(j) == 0u; }
    // row maximum as one signed key: (h << 16) | j  (h < 2^15, j < 2^16)
    typedef int key_t;
    static constexpr unsigned kStateBytes = 4;
    static __device__ __forceinline__ key_t key(int h, int j) { return fma_mad(h, 65536, j); }
    static __device__ __forceinline__ int key_h(key_t k) { return k >> 16; }
    static __device__ __forceinline__ int key_j(key_t k) { return k & 0xFFFF; }
};

struct SmemPacked8 {           // H | E<<8 in 16 bits: jobs whose best possible score fits 8 bits (the 2x151 bp workload)
    unsigned base;             // shared-window address of the thread's column 0
    unsigned stride;           // blockDim.x * 2 bytes
    __device__ __forceinline__ uint32_t ldw(int j) const {
        uint16_t w; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(w) : "r"(base + (unsigned) j * stride)); return (uint32_t) w;
    }
    __device__ __forceinline__ void stw(int j, uint32_t w) const {
        asm volatile("st.shared.u16 [%0], %1;" :: "r"(base + (unsigned) j * stride), "h"((uint16_t) w) : "memory");
    }
    __device__ __forceinline__ void get(int j, int &h, int &e) const { uint32_t w = ldw(j); e = (int) fma_shr(w, 1u << 24); h = fma_mad(e, -256, (int) w); }
    __device__ __forceinline__ void put(int j, int h, int e) const { stw(j, (uint32_t) fma_mad(e, 256, h)); }
    __device__ __forceinline__ bool zero(int j) const { return ldw(j) == 0u; }
    typedef int key_t;
    static constexpr unsigned kStateBytes = 2;
    static __device__ __forceinline__ key_t key(int h, int j) { return fma_mad(h, 65536, j); }
    static __device__ __forceinline__ int key_h(key_t k) { return k >> 16; }
    static __device__ __forceinline__ int key_j(key_t k) { return k & 0xFFFF; }
};

struct GmemWide {              // {H,E} int32 in global memory, private stripe per thread
    int2 *base;
    __device__ __forceinline__ void get(int j, int &h, int &e) const { int2 v = base[j]; h = v.x; e = v.y; }
    __device__ __forceinline__ void put(int j, int h, int e) const { base[j] = make_int2(h, e); }
    __device__ __forceinline__ bool zero(int j) const { int2 v = base[j]; return (v.x | v.y) == 0; }
    typedef long long key_t;     // 32-bit scores: (h << 32) | j
    static __device__ __forceinline__ key_t key(int h, int j) { return ((long long) h << 32) | (unsigned) j; }
    static __device__ __forceinline__ int key_h(key_t k) { return (int) (k >> 32); }
    static __device__ __forceinline__ int key_j(key_t k) { return (int) (k & 0xFFFFFFFFLL); }
};

template <class St, class QFetch>
__device__ __forceinline__ void bsw_extend_one(const St &st, const QFetch &qf, const uint8_t *__restrict__ tptr, int tstride,
                                               int qlen, int tlen, int h0, const BswParams &p, BswOut &o,
                                               unsigned long long &cells)
{
    const int oe_del = p.o_del + p.e_del, oe_ins = p.o_ins + p.e_ins;
    const int e_del = p.e_del, e_ins = p.e_ins, sa = p.a, sb = -p.b;
    // first row (bandedSWA.cpp:141-144); columns 0..qlen, E = 0
    {
        int h = h0;
        st.put(0, h, 0);
        h = h0 > oe_ins ? h0 - oe_ins : 0;
        for (int j = 1; j <= qlen; ++j) {
            st.put(j, h, 0);
            h = h > e_ins ? h - e_ins : 0;
        }
        // NB: reference stops writing when the value reaches <= e_ins and leaves zeros; identical.
    }
    // band (SIMD wrapper arithmetic, bandedSWA.cpp:2905-2926; == scalar :146-156 when e == 1)
    int w = p.w;
    const BswQuirk qk = bsw_quirk(qlen, tlen, h0, p);
    {
        unsigned t1 = ((unsigned) (qlen * sa) + (unsigned) (p.end_bonus - p.o_ins)) & qk.band_mask;
        int max_ins = (int) (t1 / (unsigned) e_ins) + 1; if (max_ins < 1) max_ins = 1;
        unsigned t2 = ((unsigned) (qlen * sa) + (unsigned) (p.end_bonus - p.o_del)) & qk.band_mask;
        int max_del = (int) (t2 / (unsigned) e_del) + 1; if (max_del < 1) max_del = 1;
        if (w > max_ins) w = max_ins;
        if (w > max_del) w = max_del;
    }
    int best = h0, best_i = -1, best_j = -1, best_ie = -1, gscore = -1, max_off = 0;
    int beg = 0, end = qlen;
    unsigned long long ncell = 0;
    for (int i = 0; i < tlen; ++i) {
        if (beg < i - w) beg = i - w;
        if (end > i + w + 1) end = i + w + 1;
        if (end > qlen) end = qlen;
        int h1;
        if (beg == 0) { h1 = h0 - (p.o_del + e_del * (i + 1)); if (h1 < 0) h1 = 0; }
        else h1 = 0;
        const int tb = tptr[(long long) i * tstride];
        // score of target base tb against query base q = 0..3 as four signed bytes; q = 4 (or tb > 3) -> -1
        const uint32_t sb8 = (uint32_t) sb & 0xFFu, sa8 = (uint32_t) sa & 0xFFu;
        uint32_t tbl = sb8 * 0x01010101u;
        tbl = tb > 3 ? 0xFFFFFFFFu : ((tbl & ~(0xFFu << (8 * tb))) | (sa8 << (8 * tb)));
        int f = 0;
        typename St::key_t mkey = -1;                // (h, j) packed; signed max => last column attaining the row maximum
        int j = beg;
        auto cell = [&](const int jj, const uint32_t qb) {
            int hd, e;
            st.get(jj, hd, e);
            // PRMT: byte 0 = tbl[qb] (qb = 4 selects the 0xFF byte of the second operand), bytes 1..3 = its sign
            int s;     // (inline PTX: the __byte_perm intrinsic masks the sign-replicate bit of the selector nibbles)
            asm("prmt.b32 %0, %1, %2, %3;" : "=r"(s) : "r"(tbl), "r"(0xFFFFFFFFu), "r"(qb * 0x1111u + 0x8880u));
            // hd ? hd + s : 0, clamped at 0 (h, e and f are >= 0, so a negative M never shows): min against hd * 1024 is the hd == 0 test
            const int M = max(min(hd + s, hd * 1024), 0);
            const int h = (int) max(max((unsigned) M, (unsigned) e), (unsigned) f);     // all three are >= 0
            int t = max(M - oe_del, 0);
            e = max(e - e_del, t);
            st.put(jj, h1, e);
            t = max(M - oe_ins, 0);
            f = max(f - e_ins, t);
            h1 = h;
            mkey = max(mkey, St::key(h, jj));
        };
        if (QFetch::kPacked) {
            // head (to the next multiple of 8 columns), 8-column groups with one query word each, tail
            if (j < end && (j & 7)) {
                uint32_t qw = qf.word(j >> 3) >> ((j & 7) * 4);
                const int he = min(end, (j + 7) & ~7);
                for (; j < he; ++j) { const uint32_t nx = fma_shr(qw, 1u << 28); cell(j, (uint32_t) fma_mad((int) nx, -16, (int) qw)); qw = nx; }
            }
            for (; j + 8 <= end; j += 8) {
                uint32_t qw = qf.word(j >> 3);
#pragma unroll
                for (int u = 0; u < 8; ++u) { const uint32_t nx = fma_shr(qw, 1u << 28); cell(j + u, (uint32_t) fma_mad((int) nx, -16, (int) qw)); qw = nx; }
            }
            if (j < end) {
                uint32_t qw = qf.word(j >> 3);
                for (; j < end; ++j) { const uint32_t nx = fma_shr(qw, 1u << 28); cell(j, (uint32_t) fma_mad((int) nx, -16, (int) qw)); qw = nx; }
            }
        } else {
            typename QFetch::Cursor qc = qf.cursor(beg);
            for (; j < end; ++j) cell(j, (uint32_t) qf.next(qc, j));
        }
        const int m = mkey < 0 ? 0 : St::key_h(mkey);
        const int mj = mkey < 0 ? -1 : St::key_j(mkey);
        if (end > beg) ncell += (unsigned) (end - beg);
        st.put(end, h1, 0);
        if (j == qlen) {
            if (h1 >= gscore) best_ie = i;
            if (h1 > gscore) gscore = h1;
        }
        if (m == 0) break;
        if (m > best) {
            best = m; best_i = i; best_j = mj;
            int d = mj - i; d = d < 0 ? -d : d;
            if (d > max_off) max_off = d;
            if (0 > qk.zthr) break;
        } else {
            int di = i - best_i, dj = mj - best_j;
            int pen = di > dj ? di - dj : dj - di;       // SIMD z-drop: no e_del/e_ins factor, no `zdrop > 0` guard (ZSCORE8/16)
            if (best - m - pen > qk.zthr) break;
        }
        for (j = beg; j < end && st.zero(j); ++j) {}
        beg = j;
        for (j = end; j >= beg && st.zero(j); --j) {}
        end = j + 2 < qlen ? j + 2 : qlen;
    }
    o.score = best; o.qle = best_j + 1; o.tle = best_i + 1; o.gtle = best_ie + 1; o.gscore = gscore; o.max_off = max_off;
    cells += ncell;
}

// query packed 4 bit / base in shared memory words [word][thread]
struct QSmem4 {                // query packed 4 bit / base, [word][thread]
    unsigned base;             // shared-window address of &sh[W * blockDim.x + threadIdx.x]
    unsigned stride;
    static constexpr bool kPacked = true;
    struct Cursor { uint32_t w; };
    __device__ __forceinline__ uint32_t word(int k) const { return ldw(k); }
    __device__ __forceinline__ uint32_t ldw(int k) const {
        uint32_t w; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(base + (unsigned) k * stride)); return w;
    }
    __device__ __forceinline__ Cursor cursor(int j) const { Cursor c; c.w = ldw(j >> 3) >> ((j & 7) * 4); return c; }
    __device__ __forceinline__ int next(Cursor &c, int j) const {
        if ((j & 7) == 0) c.w = ldw(j >> 3);
        const uint32_t nxt = fma_shr(c.w, 1u << 28);           // c.w >> 4 on the FMA pipe
        const int b = fma_mad((int) nxt, -16, (int) c.w);          // c.w & 15
        c.w = nxt;
        return b;
    }
};

struct QGmem {                 // query bytes straight from global memory
    const uint8_t *ptr; int stride;
    static constexpr bool kPacked = false;
    __device__ __forceinline__ uint32_t word(int) const { return 0; }
    struct Cursor { int dummy; };
    __device__ __forceinline__ Cursor cursor(int) const { return Cursor(); }
    __device__ __forceinline__ int next(Cursor &, int j) const { return ptr[(long long) j * stride]; }
};

template <class St>
__global__ void __launch_bounds__(BSW_THREADS)
bsw_thread_kernel(const BswJob *__restrict__ jobs, const int32_t *__restrict__ perm, const int32_t *__restrict__ class_off,
                  int cls, BswOut *__restrict__ out, const uint8_t *__restrict__ tbase, const uint8_t *__restrict__ qbase,
                  BswParams p, int W, unsigned long long *cells)
{
    extern __shared__ uint32_t sh[];
    const int first = class_off[cls], last = class_off[cls + 1];
    const int nthr = blockDim.x;
    const unsigned state_bytes = St::kStateBytes;
    // state columns first (W entries of state_bytes per thread), then the packed query words
    const unsigned q_off_words = ((unsigned) W * nthr * state_bytes + 3u) / 4u;
    unsigned long long ncell = 0;
    for (int blk = blockIdx.x; first + blk * nthr < last; blk += gridDim.x) {      // persistent CTAs: long jobs first
        const int g = first + blk * nthr + threadIdx.x;
        if (g < last) {
            const int id = perm[g];
            const BswJob job = jobs[id];
            const uint8_t *qp = qbase + job.qoff;
            uint32_t *qs = sh + q_off_words + threadIdx.x;
            for (int k = 0; k < job.qlen; k += 8) {
                uint32_t wv = 0;
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    int jj = k + u;
                    uint32_t b = jj < job.qlen ? (uint32_t) qp[(long long) jj * job.qstride] : 4u;
                    if (b > 4u) b = 4u;
                    wv |= b << (4 * u);
                }
                qs[(k >> 3) * nthr] = wv;
            }
            St st; st.base = (unsigned) __cvta_generic_to_shared(sh) + threadIdx.x * state_bytes; st.stride = (unsigned) nthr * state_bytes;
            QSmem4 qf; qf.base = (unsigned) __cvta_generic_to_shared(qs); qf.stride = (unsigned) nthr * 4u;
            BswOut o;
            bsw_extend_one(st, qf, tbase + job.toff, (int) job.tstride, job.qlen, job.tlen, job.h0, p, o, ncell);
            out[id] = o;
        }
    }
    if (cells) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) ncell += __shfl_xor_sync(0xffffffffu, ncell, d);
        if ((threadIdx.x & 31) == 0 && ncell) atomicAdd(cells, ncell);
    }
}

// ---------------------------------------------------------------------------------------------
// One job per thread, two adjacent columns per packed instruction (bsw_col2.cuh): the 8-bit-score classes with at most
// 256 query columns, i.e. every job of a 2x151 bp read.  Shared memory: state words {H, E} x 2 columns [pair][thread],
// then the query as one PRMT selector byte per column, 4 columns per word [word][thread].
// ---------------------------------------------------------------------------------------------
template <int NTHR>                     // compile-time strides: the pair loop walks the columns with constant pointer increments
struct Col2MemShared {
    unsigned st_base, q_base;           // shared-window byte addresses of the thread's pair 0 (state words / 16-bit selector pairs)
    static constexpr unsigned stride = NTHR * 4u, qstride = NTHR * 2u;
    __device__ __forceinline__ uint32_t ldw(int q) const {
        uint32_t w; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(st_base + (unsigned) q * stride)); return w;
    }
    __device__ __forceinline__ void stw(int q, uint32_t w) const {
        asm volatile("st.shared.u32 [%0], %1;" :: "r"(st_base + (unsigned) q * stride), "r"(w) : "memory");
    }
    __device__ __forceinline__ uint32_t ldh(int j) const {
        uint16_t w; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(w) : "r"(st_base + (unsigned) (j >> 1) * stride + 2u * (unsigned) (j & 1))); return (uint32_t) w;
    }
    __device__ __forceinline__ void sth(int j, uint32_t v) const {
        asm volatile("st.shared.u16 [%0], %1;" :: "r"(st_base + (unsigned) (j >> 1) * stride + 2u * (unsigned) (j & 1)), "h"((uint16_t) v) : "memory");
    }
    __device__ __forceinline__ uint32_t sel16(int q) const {
        uint16_t w; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(w) : "r"(q_base + (unsigned) q * qstride)); return (uint32_t) w;
    }
};

template <int NTHR>
__global__ void __launch_bounds__(NTHR)
bsw_col2_kernel(const BswJob *__restrict__ jobs, const int32_t *__restrict__ perm, const int32_t *__restrict__ class_off,
                int cls, BswOut *__restrict__ out, const uint8_t *__restrict__ tbase, const uint8_t *__restrict__ qbase,
                BswParams p, int NP, unsigned long long *cells, int reg_shrink, int *next_job)
{
    extern __shared__ uint32_t sh[];
    const int first = class_off[cls], last = class_off[cls + 1];
    Col2MemShared<NTHR> mem;
    mem.st_base = (unsigned) __cvta_generic_to_shared(sh) + threadIdx.x * 4u;
    mem.q_base = (unsigned) __cvta_generic_to_shared(sh) + (unsigned) NP * NTHR * 4u + threadIdx.x * 2u;
    const bool same_oe = p.o_del + p.e_del == p.o_ins + p.e_ins;
    unsigned long long ncell = 0;
    // Persistent warps, long jobs first.  next_job != nullptr: every WARP takes the next 32 jobs of the sorted class from a counter when it
    // is done with its own (the warps of a CTA never synchronise), so that the launch ends within one short job of the last fetch instead of
    // with the CTAs that the static round-robin happened to give the longer blocks (ncu r2c: 22.4 % of the warp slots active against 25 %
    // resident = a tenth of every launch was its tail).  nullptr: the static order (BM2_BSW_DYN=0, A/B measurements).
    const int lane = threadIdx.x & 31;
    for (int blk = blockIdx.x; ; blk += gridDim.x) {
        int g;
        if (next_job) {
            int b = 0;
            if (lane == 0) b = atomicAdd(next_job, 32);
            g = first + __shfl_sync(0xffffffffu, b, 0) + lane;
            if (g - lane >= last) break;
        } else {
            if (first + blk * NTHR >= last) break;
            g = first + blk * NTHR + threadIdx.x;
        }
        if (g < last) {
            const int id = perm[g];
            const BswJob job = jobs[id];
            const uint8_t *qp = qbase + job.qoff;
            // selector bytes of columns 2q, 2q+1 as one 16-bit word per pair, up to the pair that holds column qlen (read masked)
            for (int k = 0; k <= job.qlen; k += 2) {
                const int b0 = k < job.qlen ? (int) qp[(long long) k * job.qstride] : 4;
                const int b1 = k + 1 < job.qlen ? (int) qp[(long long) (k + 1) * job.qstride] : 4;
                const uint32_t wv = c2_selector_byte(b0) | (c2_selector_byte(b1) << 8);
                asm volatile("st.shared.u16 [%0], %1;" :: "r"(mem.q_base + (unsigned) (k >> 1) * (NTHR * 2u)), "h"((uint16_t) wv) : "memory");
            }
            BswOut o;
            if (same_oe && reg_shrink == 1) bsw_col2_extend<true>(mem, tbase + job.toff, (int) job.tstride, job.qlen, job.tlen, job.h0, p, o, ncell);
            else if (same_oe && reg_shrink == 2) bsw_col2_extend<true, Col2MemShared<NTHR>, 0, 8>(mem, tbase + job.toff, (int) job.tstride, job.qlen, job.tlen, job.h0, p, o, ncell);
            else if (same_oe && reg_shrink == 3) bsw_col2_extend<true, Col2MemShared<NTHR>, 2>(mem, tbase + job.toff, (int) job.tstride, job.qlen, job.tlen, job.h0, p, o, ncell);
            else if (same_oe) bsw_col2_extend<true, Col2MemShared<NTHR>, 0>(mem, tbase + job.toff, (int) job.tstride, job.qlen, job.tlen, job.h0, p, o, ncell);
            else bsw_col2_extend<false>(mem, tbase + job.toff, (int) job.tstride, job.qlen, job.tlen, job.h0, p, o, ncell);
            out[id] = o;
        }
    }
    if (cells) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) ncell += __shfl_xor_sync(0xffffffffu, ncell, d);
        if ((threadIdx.x & 31) == 0 && ncell) atomicAdd(cells, ncell);
    }
}

// ---------------------------------------------------------------------------------------------
// Two jobs per thread (bsw_pair.cuh): consecutive jobs of the sorted pair class share a thread, job A in the low
// halves, job B in the high halves.  Shared memory: packed state {H_A, E_A, H_B, E_B} one word per column
// [column][thread], then the PRMT selectors of the query pair, 16 bit per column [column][thread].
// ---------------------------------------------------------------------------------------------
template <int NTHR>                     // compile-time strides: the unrolled cell loop addresses columns as [base + immediate]
struct PairMemShared {
    unsigned st_base, sel_base;         // shared-window byte addresses of the thread's column 0 (state words, selectors)
    static constexpr unsigned st_stride = NTHR * 4u, sel_stride = NTHR * 2u;
    __device__ __forceinline__ uint32_t ld(int j) const {
        uint32_t w; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(st_base + (unsigned) j * st_stride)); return w;
    }
    __device__ __forceinline__ void st(int j, uint32_t w) const {
        asm volatile("st.shared.u32 [%0], %1;" :: "r"(st_base + (unsigned) j * st_stride), "r"(w) : "memory");
    }
    __device__ __forceinline__ uint32_t ld_half(int j, int l) const {
        uint16_t w; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(w) : "r"(st_base + (unsigned) j * st_stride + 2u * (unsigned) l)); return (uint32_t) w;
    }
    __device__ __forceinline__ void st_half(int j, int l, uint32_t v) const {
        asm volatile("st.shared.u16 [%0], %1;" :: "r"(st_base + (unsigned) j * st_stride + 2u * (unsigned) l), "h"((uint16_t) v) : "memory");
    }
    __device__ __forceinline__ uint32_t sel(int j) const {
        uint16_t w; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(w) : "r"(sel_base + (unsigned) j * sel_stride)); return (uint32_t) w;
    }
    __device__ __forceinline__ void set_sel(int j, uint32_t v) const {
        asm volatile("st.shared.u16 [%0], %1;" :: "r"(sel_base + (unsigned) j * sel_stride), "h"((uint16_t) v) : "memory");
    }
};

template <int NTHR>
__global__ void __launch_bounds__(NTHR)
bsw_pair_kernel(const BswJob *__restrict__ jobs, const int32_t *__restrict__ perm, const int32_t *__restrict__ class_off,
                int cls, BswOut *__restrict__ out, const uint8_t *__restrict__ tbase, const uint8_t *__restrict__ qbase,
                BswParams p, int W, unsigned long long *cells)
{
    extern __shared__ uint32_t sh[];
    const int first = class_off[cls], last = class_off[cls + 1];
    constexpr int nthr = NTHR;
    PairMemShared<NTHR> mem;
    mem.st_base = (unsigned) __cvta_generic_to_shared(sh) + threadIdx.x * 4u;
    mem.sel_base = (unsigned) __cvta_generic_to_shared(sh) + (unsigned) W * nthr * 4u + threadIdx.x * 2u;
    unsigned long long ncell = 0;
    for (int blk = blockIdx.x; first + 2 * blk * nthr < last; blk += gridDim.x) {      // persistent CTAs: long jobs first
        const int g = first + 2 * (blk * nthr + threadIdx.x);
        if (g < last) {
            const int nj = g + 1 < last ? 2 : 1;
            const int idA = perm[g], idB = nj == 2 ? perm[g + 1] : idA;
            const BswJob ja = jobs[idA], jb = jobs[idB];
            const int qlen[2] = {ja.qlen, nj == 2 ? jb.qlen : 0}, tlen[2] = {ja.tlen, nj == 2 ? jb.tlen : 0}, h0[2] = {ja.h0, nj == 2 ? jb.h0 : 0};
            const uint8_t *qa = qbase + ja.qoff, *qb = qbase + jb.qoff;
            const int qmax = qlen[0] > qlen[1] ? qlen[0] : qlen[1];
            for (int j = 0; j <= qmax; ++j) {
                const int ba = j < qlen[0] ? (int) qa[(long long) j * ja.qstride] : 0, bb = j < qlen[1] ? (int) qb[(long long) j * jb.qstride] : 0;
                mem.set_sel(j, p2_selector(ba & 3, bb & 3));
            }
            BswOut o[2];
            bsw_pair_extend(mem, tbase + ja.toff, (int) ja.tstride, tbase + jb.toff, (int) jb.tstride, qlen, tlen, h0, nj, p, o, ncell);
            out[idA] = o[0];
            if (nj == 2) out[idB] = o[1];
        }
    }
    if (cells) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) ncell += __shfl_xor_sync(0xffffffffu, ncell, d);
        if ((threadIdx.x & 31) == 0 && ncell) atomicAdd(cells, ncell);
    }
}

// ---------------------------------------------------------------------------------------------
// Warp-per-job kernel for long queries (the wide class: qlen > 1024 or 32-bit scores; long reads).
// A row of the band (<= 2w+1 columns) is split over the 32 lanes, CMAX columns per lane.  F, the only state
// that runs along the row, depends on M(k), k < j only:
//     F(j) = max(0, max_{beg<=k<j} (max(M(k) - oe_ins, 0) - (j-1-k) e_ins))
// so one exclusive max-scan per row (5 shuffles) replaces the sequential sweep; everything else is per column.
// State {H(i-1,j-1), E(i,j)} lives in a per-warp circular buffer of WCAP >= 2w+8 columns in shared memory;
// columns the band has never reached are initialised on demand with the first-row values, which reproduces the
// reference's "stale eh[] entries" exactly (tests/host_emul/bsw_rowscan.cpp is the CPU model of this kernel).
// ---------------------------------------------------------------------------------------------
#define BSWW_WARPS 4
template <int CMAX>
__global__ void __launch_bounds__(BSWW_WARPS * 32)
bsw_warp_kernel(const BswJob *__restrict__ jobs, const int32_t *__restrict__ perm, const int32_t *__restrict__ class_off,
                BswOut *__restrict__ out, const uint8_t *__restrict__ tbase, const uint8_t *__restrict__ qbase, BswParams p,
                int *next_job, unsigned long long *cells)
{
    constexpr int WCAP = 32 * CMAX + 8;
    __shared__ int shH[BSWW_WARPS][WCAP], shE[BSWW_WARPS][WCAP];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int *H = shH[wid], *E = shE[wid];
    const int first = class_off[BSW_NCLASS], last = class_off[BSW_NCLASS + 1];
    const int oe_del = p.o_del + p.e_del, oe_ins = p.o_ins + p.e_ins, e_del = p.e_del, e_ins = p.e_ins;
    const int NEG = -(1 << 29);
    unsigned long long ncell = 0;
    for (;;) {
        int g = 0;
        if (lane == 0) g = first + atomicAdd(next_job, 1);
        g = __shfl_sync(0xffffffffu, g, 0);
        if (g >= last) break;
        const int id = perm[g];
        const BswJob job = jobs[id];
        const uint8_t *qp = qbase + job.qoff, *tp = tbase + job.toff;
        const int qlen = job.qlen, tlen = job.tlen, h0 = job.h0;
        int w = p.w;
        {
            unsigned t1 = ((unsigned) (qlen * p.a) + (unsigned) (p.end_bonus - p.o_ins)) & 0xFFFFu;
            int max_ins = (int) (t1 / (unsigned) e_ins) + 1; if (max_ins < 1) max_ins = 1;
            unsigned t2 = ((unsigned) (qlen * p.a) + (unsigned) (p.end_bonus - p.o_del)) & 0xFFFFu;
            int max_del = (int) (t2 / (unsigned) e_del) + 1; if (max_del < 1) max_del = 1;
            if (w > max_ins) w = max_ins;
            if (w > max_del) w = max_del;
        }
        const int zthr = bsw_quirk(qlen, tlen, h0, p).zthr;      // (never the 8-bit class here: 16-bit threshold, no guard)
        const bool packed_key = qlen < 65536 && (long long) h0 + (long long) (qlen < tlen ? qlen : tlen) * p.a < 32768;
        // the launcher guarantees 2*w+2 <= 32*CMAX for this instantiation
        int max_init = -1;
        int best = h0, best_i = -1, best_j = -1, best_ie = -1, gscore = -1, max_off = 0;
        int beg = 0, end = qlen;
        for (int i = 0; i < tlen; ++i) {
            if (beg < i - w) beg = i - w;
            if (end > i + w + 1) end = i + w + 1;
            if (end > qlen) end = qlen;
            // first visit of columns (max_init, end]: first-row values  H(-1, j-1), E = 0
            for (int j = max_init + 1 + lane; j <= end; j += 32) {
                int v = j == 0 ? h0 : h0 - oe_ins - (j - 1) * e_ins;
                H[j % WCAP] = v > 0 ? v : 0; E[j % WCAP] = 0;
            }
            if (end > max_init) max_init = end;
            __syncwarp();
            int h1_init = 0;
            if (beg == 0) { h1_init = h0 - (p.o_del + e_del * (i + 1)); if (h1_init < 0) h1_init = 0; }
            const int n = end - beg;
            const int c = (n + 31) >> 5;
            const int tb = tp[(long long) i * job.tstride];
            const int j0 = beg + lane * c;
            int Mr[CMAX], Er[CMAX], Pl[CMAX];
            int run = NEG;
#pragma unroll
            for (int k = 0; k < CMAX; ++k) {
                const int j = j0 + k;
                Mr[k] = 0; Er[k] = 0; Pl[k] = NEG;
                if (k < c && j < end) {
                    const int hd = H[j % WCAP];
                    Er[k] = E[j % WCAP];
                    const int qb = qp[(long long) j * job.qstride];
                    const int s = (qb > 3 || tb > 3) ? -1 : (qb == tb ? p.a : -p.b);
                    const int m = hd ? hd + s : 0;
                    Mr[k] = m;
                    Pl[k] = run;
                    run = max(run, max(m - oe_ins, 0) + j * e_ins);
                }
            }
            // exclusive max-scan of the lane aggregates
            int incl = run;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { int o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl = max(incl, o); }
            int lp = __shfl_up_sync(0xffffffffu, incl, 1); if (lane == 0) lp = NEG;
            __syncwarp();
            // finish the cells, write the next row's state
            int lm = -1, lmj = -1, hlast = 0;                // (m, mj) per lane: 32-bit scores do not fit one packed key
#pragma unroll
            for (int k = 0; k < CMAX; ++k) {
                const int j = j0 + k;
                if (k < c && j < end) {
                    const int P = max(lp, Pl[k]);
                    int f = P - (j - 1) * e_ins; if (f < 0 || P == NEG) f = 0;
                    const int h = max(max(Mr[k], Er[k]), f);
                    E[j % WCAP] = max(Er[k] - e_del, max(Mr[k] - oe_del, 0));
                    if (k > 0) H[j % WCAP] = hlast;           // H(i, j-1) = h of the previous column of this lane
                    hlast = h;
                    if (h >= lm) { lm = h; lmj = j; }
                }
            }
            // first column of each lane takes the last h of the previous lane (or h1_init at column beg)
            const int ncols_lane = max(0, min(c, end - j0));
            int carry = __shfl_up_sync(0xffffffffu, hlast, 1);
            if (ncols_lane > 0) H[j0 % WCAP] = (lane == 0) ? h1_init : carry;
            // h1 = h of column end-1 (owner: lane (n-1)/c), H[end] = h1, E[end] = 0
            int h1 = h1_init;
            if (n > 0) h1 = __shfl_sync(0xffffffffu, hlast, (n - 1) / c);
            if (lane == 0) { H[end % WCAP] = h1; E[end % WCAP] = 0; }
            ncell += (lane == 0 && n > 0) ? (unsigned) n : 0u;
            // row maximum: largest h, among equals the largest column.  Scores below 2^15 and columns below 2^16 (every long-read job with the
            // default scoring) pack into one key and one REDUX instruction; otherwise ten shuffles
            int m = lm, mj = lmj;
            if (packed_key) {
                const int kmax = __reduce_max_sync(0xffffffffu, lm < 0 ? -1 : ((lm << 16) | lmj));
                m = kmax < 0 ? -1 : kmax >> 16; mj = kmax < 0 ? -1 : (kmax & 0xFFFF);
            } else {
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) {
                    const int om = __shfl_xor_sync(0xffffffffu, m, d), oj = __shfl_xor_sync(0xffffffffu, mj, d);
                    if (om > m || (om == m && oj > mj)) { m = om; mj = oj; }
                }
            }
            if (m < 0) { m = 0; mj = -1; }
            __syncwarp();
            if (end == qlen) {
                if (h1 >= gscore) best_ie = i;
                if (h1 > gscore) gscore = h1;
            }
            if (m == 0) break;
            if (m > best) {
                best = m; best_i = i; best_j = mj;
                int dd = mj - i; dd = dd < 0 ? -dd : dd;
                if (dd > max_off) max_off = dd;
                if (0 > zthr) break;
            } else {
                const int di = i - best_i, dj = mj - best_j;
                const int pen = di > dj ? di - dj : dj - di;
                if (best - m - pen > zthr) break;
            }
            // shrink the band to the non-zero support of the row just written
            int fz = end, lz = beg - 1;                       // first / last non-zero column in [beg, end]
            for (int j = beg + lane; j <= end; j += 32) {
                if ((H[j % WCAP] | E[j % WCAP]) != 0) { if (j < end && j < fz) fz = j; if (j > lz) lz = j; }
            }
            fz = __reduce_min_sync(0xffffffffu, fz);
            lz = __reduce_max_sync(0xffffffffu, lz);
            if (lz < fz) lz = fz - 1;                          // (all zero: cannot happen after m > 0; scalar semantics anyway)
            beg = fz;                                          // == end when the whole row is zero
            end = lz + 2 < qlen ? lz + 2 : qlen;
            __syncwarp();
        }
        if (lane == 0) {
            BswOut o; o.score = best; o.qle = best_j + 1; o.tle = best_i + 1; o.gtle = best_ie + 1; o.gscore = gscore; o.max_off = max_off;
            out[id] = o;
        }
        __syncwarp();
    }
    if (cells && lane == 0 && ncell) atomicAdd(cells, ncell);
}

// jobs whose scores need 32 bits or whose query does not fit the shared-memory classes:
// state in a private global-memory stripe (correctness path for the rare scalar class,
// reference src/bwamem.cpp:2310; long reads get the warp-per-job kernel in a later round).
__global__ void __launch_bounds__(64)
bsw_wide_kernel(const BswJob *__restrict__ jobs, const int32_t *__restrict__ perm, const int32_t *__restrict__ class_off,
                BswOut *__restrict__ out, const uint8_t *__restrict__ tbase, const uint8_t *__restrict__ qbase, BswParams p,
                int2 *state, const long long *state_off, unsigned long long *cells)
{
    const int first = class_off[BSW_NCLASS], last = class_off[BSW_NCLASS + 1];
    for (int g = first + blockIdx.x * blockDim.x + threadIdx.x; g < last; g += gridDim.x * blockDim.x) {
        const int id = perm[g];
        const BswJob job = jobs[id];
        GmemWide st; st.base = state + state_off[g - first];
        QGmem qf; qf.ptr = qbase + job.qoff; qf.stride = job.qstride;
        BswOut o; unsigned long long ncell = 0;
        bsw_extend_one(st, qf, tbase + job.toff, (int) job.tstride, job.qlen, job.tlen, job.h0, p, o, ncell);
        out[id] = o;
        if (cells && ncell) atomicAdd(cells, ncell);
    }
}

// exclusive prefix of (qlen+2) over the wide class, single thread block (the class is tiny)
__global__ void bsw_wide_off_kernel(const BswJob *jobs, const int32_t *perm, const int32_t *class_off, long long *state_off,
                                    long long *total) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int first = class_off[BSW_NCLASS], last = class_off[BSW_NCLASS + 1];
    long long s = 0;
    for (int g = first; g < last; ++g) { state_off[g - first] = s; s += jobs[perm[g]].qlen + 2; }
    *total = s;
}

size_t bsw_scratch_bytes(int n) {
    size_t cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (uint32_t *) nullptr, (uint32_t *) nullptr, (int32_t *) nullptr,
                                    (int32_t *) nullptr, n > 0 ? n : 1);
    size_t per = ((size_t) (n > 0 ? n : 1) * 4 + 255) / 256 * 256;
    return 4 * per + 512 + 256 + ((cub_bytes + 255) / 256 * 256) + 256;
}

struct BswWideScratch { int2 *state; long long *state_off; long long *total; size_t cap_words; size_t cap_jobs; };
#define BSW_MAX_DEV 64
static BswWideScratch g_wide_dev[BSW_MAX_DEV];      // per device ordinal (a process may hold one context per GPU), zero-initialised

int bsw_launch_with_scratch(bm2_ctx *ctx_for_error, cudaStream_t stream, const BswJob *d_jobs, BswOut *d_out, int n,
                            const uint8_t *d_tbase, const uint8_t *d_qbase, const BswParams &prm,
                            unsigned long long *d_cells, void *scratch, size_t scratch_bytes, int wide_possible)
{
    if (n <= 0) return 0;
    if (scratch_bytes < bsw_scratch_bytes(n)) { bm2_set_error(ctx_for_error, "bsw: scratch too small"); return 1; }
    size_t per = ((size_t) n * 4 + 255) / 256 * 256;
    char *s = (char *) scratch;
    uint32_t *keys_in = (uint32_t *) s; s += per;
    uint32_t *keys_out = (uint32_t *) s; s += per;
    int32_t *idx_in = (int32_t *) s; s += per;
    int32_t *idx_out = (int32_t *) s; s += per;
    int32_t *class_cnt = (int32_t *) s; s += 512;       // [0, BSW_NALL) job counts; 48: job queue of the warp kernel; 64 + c: job queue of class c
    int32_t *class_off = (int32_t *) s; s += 256;
    void *cub_tmp = s;
    size_t cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, keys_in, keys_out, idx_in, idx_out, n);

    BM2_CUDA_OK(cudaMemsetAsync(class_cnt, 0, 512, stream));
    // Two-jobs-per-thread kernel (bsw_pair.cuh): bit-exact, but slower than the thread-per-job kernel in an A/B (the lanes of
    // a warp spend the pre/post column segments of their pairs apart), so it is off unless BM2_BSW_PAIR=1 asks for it (experiments, tests).
    const char *pair_env = getenv("BM2_BSW_PAIR");
    const int pair_ok = (pair_env && pair_env[0] == '1' && p2_params_ok(prm)) ? 1 : 0;
    bsw_keys_kernel<<<(n + 255) / 256, 256, 0, stream>>>(d_jobs, n, prm.a, pair_ok, d_qbase, keys_in, idx_in, class_cnt);
    BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, keys_in, keys_out, idx_in, idx_out, n, 0, 32, stream));
    bsw_class_off_kernel<<<1, 32, 0, stream>>>(class_cnt, class_off);

    int dev = 0, n_sm = 132;
    BM2_CUDA_OK(cudaGetDevice(&dev));
    BM2_CUDA_OK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    if (dev < 0 || dev >= BSW_MAX_DEV) { bm2_set_error(ctx_for_error, "bsw: device ordinal out of range"); return 1; }
    static bool attr_set_dev[BSW_MAX_DEV];          // the attribute is per device: one flag per ordinal
    static std::mutex attr_mu;                      // launches come from several host threads (sub-batch lanes, contexts)
    std::unique_lock<std::mutex> attr_lock(attr_mu);
    bool &attr_set = attr_set_dev[dev];
    if (!attr_set) {   // one function, several dynamic sizes: raise the limit once per device
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_thread_kernel<SmemPacked>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_thread_kernel<SmemPacked8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_col2_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_col2_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_col2_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_pair_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_pair_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_pair_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        BM2_CUDA_OK(cudaFuncSetAttribute(bsw_pair_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        attr_set = true;
    }
    attr_lock.unlock();
    // Two columns of one job per packed instruction (bsw_col2.cuh) for the 8-bit-score classes; BM2_BSW_COL2=0 keeps the
    // one-cell-per-instruction kernel for them (A/B measurements, tests of both kernels).
    const char *col2_env = getenv("BM2_BSW_COL2");
    const int col2_ok = (!(col2_env && col2_env[0] == '0') && c2_params_ok(prm)) ? 1 : 0;
    // shared memory the persistent CTAs of one launch may occupy per SM: the rest stays free for the kernels of the other
    // sub-batches in flight (latency-bound SMEM / chain / tail kernels co-resident with the ALU-bound extension)
    size_t smem_budget = 227 * 1024;
    if (const char *e = getenv("BM2_BSW_SMEM_KB")) { int kb = atoi(e); if (kb >= 48 && kb <= 227) smem_budget = (size_t) kb * 1024; }
    int max_ctas = 16;            // ... and a plain cap on its CTAs per SM (warp slots / registers left for the others)
    if (const char *e = getenv("BM2_BSW_MAX_CTAS")) { int v = atoi(e); if (v >= 1 && v <= 16) max_ctas = v; }
    for (int c = 0; c < BSW_NCLASS; ++c) {
        const int bound = h_class_bound[c >> 1];
        const int is16 = c & 1;
        const int W = bound + 2;
        const int QW = bound / 8 + 1;            // +1: cursor(beg) may touch word qlen>>3 when beg == qlen
        const size_t per_thread = (size_t) W * (is16 ? 4 : 2) + (size_t) QW * 4 + 4;
        // threads per CTA: as many as fit ~112 KB (2 CTAs/SM), capped at BSW_THREADS
        int nthr = BSW_THREADS;
        while (nthr > 32 && per_thread * nthr > 112 * 1024) nthr >>= 1;
        const size_t smem = per_thread * nthr;
        if (smem > 227 * 1024) { bm2_set_error(ctx_for_error, "bsw: class does not fit shared memory"); return 1; }
        int ctas_per_sm = (int) (smem_budget / (smem + 1024)); if (ctas_per_sm < 1) ctas_per_sm = 1; if (ctas_per_sm > max_ctas) ctas_per_sm = max_ctas;
        int nblk = (n + nthr - 1) / nthr;
        const int cap_blk = n_sm * ctas_per_sm;
        if (nblk > cap_blk) nblk = cap_blk;
        if (col2_ok && !is16 && bound <= 256) {
            // two columns per packed instruction (bsw_col2.cuh): state 2 B per column in pair words, selectors 1 B per column
            const int NP = (W + 1) / 2;                       // state words: pairs over columns 0 .. bound + 1; selectors: 2 B per pair
            // threads per CTA: the size that keeps the most threads resident per SM (shared memory is what limits this kernel's
            // occupancy: 6 B per column pair and thread; 64- or 96-thread CTAs waste less of the 227 KB than 128-thread ones)
            // Band shrink of a row (first / last column with a non-zero state): 0 = scans over shared memory; 1 = the two columns at either edge
            // from the words just written, then the scans: slower than 0 in an A/B (the extra branches cost more
            // than the loads they save); 2 (default) = only the ONE column at either edge from registers, then the scans (the fastest of the
            // three in an A/B).  BM2_BSW_REGSHRINK selects (A/B); BM2_BSW_UNROLL8=1: the scans with the pair loop unrolled x8 (no gain).
            const char *rs_env = getenv("BM2_BSW_REGSHRINK");
            int reg_shrink = 3;
            if (rs_env && rs_env[0] == '0') reg_shrink = 0; else if (rs_env && rs_env[0] == '1') reg_shrink = 1;
            if (const char *e = getenv("BM2_BSW_UNROLL8")) { if (e[0] == '1') reg_shrink = 2; }
            const char *dyn_env = getenv("BM2_BSW_DYN");
            const int dyn = (dyn_env && dyn_env[0] == '0') ? 0 : 1;           // per-warp job counters: class_cnt[64 + c], zeroed with class_cnt above
            int nthr2 = 128, best_res = 0, best_cps = 1;
            int t_lo = 128, t_hi = 128;           // 128-thread CTAs: faster than 96 / 64 and than the most-resident-threads choice in an A/B
            if (const char *e = getenv("BM2_BSW_NTHR")) { const int v = atoi(e); if (v == 64 || v == 96 || v == 128) t_lo = t_hi = v; }      // A/B measurements
            for (int t = t_hi; t >= t_lo; t -= 32) {
                int cps = (int) (smem_budget / ((size_t) NP * 6 * t + 1024)); if (cps < 1) cps = 1; if (cps > max_ctas * (128 / t)) cps = max_ctas * (128 / t);
                if (cps > 32) cps = 32;
                if (cps * t > best_res) { best_res = cps * t; nthr2 = t; best_cps = cps; }
            }
            const size_t smem2 = (size_t) NP * 6 * nthr2;
            int nb = (n + nthr2 - 1) / nthr2; if (nb > n_sm * best_cps) nb = n_sm * best_cps;
#define BM2_COL2_LAUNCH(T) bsw_col2_kernel<T><<<nb, T, smem2, stream>>>(d_jobs, idx_out, class_off, c, d_out, d_tbase, d_qbase, prm, NP, d_cells, reg_shrink, dyn ? class_cnt + 64 + c : nullptr)
            if (nthr2 == 128) BM2_COL2_LAUNCH(128); else if (nthr2 == 96) BM2_COL2_LAUNCH(96); else BM2_COL2_LAUNCH(64);
#undef BM2_COL2_LAUNCH
            continue;
        }
        if (is16) bsw_thread_kernel<SmemPacked><<<nblk, nthr, smem, stream>>>(d_jobs, idx_out, class_off, c, d_out, d_tbase, d_qbase, prm, W, d_cells);
        else bsw_thread_kernel<SmemPacked8><<<nblk, nthr, smem, stream>>>(d_jobs, idx_out, class_off, c, d_out, d_tbase, d_qbase, prm, W, d_cells);
    }
    for (int c = 0; pair_ok && c < BSW_NPAIR; ++c) {
        const int W = h_class_bound[c] + 2;
        const size_t per_thread = (size_t) W * 6;
        // threads per CTA: the size that keeps the most threads resident per SM
        int nthr = 32, best_res = 0;
        for (int t = 128; t >= 32; t -= 32) {
            const int ctas = (int) ((227 * 1024) / (per_thread * t + 1024));
            const int res = (ctas > 16 ? 16 : ctas) * t;
            if (res > best_res) { best_res = res; nthr = t; }
        }
        const size_t smem = per_thread * nthr;
        int ctas_per_sm = (int) ((227 * 1024) / (smem + 1024)); if (ctas_per_sm < 1) ctas_per_sm = 1; if (ctas_per_sm > 16) ctas_per_sm = 16;
        int nblk = (n + 2 * nthr - 1) / (2 * nthr);
        if (nblk > n_sm * ctas_per_sm) nblk = n_sm * ctas_per_sm;
#define BM2_PAIR_LAUNCH(T) bsw_pair_kernel<T><<<nblk, T, smem, stream>>>(d_jobs, idx_out, class_off, BSW_PAIR0 + c, d_out, d_tbase, d_qbase, prm, W, d_cells)
        if (nthr == 128) BM2_PAIR_LAUNCH(128); else if (nthr == 96) BM2_PAIR_LAUNCH(96); else if (nthr == 64) BM2_PAIR_LAUNCH(64); else BM2_PAIR_LAUNCH(32);
#undef BM2_PAIR_LAUNCH
    }
    if (wide_possible) {
        int *next_job = class_cnt + 48;                    // zeroed with class_cnt above
        const int wblocks = n_sm * 4;
        if (2 * prm.w + 2 <= 32 * 7)       // 72 registers, 7.4 KB of shared memory per CTA: seven CTAs of four warps fit an SM (the jobs come from a queue)
            bsw_warp_kernel<7><<<n_sm * 7, BSWW_WARPS * 32, 0, stream>>>(d_jobs, idx_out, class_off, d_out, d_tbase, d_qbase, prm, next_job, d_cells);
        else if (2 * prm.w + 2 <= 32 * 13)
            bsw_warp_kernel<13><<<wblocks, BSWW_WARPS * 32, 0, stream>>>(d_jobs, idx_out, class_off, d_out, d_tbase, d_qbase, prm, next_job, d_cells);
        else if (2 * prm.w + 2 <= 32 * 32)
            bsw_warp_kernel<32><<<wblocks, BSWW_WARPS * 32, 0, stream>>>(d_jobs, idx_out, class_off, d_out, d_tbase, d_qbase, prm, next_job, d_cells);
        else {
        // very wide bands: state in global memory, one job per thread; the class size is needed on the host.  The scratch is
        // shared by all contexts of the process: one launch of this (rare) path at a time, held until the kernel has finished.
        static std::mutex wide_mu;
        std::lock_guard<std::mutex> wide_lock(wide_mu);
        BswWideScratch &g_wide = g_wide_dev[dev];
        int32_t h_off[2];
        BM2_CUDA_OK(cudaMemcpyAsync(h_off, class_off + BSW_NCLASS, 8, cudaMemcpyDeviceToHost, stream));
        BM2_CUDA_OK(cudaStreamSynchronize(stream));
        int nw = h_off[1] - h_off[0];
        if (nw > 0) {
            if (g_wide.cap_jobs < (size_t) nw) {
                if (g_wide.state_off) cudaFree(g_wide.state_off);
                if (!g_wide.total) BM2_CUDA_OK(cudaMalloc(&g_wide.total, 8));
                BM2_CUDA_OK(cudaMalloc(&g_wide.state_off, (size_t) nw * 8));
                g_wide.cap_jobs = nw;
            }
            bsw_wide_off_kernel<<<1, 32, 0, stream>>>(d_jobs, idx_out, class_off, g_wide.state_off, g_wide.total);
            long long total = 0;
            BM2_CUDA_OK(cudaMemcpyAsync(&total, g_wide.total, 8, cudaMemcpyDeviceToHost, stream));
            BM2_CUDA_OK(cudaStreamSynchronize(stream));
            if (g_wide.cap_words < (size_t) total) {
                if (g_wide.state) cudaFree(g_wide.state);
                BM2_CUDA_OK(cudaMalloc(&g_wide.state, (size_t) total * sizeof(int2)));
                g_wide.cap_words = total;
            }
            int blocks = (nw + 63) / 64; if (blocks > n_sm * 8) blocks = n_sm * 8;
            bsw_wide_kernel<<<blocks, 64, 0, stream>>>(d_jobs, idx_out, class_off, d_out, d_tbase, d_qbase, prm, g_wide.state,
                                                       g_wide.state_off, d_cells);
            BM2_CUDA_OK(cudaStreamSynchronize(stream));
        }
        }
    }
    BM2_CUDA_OK(cudaGetLastError());
    return 0;
}

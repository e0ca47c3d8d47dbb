// fmi_build.cu — bm2_index_build: the second step of bm2_index, FMI_search::build_index + build_fm_index (reference src/FMI_search.cpp:83-302,
// :306-382), on the GPU.  From <prefix>.pac it writes <prefix>.0123 (the text: forward then reverse complement, one code per byte) and
// <prefix>.bwt.2bit.64 (N = n + 1, count[5], CP_OCC per 64 rows, every 8th row's SA as sa_ms int8 + sa_ls uint32, the sentinel row), the
// layout bm2_index_load reads and index_build.py writes.
//
// The suffix array is index_build.py's algorithm in a layout that keeps about 5.25 bytes per text position on the device: the text at 2 bits
// per base and the inverse suffix array (ISA, rank = the slot of the suffix's tie group in SA order) as 40-bit values.  The SA itself is
// never held; it is scattered from the ISA one window of rows at a time.
//   pass 1   histogram of the first b bases of every suffix; bucket groups that fit the work buffers, each compacted by a scan over the text,
//            keyed by its 31-mer and radix sorted; ISA = the global start of each suffix's tie group.  The positions of tied suffixes, in SA
//            order, form the unresolved list (on the device, or in host memory when it does not fit).
//   rounds   Larsson-Sadakane doubling over the unresolved list in pieces that end at tie-group boundaries: key2 = ISA[p + h] (fmi_key2),
//            one radix sort on (group ordinal in the piece, key2), new group starts written to the ISA, still-tied positions kept in order.
//            Inside a piece all gathers come before the writes.  A piece may read ranks that an earlier piece of the same round has already
//            refined; refined ranks stay consistent with the true order, so the result is the same (the comment in index_build.py).
//   emit     per window of rows: SA[ISA[p] + 1 - r0] = p over all p, every slot checked to be written exactly once; then the BWT characters,
//            CP_OCC entries with their running counts and every 8th row's SA, written at their offsets in a temporary file that is renamed
//            only when every window passed.
#include "bm2_b200.h"
#include "fmi_device.cuh"
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

struct bm2_ctx;
void bm2_set_error(bm2_ctx *ctx, const std::string &msg);

namespace {

constexpr uint64_t EMPTY = ~0ull;
constexpr int TPB = 256;

unsigned grid_for(int64_t n) { return (unsigned) std::max<int64_t>(1, std::min<int64_t>((n + TPB - 1) / TPB, (int64_t) 1 << 20)); }

struct Err : std::runtime_error { using std::runtime_error::runtime_error; };
#define FMI_CK(x) do { const cudaError_t e_ = (x); if (e_ != cudaSuccess) throw Err(std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)

// ---- kernels ----

// the 2-bit text of fwd + reverse complement from the .pac bytes (first base in the top bits); zero past n
__global__ void pack_text_kernel(const uint8_t *pac, int64_t l_pac, int64_t n, uint64_t *w, int64_t n_words) {
    for (int64_t q = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; q < n_words; q += (int64_t) gridDim.x * blockDim.x) {
        uint64_t v = 0;
        for (int j = 0; j < 32; ++j) {
            const int64_t i = q * 32 + j;
            uint32_t c = 0;
            if (i < l_pac) c = pac[i >> 2] >> ((~i & 3) << 1) & 3;
            else if (i < n) { const int64_t f = n - 1 - i; c = 3 - (pac[f >> 2] >> ((~f & 3) << 1) & 3); }
            v |= (uint64_t) c << (62 - 2 * j);
        }
        w[q] = v;
    }
}

__global__ void unpack_text_kernel(const uint64_t *w, int64_t i0, int64_t m, uint8_t *out) {
    for (int64_t j = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (int64_t) gridDim.x * blockDim.x) out[j] = (uint8_t) fmi_base(w, i0 + j);
}

__global__ void hist_kernel(const uint64_t *w, int64_t n, int b, unsigned long long *hist) {
    for (int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t) gridDim.x * blockDim.x) atomicAdd(&hist[fmi_bucket(w, p, b)], 1ull);
}

// positions whose bucket is in [lo, hi), with their keys; warp-aggregated slots (the order is free: the sort and the ranks ignore it)
__global__ void select_kernel(const uint64_t *w, int64_t n, int b, uint32_t lo, uint32_t hi, uint64_t *pos, uint64_t *key, unsigned long long *cnt) {
    const int lane = threadIdx.x & 31;
    for (int64_t b0 = (int64_t) blockIdx.x * blockDim.x; b0 < n; b0 += (int64_t) gridDim.x * blockDim.x) {
        const int64_t p = b0 + threadIdx.x;
        uint64_t k = 0; bool in = false;
        if (p < n) { k = fmi_kmer(w, p); const uint32_t bk = (uint32_t) (k >> (62 - 2 * b)); in = bk >= lo && bk < hi; }
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (!m) continue;
        unsigned long long at = 0;
        if (lane == 0) at = atomicAdd(cnt, (unsigned long long) __popc(m));
        at = __shfl_sync(0xffffffffu, at, 0);
        if (in) { const unsigned long long j = at + __popc(m & ((1u << lane) - 1)); pos[j] = (uint64_t) p; key[j] = k; }
    }
}

// start[j] = j at the first of each run of equal keys, else 0 (a max-scan then gives every slot its run's start)
__global__ void run_start_kernel(const uint64_t *key, int m, int32_t *start) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) start[j] = (j == 0 || key[j] != key[j - 1]) ? j : 0;
}

// pass 1: ISA[pos] = base + the slot's run start; tied: the run has more than one slot
__global__ void p1_write_kernel(const uint64_t *pos, const int32_t *start, int m, uint64_t base, uint32_t *lo, uint8_t *hi, uint8_t *tied) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        fmi_put40(lo, hi, (int64_t) pos[j], base + (uint64_t) start[j]);
        const bool single = start[j] == j && (j + 1 == m || start[j + 1] == j + 1);
        tied[j] = !single;
    }
}

// a refinement piece, before the sort: group starts (flag) and their ranks, and the last group start of the loaded slots
__global__ void r_groups_kernel(const uint64_t *pos, int m, const uint32_t *lo, const uint8_t *hi, int32_t *flag, uint64_t *g, int *last_start) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const uint64_t gj = fmi_get40(lo, hi, (int64_t) pos[j]);
        const bool f = j == 0 || gj != fmi_get40(lo, hi, (int64_t) pos[j - 1]);
        flag[j] = f; g[j] = gj;
        if (f) atomicMax(last_start, j);
    }
}

// sort keys (group ordinal, key2); per ordinal, the group's rank and its first slot in the piece
__global__ void r_keys_kernel(const uint64_t *pos, const int32_t *flag, const int32_t *ord1, const uint64_t *g, int m, const uint32_t *lo,
                              const uint8_t *hi, int64_t n, int64_t h, int k2bits, uint64_t *key, uint64_t *gval, int32_t *gfirst) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const int o = ord1[j] - 1;
        if (flag[j]) { gval[o] = g[j]; gfirst[o] = j; }
        key[j] = (uint64_t) o << k2bits | fmi_key2(lo, hi, n, (int64_t) pos[j], h);
    }
}

// after the sort: new rank = the group's rank + (first slot of the equal-key run - the group's first slot); tied as in pass 1
__global__ void r_write_kernel(const uint64_t *key, const uint64_t *pos, const int32_t *start, int m, int k2bits, const uint64_t *gval,
                               const int32_t *gfirst, uint32_t *lo, uint8_t *hi, uint8_t *tied) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const int o = (int) (key[j] >> k2bits);
        fmi_put40(lo, hi, (int64_t) pos[j], gval[o] + (uint64_t) (start[j] - gfirst[o]));
        const bool single = start[j] == j && (j + 1 == m || key[j + 1] != key[j]);
        tied[j] = !single;
    }
}

// emit: SA[row - r0] = p for the rows of the window (row = ISA[p] + 1; row 0 is the suffix at n), counting slots written twice
__global__ void scatter_kernel(const uint32_t *lo, const uint8_t *hi, int64_t n, int64_t r0, int64_t r1, unsigned long long *sa, unsigned long long *dup) {
    for (int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t) gridDim.x * blockDim.x) {
        const int64_t r = (int64_t) fmi_get40(lo, hi, p) + 1;
        if (r >= r0 && r < r1 && atomicExch(&sa[r - r0], (unsigned long long) p) != EMPTY) atomicAdd(dup, 1ull);
    }
}

// emit: BWT characters of the window's rows (6 past the last row), every 8th row's SA, the sentinel row, slots never written
__global__ void rows_kernel(const uint64_t *w, const unsigned long long *sa, int64_t r0, int64_t m, int64_t n_rows, uint8_t *bw, int8_t *ms,
                            uint32_t *ls, long long *sentinel, unsigned long long *missing) {
    for (int64_t j = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (int64_t) gridDim.x * blockDim.x) {
        const int64_t r = r0 + j;
        if (r >= n_rows) { bw[j] = 6; continue; }
        const uint64_t s = sa[j];
        if (s == EMPTY) { atomicAdd(missing, 1ull); bw[j] = 6; continue; }
        bw[j] = fmi_bwt_char(w, s);
        if (s == 0) *sentinel = r;
        if ((r & 7) == 0) { ms[j >> 3] = (int8_t) (s >> 32 & 0xff); ls[j >> 3] = (uint32_t) s; }
    }
}

struct Cnt4 { long long c[4]; };
struct Cnt4Sum {
    __host__ __device__ Cnt4 operator()(const Cnt4 &a, const Cnt4 &b) const { Cnt4 r; for (int k = 0; k < 4; ++k) r.c[k] = a.c[k] + b.c[k]; return r; }
};

__global__ void blocks_kernel(const uint8_t *bw, int64_t nb, FmiCpOcc *cp, Cnt4 *cnt) {
    for (int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (int64_t) gridDim.x * blockDim.x) {
        const int64_t zero[4] = { 0, 0, 0, 0 };
        int64_t add[4];
        FmiCpOcc e;
        fmi_cp_entry(bw + b * 64, zero, &e, add);
        cp[b] = e;
        for (int k = 0; k < 4; ++k) cnt[b].c[k] = add[k];
    }
}

__global__ void run_counts_kernel(const Cnt4 *excl, Cnt4 carry, int64_t nb, FmiCpOcc *cp) {
    for (int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (int64_t) gridDim.x * blockDim.x)
        for (int k = 0; k < 4; ++k) cp[b].cp_count[k] = excl[b].c[k] + carry.c[k];
}

// ---- host driver ----

double secs() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
int bits_for(uint64_t v) { int b = 0; while (b < 64 && (v >> b)) ++b; return b; }

// device allocations with the running and peak total
struct Mem {
    std::map<void *, size_t> live; int64_t cur = 0, peak = 0;
    template <class T> T *get(size_t count, const char *what) {
        void *p = nullptr; const size_t bytes = std::max<size_t>(count * sizeof(T), 16);
        if (cudaMalloc(&p, bytes) != cudaSuccess) {
            cudaGetLastError();
            size_t fr = 0, tot = 0; cudaMemGetInfo(&fr, &tot);
            throw Err(std::string("cannot allocate ") + what + ": " + std::to_string(bytes) + " bytes needed, " + std::to_string(fr) + " bytes free");
        }
        live[p] = bytes; cur += (int64_t) bytes; peak = std::max(peak, cur);
        return (T *) p;
    }
    template <class T> void put(T *&p) { if (!p) return; auto it = live.find((void *) p); cur -= (int64_t) it->second; live.erase(it); cudaFree((void *) p); p = nullptr; }
    ~Mem() { for (auto &kv : live) cudaFree(kv.first); }
};

// the unresolved list: text positions of tied suffixes in SA order; on the device while it fits its share of the work budget, else in host memory
struct UList {
    Mem &mem; uint64_t *dev = nullptr; size_t dev_cap = 0; std::vector<uint64_t> host; bool on_host = false; size_t n = 0;
    UList(Mem &m, size_t cap) : mem(m), dev_cap(cap) { dev = mem.get<uint64_t>(cap, "the unresolved list"); }
    uint64_t *at(size_t i) { return on_host ? host.data() + i : dev + i; }
    void write(size_t i, const uint64_t *src, size_t cnt) {
        if (!on_host && i + cnt > dev_cap) {
            host.resize(std::max(i + cnt, n));
            FMI_CK(cudaMemcpy(host.data(), dev, n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
            mem.put(dev); on_host = true;
        }
        if (on_host && host.size() < i + cnt) host.resize(i + cnt);
        if (cnt) FMI_CK(cudaMemcpy(at(i), src, cnt * sizeof(uint64_t), cudaMemcpyDefault));
        n = std::max(n, i + cnt);
    }
};

struct CubTemp {
    Mem &mem; void *p = nullptr; size_t bytes = 0;
    explicit CubTemp(Mem &m) : mem(m) {}
    void need(size_t b) { if (b > bytes) { char *q = (char *) p; mem.put(q); p = mem.get<char>(b, "sort scratch"); bytes = b; } }
};

void write_at(FILE *f, int64_t off, const void *p, size_t n, const std::string &path) {
    if (n == 0) return;
    if (fseeko(f, (off_t) off, SEEK_SET) != 0 || fwrite(p, 1, n, f) != n) throw Err("cannot write " + path);
}

void build(int device, const std::string &prefix, int64_t work_bytes, bm2_index_build_stats &st) {
    const double t0 = secs();
    FMI_CK(cudaSetDevice(device));
    // .pac -> l_pac (pac_seq_len, src/FMI_search.cpp:70-81)
    std::vector<uint8_t> pac;
    {
        FILE *f = fopen((prefix + ".pac").c_str(), "rb");
        if (!f) throw Err("cannot open " + prefix + ".pac");
        fseeko(f, 0, SEEK_END); const int64_t sz = (int64_t) ftello(f); fseeko(f, 0, SEEK_SET);
        pac.resize((size_t) std::max<int64_t>(sz, 0));
        const bool ok = sz >= 2 && fread(pac.data(), 1, (size_t) sz, f) == (size_t) sz;
        fclose(f);
        if (!ok) throw Err(prefix + ".pac is truncated");
    }
    const int64_t l_pac = ((int64_t) pac.size() - 2) * 4 + pac.back();
    if (l_pac <= 0 || pac.back() > 3) throw Err(prefix + ".pac is not a .pac file (bad trailer)");
    const int64_t n = 2 * l_pac, n_rows = n + 1;
    if (n >= ((int64_t) 1 << 33)) throw Err("the text is longer than 2^33 bases (8.6 G): past the 40-bit ranks and 64-bit sort keys of this builder");
    st.n = n;

    Mem mem;
    const int64_t n_words = n / 32 + 2;
    const int64_t persistent = n_words * 8 + n * 5;
    size_t free_b = 0, total_b = 0;
    FMI_CK(cudaMemGetInfo(&free_b, &total_b));
    const int64_t reserve = (int64_t) 1 << 30;      // the CUDA context and cub's own allocations
    if (work_bytes <= 0) work_bytes = std::min<int64_t>((int64_t) 16 << 30, (int64_t) free_b - persistent - reserve);
    // one slot of a group or piece: keys, positions (double buffers), two int32 scans, flags, the ordinal tables; sort scratch comes on top
    const int64_t per_slot = 8 * 4 + 4 * 2 + 1 + 8 + 4 + 8;
    const int64_t min_work = 64 * per_slot;
    if (persistent + std::max(work_bytes, min_work) > (int64_t) free_b)
        throw Err("the text and the inverse suffix array (" + std::to_string(persistent) + " bytes) and a minimal group (" + std::to_string(min_work) +
                  " bytes) do not fit: " + std::to_string(persistent + min_work) + " bytes needed, " + std::to_string(free_b) + " bytes free");
    work_bytes = std::max(work_bytes, min_work);

    // the text, on the device and written to .0123
    uint64_t *w = mem.get<uint64_t>((size_t) n_words, "the text");
    {
        uint8_t *d_pac = mem.get<uint8_t>(pac.size(), "the .pac bytes");
        FMI_CK(cudaMemcpy(d_pac, pac.data(), pac.size(), cudaMemcpyHostToDevice));
        pack_text_kernel<<<grid_for(n_words), TPB>>>(d_pac, l_pac, n, w, n_words);
        FMI_CK(cudaGetLastError());
        mem.put(d_pac);
        const std::string path = prefix + ".0123";
        FILE *f = fopen(path.c_str(), "wb");
        if (!f) throw Err("cannot write " + path);
        const int64_t chunk = std::min<int64_t>(n, std::max<int64_t>(work_bytes / 2, 1 << 16));
        uint8_t *d_b = mem.get<uint8_t>((size_t) chunk, "the .0123 chunk");
        std::vector<uint8_t> hb((size_t) chunk);
        for (int64_t i = 0; i < n; i += chunk) {
            const int64_t m = std::min(chunk, n - i);
            unpack_text_kernel<<<grid_for(m), TPB>>>(w, i, m, d_b);
            FMI_CK(cudaMemcpy(hb.data(), d_b, (size_t) m, cudaMemcpyDeviceToHost));
            if (fwrite(hb.data(), 1, (size_t) m, f) != (size_t) m) { fclose(f); throw Err("cannot write " + path); }
        }
        mem.put(d_b);
        if (fclose(f) != 0) throw Err("cannot write " + path);
    }
    uint32_t *isa_lo = mem.get<uint32_t>((size_t) n, "the inverse suffix array");
    uint8_t *isa_hi = mem.get<uint8_t>((size_t) n, "the inverse suffix array");
    const double t1 = secs();
    st.load_s = t1 - t0;

    // ---- pass 1 ----
    // slots per group: three quarters of the work budget; the rest holds the unresolved list on the device.  b: enough bucket bits that
    // the average bucket is a small part of a group
    int64_t cap = std::min<int64_t>(std::max<int64_t>(64, work_bytes * 3 / 4 / per_slot), n + 1);
    int b = 1;
    while (b < 12 && (n >> (2 * b)) * 16 > cap) ++b;
    std::vector<unsigned long long> hist((size_t) 1 << (2 * b));
    {
        unsigned long long *d_hist = mem.get<unsigned long long>(hist.size(), "the bucket histogram");
        FMI_CK(cudaMemset(d_hist, 0, hist.size() * 8));
        hist_kernel<<<grid_for(n), TPB>>>(w, n, b, d_hist);
        FMI_CK(cudaMemcpy(hist.data(), d_hist, hist.size() * 8, cudaMemcpyDeviceToHost));
        mem.put(d_hist);
    }
    // a tie group never spans buckets, so a bucket bigger than the budget's groups widens them (the peak shows it)
    const int64_t max_bucket = (int64_t) *std::max_element(hist.begin(), hist.end());
    cap = std::min<int64_t>(std::max<int64_t>(cap, max_bucket + 1), (int64_t) 1 << 30);
    if (max_bucket + 1 > cap) throw Err("a bucket of " + std::to_string(max_bucket) + " suffixes with one 31-mer prefix: past this builder's 2^30-slot groups");
    const int64_t u_bytes = std::max<int64_t>(work_bytes - cap * per_slot, 4096);
    UList U(mem, (size_t) std::min<int64_t>(u_bytes / 8, n));

    uint64_t *keyA = mem.get<uint64_t>((size_t) cap, "sort keys"), *keyB = mem.get<uint64_t>((size_t) cap, "sort keys");
    uint64_t *posA = mem.get<uint64_t>((size_t) cap, "positions"), *posB = mem.get<uint64_t>((size_t) cap, "positions");
    int32_t *i32A = mem.get<int32_t>((size_t) cap, "scans"), *i32B = mem.get<int32_t>((size_t) cap, "scans");
    uint8_t *flag = mem.get<uint8_t>((size_t) cap, "flags");
    uint64_t *gval = mem.get<uint64_t>((size_t) cap, "group ranks");
    int32_t *gfirst = mem.get<int32_t>((size_t) cap, "group slots");
    unsigned long long *d_cnt = mem.get<unsigned long long>(2, "counters");
    int *d_last = (int *) (d_cnt + 1);
    CubTemp tmp(mem);
    {
        size_t s1 = 0, s2 = 0, s3 = 0, s4 = 0;
        cub::DoubleBuffer<uint64_t> kb(keyA, keyB), vb(posA, posB);
        FMI_CK(cub::DeviceRadixSort::SortPairs(nullptr, s1, kb, vb, (int) cap));
        FMI_CK(cub::DeviceScan::InclusiveScan(nullptr, s2, i32A, i32B, cub::Max(), (int) cap));
        FMI_CK(cub::DeviceScan::InclusiveSum(nullptr, s3, i32A, i32B, (int) cap));
        FMI_CK(cub::DeviceSelect::Flagged(nullptr, s4, posA, flag, posB, d_cnt, (int) cap));
        tmp.need(std::max(std::max(s1, s2), std::max(s3, s4)));
    }
    auto select_tied = [&](const uint64_t *src, uint64_t *dst, int m) -> size_t {
        size_t tb = tmp.bytes;
        FMI_CK(cub::DeviceSelect::Flagged(tmp.p, tb, src, flag, dst, d_cnt, m));
        unsigned long long c = 0;
        FMI_CK(cudaMemcpy(&c, d_cnt, 8, cudaMemcpyDeviceToHost));
        return (size_t) c;
    };

    uint64_t base = 0;
    for (size_t blo = 0; blo < hist.size();) {
        size_t bhi = blo; int64_t m = 0;
        while (bhi < hist.size() && m + (int64_t) hist[bhi] <= cap) m += (int64_t) hist[bhi++];
        if (m > 0) {
            ++st.groups;
            FMI_CK(cudaMemset(d_cnt, 0, 8));
            select_kernel<<<grid_for(n), TPB>>>(w, n, b, (uint32_t) blo, (uint32_t) bhi, posA, keyA, d_cnt);
            cub::DoubleBuffer<uint64_t> kb(keyA, keyB), vb(posA, posB);
            size_t tb = tmp.bytes;
            FMI_CK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, kb, vb, (int) m, 0, 2 * FMI_K));
            run_start_kernel<<<grid_for(m), TPB>>>(kb.Current(), (int) m, i32A);
            tb = tmp.bytes;
            FMI_CK(cub::DeviceScan::InclusiveScan(tmp.p, tb, i32A, i32B, cub::Max(), (int) m));
            p1_write_kernel<<<grid_for(m), TPB>>>(vb.Current(), i32B, (int) m, base, isa_lo, isa_hi, flag);
            const size_t k = select_tied(vb.Current(), vb.Alternate(), (int) m);
            U.write(U.n, vb.Alternate(), k);
        }
        base += (uint64_t) m;
        blo = bhi;
    }
    if ((int64_t) base != n) throw Err("pass 1 placed " + std::to_string(base) + " of " + std::to_string(n) + " suffixes");
    FMI_CK(cudaDeviceSynchronize());
    const double t2 = secs();
    st.pass1_s = t2 - t1;
    st.unresolved = (int64_t) U.n;

    // ---- refinement rounds ----
    const int k2bits = bits_for((uint64_t) 2 * n);
    for (int64_t h = FMI_K; U.n > 0; h *= 2) {
        if (++st.rounds > 40) throw Err("suffix array refinement did not converge");
        const size_t nU = U.n;
        size_t u0 = 0, wcur = 0;
        while (u0 < nU) {
            const int L = (int) std::min<size_t>((size_t) cap, nU - u0);
            FMI_CK(cudaMemcpy(posA, U.at(u0), (size_t) L * 8, cudaMemcpyDefault));
            FMI_CK(cudaMemset(d_last, 0, sizeof(int)));
            r_groups_kernel<<<grid_for(L), TPB>>>(posA, L, isa_lo, isa_hi, i32A, keyB, d_last);
            int P = L;
            if (u0 + (size_t) L < nU) {          // the last loaded group may go on past the load: the piece ends before it
                FMI_CK(cudaMemcpy(&P, d_last, sizeof(int), cudaMemcpyDeviceToHost));
                if (P == 0) throw Err("a tie group larger than the refinement piece");
            }
            size_t tb = tmp.bytes;
            FMI_CK(cub::DeviceScan::InclusiveSum(tmp.p, tb, i32A, i32B, P));
            int n_groups = 0;
            FMI_CK(cudaMemcpy(&n_groups, i32B + P - 1, sizeof(int), cudaMemcpyDeviceToHost));
            const int obits = bits_for((uint64_t) n_groups);
            if (obits + k2bits > 64) throw Err("refinement sort key wider than 64 bits");
            r_keys_kernel<<<grid_for(P), TPB>>>(posA, i32A, i32B, keyB, P, isa_lo, isa_hi, n, h, k2bits, keyA, gval, gfirst);
            cub::DoubleBuffer<uint64_t> kb(keyA, keyB), vb(posA, posB);
            tb = tmp.bytes;
            FMI_CK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, kb, vb, P, 0, obits + k2bits));
            run_start_kernel<<<grid_for(P), TPB>>>(kb.Current(), P, i32A);
            tb = tmp.bytes;
            FMI_CK(cub::DeviceScan::InclusiveScan(tmp.p, tb, i32A, i32B, cub::Max(), P));
            r_write_kernel<<<grid_for(P), TPB>>>(kb.Current(), vb.Current(), i32B, P, k2bits, gval, gfirst, isa_lo, isa_hi, flag);
            const size_t k = select_tied(vb.Current(), vb.Alternate(), P);
            U.write(wcur, vb.Alternate(), k);          // in place: the kept slots never pass the slots still to load
            wcur += k; u0 += (size_t) P; ++st.pieces;
        }
        U.n = wcur;
    }
    FMI_CK(cudaDeviceSynchronize());
    st.unresolved_on_host = U.on_host;
    const double t3 = secs();
    st.refine_s = t3 - t2;
    mem.put(keyA); mem.put(keyB); mem.put(posA); mem.put(posB); mem.put(i32A); mem.put(i32B); mem.put(flag); mem.put(gval); mem.put(gfirst);
    { char *q = (char *) tmp.p; mem.put(q); tmp.p = nullptr; tmp.bytes = 0; }
    if (!U.on_host) mem.put(U.dev);

    // ---- emit ----
    // a row costs its SA slot (8), its BWT character (1), 1/64 of a CP_OCC entry and its counts (1.5) and 1/8 of a sample (0.625)
    const int64_t nb_all = (n_rows + 63) / 64;
    const int64_t win = std::max<int64_t>(64, std::min<int64_t>(nb_all * 64, work_bytes / 12 / 64 * 64));
    const int64_t nbw = win / 64;
    unsigned long long *sa = mem.get<unsigned long long>((size_t) win, "the SA window");
    uint8_t *bw = mem.get<uint8_t>((size_t) win, "the BWT window");
    FmiCpOcc *d_cp = mem.get<FmiCpOcc>((size_t) nbw, "CP_OCC entries");
    Cnt4 *cnt = mem.get<Cnt4>((size_t) nbw, "block counts"), *excl = mem.get<Cnt4>((size_t) nbw, "block counts");
    int8_t *d_ms = mem.get<int8_t>((size_t) win / 8, "SA samples");
    uint32_t *d_ls = mem.get<uint32_t>((size_t) win / 8, "SA samples");
    unsigned long long *d_chk = mem.get<unsigned long long>(3, "checks");
    long long *d_sent = (long long *) (d_chk + 2);
    {
        size_t s = 0;
        FMI_CK(cub::DeviceScan::ExclusiveScan(nullptr, s, cnt, excl, Cnt4Sum(), Cnt4{ { 0, 0, 0, 0 } }, (int) nbw));
        tmp.need(s);
    }
    const int64_t n_occ = (n_rows >> 6) + 1, n_sa = (n_rows >> 3) + 1;
    const int64_t off_cp = 8 + 5 * 8, off_ms = off_cp + n_occ * 64, off_ls = off_ms + n_sa, off_sent = off_ls + n_sa * 4;
    const std::string path = prefix + ".bwt.2bit.64", tmp_path = path + ".tmp";
    FILE *f = fopen(tmp_path.c_str(), "wb");
    if (!f) throw Err("cannot write " + tmp_path);
    std::vector<FmiCpOcc> hcp((size_t) nbw); std::vector<int8_t> hms((size_t) win / 8); std::vector<uint32_t> hls((size_t) win / 8);
    Cnt4 carry{ { 0, 0, 0, 0 } };
    long long sentinel = -1;
    try {
        FMI_CK(cudaMemset(d_chk, 0, 16));
        FMI_CK(cudaMemset(d_sent, 0xff, 8));
        for (int64_t r0 = 0; r0 < nb_all * 64; r0 += win) {
            const int64_t m = std::min(win, nb_all * 64 - r0), nb = m / 64;
            ++st.windows;
            FMI_CK(cudaMemset(sa, 0xff, (size_t) m * 8));
            if (r0 == 0) { const unsigned long long s0 = (unsigned long long) n; FMI_CK(cudaMemcpy(sa, &s0, 8, cudaMemcpyHostToDevice)); }
            scatter_kernel<<<grid_for(n), TPB>>>(isa_lo, isa_hi, n, r0, r0 + m, sa, d_chk);
            rows_kernel<<<grid_for(m), TPB>>>(w, sa, r0, m, n_rows, bw, d_ms, d_ls, d_sent, d_chk + 1);
            unsigned long long chk[2];
            FMI_CK(cudaMemcpy(chk, d_chk, 16, cudaMemcpyDeviceToHost));
            if (chk[0] || chk[1])
                throw Err("suffix array rows " + std::to_string(r0) + ".." + std::to_string(r0 + m) + ": " + std::to_string(chk[0]) + " written twice, " +
                          std::to_string(chk[1]) + " never written");
            blocks_kernel<<<grid_for(nb), TPB>>>(bw, nb, d_cp, cnt);
            size_t tb = tmp.bytes;
            FMI_CK(cub::DeviceScan::ExclusiveScan(tmp.p, tb, cnt, excl, Cnt4Sum(), Cnt4{ { 0, 0, 0, 0 } }, (int) nb));
            run_counts_kernel<<<grid_for(nb), TPB>>>(excl, carry, nb, d_cp);
            FMI_CK(cudaMemcpy(hcp.data(), d_cp, (size_t) nb * sizeof(FmiCpOcc), cudaMemcpyDeviceToHost));
            Cnt4 last_e, last_c;
            FMI_CK(cudaMemcpy(&last_e, excl + nb - 1, sizeof(Cnt4), cudaMemcpyDeviceToHost));
            FMI_CK(cudaMemcpy(&last_c, cnt + nb - 1, sizeof(Cnt4), cudaMemcpyDeviceToHost));
            for (int k = 0; k < 4; ++k) carry.c[k] += last_e.c[k] + last_c.c[k];
            const int64_t n_samp = (std::min(r0 + m, n_rows) - r0 + 7) / 8;
            FMI_CK(cudaMemcpy(hms.data(), d_ms, (size_t) n_samp, cudaMemcpyDeviceToHost));
            FMI_CK(cudaMemcpy(hls.data(), d_ls, (size_t) n_samp * 4, cudaMemcpyDeviceToHost));
            write_at(f, off_cp + r0, hcp.data(), (size_t) nb * sizeof(FmiCpOcc), tmp_path);
            write_at(f, off_ms + r0 / 8, hms.data(), (size_t) n_samp, tmp_path);
            write_at(f, off_ls + r0 / 8 * 4, hls.data(), (size_t) n_samp * 4, tmp_path);
        }
        FMI_CK(cudaMemcpy(&sentinel, d_sent, 8, cudaMemcpyDeviceToHost));
        // N and count[5] (file convention: count[c] = symbols below c), then the sentinel row.  n_rows = 2 l_pac + 1 is odd, so the blocks
        // fill all (n_rows >> 6) + 1 CP_OCC entries and all (n_rows >> 3) + 1 samples
        int64_t head[6] = { n_rows, 0, 0, 0, 0, 0 };
        for (int k = 0; k < 4; ++k) head[k + 2] = head[k + 1] + carry.c[k];
        write_at(f, 0, head, sizeof head, tmp_path);
        write_at(f, off_sent, &sentinel, 8, tmp_path);
        if (fclose(f) != 0) { f = nullptr; throw Err("cannot write " + tmp_path); }
        f = nullptr;
    } catch (...) {
        if (f) fclose(f);
        remove(tmp_path.c_str());
        throw;
    }
    if (rename(tmp_path.c_str(), path.c_str()) != 0) { remove(tmp_path.c_str()); throw Err("cannot rename " + tmp_path + " to " + path); }
    const double t4 = secs();
    st.emit_s = t4 - t3;
    st.total_s = t4 - t0;
    st.peak_device_bytes = mem.peak;
}

}  // namespace

extern "C" int bm2_index_build(int device, const char *prefix, int64_t work_bytes, bm2_index_build_stats *stats) {
    bm2_index_build_stats st;
    memset(&st, 0, sizeof st);
    if (!prefix) { bm2_set_error(nullptr, "bm2_index_build: prefix is NULL"); return 1; }
    try {
        build(device, prefix, work_bytes, st);
    } catch (const std::exception &e) {
        bm2_set_error(nullptr, std::string("bm2_index_build: ") + e.what());
        return 1;
    }
    if (stats) *stats = st;
    return 0;
}

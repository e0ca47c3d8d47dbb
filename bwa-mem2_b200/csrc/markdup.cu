// markdup.cu — duplicate marking on the GPU (bm2_mem --markdup), and the optical duplicates of --markdup-metrics; the per-template and
// per-group logic is markdup_device.cuh's.
//   bm2_dup_signatures   one warp per template: its primaries found by a ballot over its records, then per primary the CIGAR's reference
//                        length (inline or CG:B,I) and the qualities >= 15 summed across the warp; lane 0 writes the template's entries into
//                        fixed slots (one pair slot, two fragment-space slots), which cub::DeviceSelect compacts in template order
//   bm2_dup_resolve      entries sorted by (k1, k2, score descending, tid): an ordinal array through one stable cub::DeviceRadixSort pass per
//                        field, least significant first, each over the bits that field uses (their OR, from one reduction kernel); then
//                        (resolve) group heads, an inclusive scan into group numbers, per group whether it holds a pair-end entry and its first
//                        other entry (atomics), and cub::DeviceSelect::Flagged of the duplicates' template ids
//   bm2_dup_signatures_ex  the same kernel with each pair entry located (its first QNAME split on ':' by a ballot per 32 bytes) and classed,
//                        and the chunk's secondary / supplementary records and unmapped primaries counted (a ballot, one atomic per warp)
//   bm2_dup_resolve_ex   the same sort and duplicates, the located entries permuted with the order, then the optical pass over the pair
//                        groups: 2 .. 32 members one warp each (adjacency rows from ballots, closed under OR); 33 .. 300000 the exact cell
//                        pass (markdup_device.cuh): the located members sorted by (group, class, tile, read group, cell, x) - the read-group
//                        pass only when some member has one (bm2_markdup) - cells found by a scan,
//                        union-find over cells with atomicMin hooking and pointer jumping, side neighbours by extremes, diagonal ones by a
//                        binary search per member
//   bm2_dup_set          the duplicate bitset, kept on the context for bm2_bam_sort_compress_ex (bam_sort.cu)
#include "bm2_common.cuh"
#include "bm2_ctx.h"
#include "markdup_device.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <vector>

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;

template <class T> __device__ __forceinline__ T warp_sum(T v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// EX (bm2_dup_signatures_ex): the pair entry goes to lpair with the template's location and class, and counts[0] / counts[1] get the
// records with 0x100 / 0x800 and the unmapped primaries (one atomic per warp); pair is then unused
template <bool EX>
__global__ void dup_sig_kernel(const uint8_t *__restrict__ in, const int64_t *__restrict__ starts, const int64_t *__restrict__ tfirst,
                               const int64_t *__restrict__ tids, int64_t n_tmpl, bm2_dup_entry *pair, bm2_dup_entry *frag, bm2_dup_loc_entry *lpair,
                               unsigned long long *counts) {
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
    int loc = 0; int32_t tile = 0, x = 0, y = 0;
    if constexpr (EX) {
        unsigned sec = 0, unm = 0;
        for (int64_t b = r0; b < r1; b += 32) {
            const int64_t i = b + lane;
            const int32_t f = i < r1 ? (int32_t) bam_le16(in + starts[i] + 18) : 0;
            sec += __popc(__ballot_sync(kFull, (f & 0x900) != 0));
            unm += __popc(__ballot_sync(kFull, (f & 0x900) == 0 && (f & 4)));
        }
        if (lane == 0 && sec) atomicAdd(counts, (unsigned long long) sec);
        if (lane == 0 && unm) atomicAdd(counts + 1, (unsigned long long) unm);
        // the first record's QNAME split on ':' by a ballot per 32 bytes: the colon count and the last three colons
        int nc = 0, c1 = -1, c2 = -1, c3 = -1, len = 0;
        const uint8_t *name = nullptr;
        if (r1 > r0) { name = in + starts[r0] + 36; len = bm2_max<int>((int) in[starts[r0] + 12] - 1, 0); }
        for (int b = 0; b < len; b += 32) {
            const int i = b + lane;
            for (unsigned m = __ballot_sync(kFull, i < len && name[i] == ':'); m; m &= m - 1) { c1 = c2; c2 = c3; c3 = b + __ffs(m) - 1; ++nc; }
        }
        if (lane == 0) loc = dup_location_from_colons(name, len, nc, c1, c2, c3, &tile, &x, &y);
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
    if constexpr (EX) {
        if (has_pair) loc |= dup_pair_class((int32_t) bam_le16(in + starts[prim[0]] + 18), (int32_t) bam_le16(in + starts[prim[1]] + 18));
        lpair[t] = bm2_dup_loc_entry{ pe, tile, x, y, loc };
    } else pair[t] = pe;
    for (int k = 0; k < 2; ++k) { if (k >= n_frag) fe[k].kind = -1; frag[2 * t + k] = fe[k]; }
}

struct IsEntry {
    __device__ __forceinline__ bool operator()(const bm2_dup_entry &e) const { return e.kind >= 0; }
    __device__ __forceinline__ bool operator()(const bm2_dup_loc_entry &e) const { return e.e.kind >= 0; }
};

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

// ---- bm2_dup_resolve_ex: the located entries, and the optical pass over the pair groups ----
__global__ void dup_loc_split_kernel(const bm2_dup_loc_entry *__restrict__ le, int64_t n, bm2_dup_entry *e) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) e[i] = le[i].e;
}

__global__ void dup_loc_permute_kernel(const bm2_dup_loc_entry *__restrict__ le, const uint32_t *__restrict__ ord, int64_t n, bm2_dup_loc_entry *s) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) s[i] = le[ord[i]];
}

// gstart[g]: the first sorted entry of group g; gstart[groups] = n
__global__ void dup_gstart_kernel(const int32_t *__restrict__ head, const int32_t *__restrict__ seg, int64_t n, int32_t *gstart) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (head[i]) gstart[seg[i] - 1] = (int32_t) i;
    if (i == n - 1) gstart[seg[i]] = (int32_t) n;
}

// pair groups of 2 .. 32 members, one warp each: lane i holds member i; its row of the link relation from 32 broadcasts, closed under OR
// (row |= rows of its set bits) in at most 5 doubling rounds; the components are the lanes that are the lowest bit of their own row
__global__ void dup_optical_small_kernel(const bm2_dup_loc_entry *__restrict__ s, const int32_t *__restrict__ gstart, int64_t groups, int64_t d,
                                         unsigned long long *count) {
    const int64_t g = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (g >= groups) return;
    const int32_t s0 = gstart[g], sz = gstart[g + 1] - s0;
    if (sz < 2 || sz > 32 || s[s0].e.kind != DUP_KIND_PAIR) return;
    const bm2_dup_loc_entry me = s[s0 + bm2_min(lane, sz - 1)];
    unsigned row = 1u << lane;
    for (int j = 0; j < sz; ++j) {
        bm2_dup_loc_entry o;
        o.loc = __shfl_sync(kFull, me.loc, j); o.tile = __shfl_sync(kFull, me.tile, j);
        o.x = __shfl_sync(kFull, me.x, j); o.y = __shfl_sync(kFull, me.y, j);
        if (dup_optical_linked(me, o, d)) row |= 1u << j;
    }
    for (int r = 0; r < 5; ++r) {
        unsigned nr = row;
        for (int j = 0; j < sz; ++j) { const unsigned rj = __shfl_sync(kFull, row, j); if ((row >> j) & 1) nr |= rj; }
        if (!__any_sync(kFull, nr != row)) break;
        row = nr;
    }
    const int comps = __popc(__ballot_sync(kFull, lane < sz && __ffs(row) - 1 == lane));
    if (lane == 0) atomicAdd(count, (unsigned long long) (sz - comps));
}

// the located members of the pair groups of 33 .. DUP_OPTICAL_MAX_SET members: the exact pass's input
__global__ void dup_optical_flag_kernel(const bm2_dup_loc_entry *__restrict__ s, const int32_t *__restrict__ seg, const int32_t *__restrict__ gstart,
                                        int64_t n, uint8_t *flag) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t g = seg[i] - 1, sz = gstart[g + 1] - gstart[g];
    flag[i] = (sz > 32 && sz <= DUP_OPTICAL_MAX_SET && s[i].e.kind == DUP_KIND_PAIR && (s[i].loc & DUP_LOC_HAS)) ? 1 : 0;
}

// the cell sort's key of each member at its place in the current order: 0 x, 1 (cx, cy), 2 (group, class, tile), 3 read group
__global__ void dup_cell_field_kernel(const bm2_dup_loc_entry *__restrict__ s, const int32_t *__restrict__ seg, const uint32_t *__restrict__ idx,
                                      int64_t m, int field, int64_t d, uint64_t *keys) {
    const int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const uint32_t i = idx[p];
    const bm2_dup_loc_entry &e = s[i];
    keys[p] = field == 0 ? (uint64_t) ((uint32_t) e.x ^ 0x80000000u) : field == 1 ? dup_cell_lo(e, d) : field == 2 ? dup_cell_hi((uint32_t) (seg[i] - 1), e)
                                                                                                                   : (uint64_t) dup_loc_rg(e.loc);
}

// the OR of the exact pass's members' read groups (0 for bm2_mem's entries, whose cell sort then skips the read-group pass)
__global__ void dup_cell_rg_or_kernel(const bm2_dup_loc_entry *__restrict__ s, const uint8_t *__restrict__ flag, int64_t n, unsigned *rg_or) {
    const int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    unsigned v = p < n && flag[p] ? dup_loc_rg(s[p].loc) : 0u;
    for (int o = 16; o; o >>= 1) v |= __shfl_xor_sync(kFull, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicOr(rg_or, v);
}

// the members in cell order: their x and y, and a 1 where a cell starts
__global__ void dup_cell_head_kernel(const bm2_dup_loc_entry *__restrict__ s, const int32_t *__restrict__ seg, const uint32_t *__restrict__ idx,
                                     int64_t m, int64_t d, int32_t *head, int32_t *mx, int32_t *my) {
    const int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const bm2_dup_loc_entry &e = s[idx[p]];
    mx[p] = e.x; my[p] = e.y;
    if (p == 0) { head[p] = 1; return; }
    const bm2_dup_loc_entry &f = s[idx[p - 1]];
    head[p] = (dup_cell_hi((uint32_t) (seg[idx[p]] - 1), e) != dup_cell_hi((uint32_t) (seg[idx[p - 1]] - 1), f) || dup_loc_rg(e.loc) != dup_loc_rg(f.loc) ||
               dup_cell_lo(e, d) != dup_cell_lo(f, d)) ? 1 : 0;
}

// per cell (cell = 1-based numbers from the scan of the heads): its first member, its keys and read group, its own root, and its y range reset
__global__ void dup_cell_init_kernel(const bm2_dup_loc_entry *__restrict__ s, const int32_t *__restrict__ seg, const uint32_t *__restrict__ idx,
                                     const int32_t *__restrict__ cell, int64_t m, int64_t d, int32_t *cstart, uint64_t *ckey, uint32_t *crg, int32_t *parent,
                                     int32_t *cy) {
    const int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    if (p == m - 1) cstart[cell[p]] = (int32_t) m;
    if (p && cell[p] == cell[p - 1]) return;
    const int32_t c = cell[p] - 1;
    const bm2_dup_loc_entry &e = s[idx[p]];
    cstart[c] = (int32_t) p; parent[c] = c;
    ckey[2 * c] = dup_cell_hi((uint32_t) (seg[idx[p]] - 1), e); ckey[2 * c + 1] = dup_cell_lo(e, d); crg[c] = dup_loc_rg(e.loc);
    cy[2 * c] = INT32_MAX; cy[2 * c + 1] = INT32_MIN;
}

__global__ void dup_cell_y_kernel(const int32_t *__restrict__ cell, const int32_t *__restrict__ my, int64_t m, int32_t *cy) {
    const int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const int32_t c = cell[p] - 1;
    atomicMin(cy + 2 * c, my[p]); atomicMax(cy + 2 * c + 1, my[p]);
}

// per cell, one thread walking it backwards: the suffix max (suf[p]) and min (suf[m + p]) of y over the cell's members from p on
__global__ void dup_cell_suffix_kernel(const int32_t *__restrict__ cstart, int64_t nc, const int32_t *__restrict__ my, int64_t m, int32_t *suf) {
    const int64_t c = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nc) return;
    int32_t hi = INT32_MIN, lo = INT32_MAX;
    for (int64_t p = cstart[c + 1] - 1; p >= cstart[c]; --p) { hi = bm2_max(hi, my[p]); lo = bm2_min(lo, my[p]); suf[p] = hi; suf[m + p] = lo; }
}

// the cell with keys (hi, rg, lo), the cells' sort order, or -1
__device__ __forceinline__ int64_t dup_find_cell(const uint64_t *__restrict__ ckey, const uint32_t *__restrict__ crg, int64_t nc, uint64_t hi, uint32_t rg,
                                                 uint64_t lo) {
    int64_t a = 0, b = nc;
    while (a < b) {
        const int64_t k = (a + b) / 2;
        if (ckey[2 * k] < hi || (ckey[2 * k] == hi && (crg[k] < rg || (crg[k] == rg && ckey[2 * k + 1] < lo)))) a = k + 1; else b = k;
    }
    return a < nc && ckey[2 * a] == hi && crg[a] == rg && ckey[2 * a + 1] == lo ? a : -1;
}

__device__ __forceinline__ int32_t dup_root(const int32_t *parent, int32_t c) { while (parent[c] != c) c = parent[c]; return c; }

__device__ __forceinline__ void dup_hook(int32_t *parent, int32_t a, int32_t b, int32_t *changed) {
    const int32_t ra = dup_root(parent, a), rb = dup_root(parent, b);
    if (ra == rb) return;
    atomicMin(parent + bm2_max(ra, rb), bm2_min(ra, rb));
    *changed = 1;
}

// one round of hooking: member p of cell B tests the cells behind B diagonally; B's first member also tests the side neighbours (cx - 1, cy)
// and (cx, cy - 1) by the cells' extremes.  Roots only move to smaller cells, so every round with a change leaves fewer components.
__global__ void dup_cell_link_kernel(const int32_t *__restrict__ cell, const int32_t *__restrict__ cstart, const uint64_t *__restrict__ ckey,
                                     const uint32_t *__restrict__ crg, const int32_t *__restrict__ cy, const int32_t *__restrict__ mx, const int32_t *__restrict__ my,
                                     const int32_t *__restrict__ suf, int64_t m, int64_t nc, int64_t d, int32_t *parent, int32_t *changed) {
    const int64_t p = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const int32_t c = cell[p] - 1;
    const uint64_t hi = ckey[2 * c], lo = ckey[2 * c + 1];
    const uint32_t rg = crg[c];
    const uint32_t x = (uint32_t) (lo >> 32), y = (uint32_t) lo;
    const uint64_t left = (uint64_t) (x - 1) << 32;        // unused when x == 0: no cell to the left
    if (p == cstart[c]) {
        const int64_t a = x ? dup_find_cell(ckey, crg, nc, hi, rg, left | y) : -1;
        if (a >= 0 && (int64_t) mx[cstart[a + 1] - 1] >= (int64_t) mx[p] - d) dup_hook(parent, (int32_t) a, c, changed);
        const int64_t b = y ? dup_find_cell(ckey, crg, nc, hi, rg, (uint64_t) x << 32 | (y - 1)) : -1;
        if (b >= 0 && (int64_t) cy[2 * b + 1] >= (int64_t) cy[2 * c] - d) dup_hook(parent, (int32_t) b, c, changed);
    }
    for (int k = 0; k < 2 && x; ++k) {
        const bool below = k == 0;
        if (below ? y == 0 : y == 0xFFFFFFFFu) continue;
        const int64_t a = dup_find_cell(ckey, crg, nc, hi, rg, left | (below ? y - 1 : y + 1));
        if (a < 0) continue;
        const int32_t s0 = cstart[a];
        if (dup_cell_diag_linked(mx + s0, suf + (below ? 0 : m) + s0, cstart[a + 1] - s0, mx[p], my[p], d, below)) dup_hook(parent, (int32_t) a, c, changed);
    }
}

__global__ void dup_cell_jump_kernel(int32_t *parent, int64_t nc) {
    const int64_t c = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (c < nc) parent[c] = dup_root(parent, (int32_t) c);
}

__global__ void dup_cell_roots_kernel(const int32_t *__restrict__ parent, int64_t nc, unsigned long long *roots) {
    const int64_t c = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned b = __ballot_sync(kFull, c < nc && parent[c] == (int32_t) c);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(roots, (unsigned long long) __popc(b));
}

enum { DD_IN, DD_STARTS, DD_TFIRST, DD_TID, DD_PAIR, DD_FRAG, DD_OUT, DD_CNT, DD_TEMP, DD_KEYS0, DD_KEYS1, DD_ORD0, DD_ORD1, DD_SORTED,
       // bm2_dup_resolve_ex: the located entries as given and sorted, group starts; the exact pass's members (flags, compacted ids, x / y,
       // suffix extremes of y, cell numbers) and cells (first members, keys, y ranges, roots)
       DD_LOC_IN, DD_LOC_SORTED, DD_GSTART, DD_OPT_FLAG, DD_OPT_IDX, DD_MXY, DD_SUF, DD_CELL, DD_CSTART, DD_CKEY, DD_CY, DD_PARENT,
       DD_CRG,                          // the cells' read groups
       DD_END };
static_assert(DD_END == std::extent<decltype(bm2_ctx::dup_d)>::value, "bm2_ctx::dup_d: one buffer per slot");
// bm2_dup_resolve reuses the signature slots: entries in DD_PAIR, group numbers / flags / ids in DD_IN / DD_STARTS / DD_TFIRST / DD_TID / DD_FRAG

int bits_of(uint64_t v) { int b = 0; while (b < 64 && (v >> b)) ++b; return b; }

int ensure_events(bm2_ctx *ctx) {
    bm2_ctx *ctx_for_error = ctx;
    for (cudaEvent_t &ev : ctx->dup_ev) if (!ev) BM2_CUDA_OK(cudaEventCreate(&ev));
    return 0;
}

// bm2_dup_signatures (EX false: pairs) and bm2_dup_signatures_ex (EX true: lpairs and counts)
template <bool EX>
int dup_signatures(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tmpl_first, const int64_t *tmpl_id,
                   int64_t n_tmpl, const bm2_dup_entry **pairs, const bm2_dup_loc_entry **lpairs, int64_t *n_pairs, const bm2_dup_entry **frags,
                   int64_t *n_frags, int64_t *counts) {
    bm2_ctx *ctx_for_error = ctx;
    const std::string fn = EX ? "bm2_dup_signatures_ex" : "bm2_dup_signatures";
    if (!ctx || n < 0 || (n && !recs) || n_recs < 0 || (n_recs && !starts) || n_tmpl < 0 || !tmpl_first || (n_tmpl && !tmpl_id) || !(EX ? (void *) lpairs : (void *) pairs) ||
        !n_pairs || !frags || !n_frags || (EX && !counts)) {
        if (ctx) bm2_set_error(ctx, fn + ": bad arguments");
        return 1;
    }
    if (n_tmpl >= (1LL << 30)) { bm2_set_error(ctx, fn + ": 2^30 templates or more in one call"); return 1; }
    if (tmpl_first[0] != 0 || tmpl_first[n_tmpl] != n_recs) { bm2_set_error(ctx, fn + ": the templates do not cover the records"); return 1; }
    for (int64_t t = 0; t < n_tmpl; ++t)
        if (tmpl_first[t + 1] < tmpl_first[t]) { bm2_set_error(ctx, fn + ": template " + std::to_string(t) + " ends before it starts"); return 1; }
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t s = starts[i];
        if (s < 0 || s + 36 > n || s + 4 + (int64_t) bam_le32(recs + s) > n || (i && s < starts[i - 1] + 4 + (int64_t) bam_le32(recs + starts[i - 1]))) {
            bm2_set_error(ctx, fn + ": record " + std::to_string(i) + " does not lie within the buffer after the one before");
            return 1;
        }
    }
    using PairT = typename std::conditional<EX, bm2_dup_loc_entry, bm2_dup_entry>::type;
    BM2_CUDA_OK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->dup_d;
    size_t temp = 0, t2 = 0;
    BM2_CUDA_OK(cub::DeviceSelect::If(nullptr, temp, (bm2_dup_entry *) nullptr, (bm2_dup_entry *) nullptr, (int64_t *) nullptr,
                                      (int) bm2_max<int64_t>(2 * n_tmpl, 1), IsEntry(), st));
    BM2_CUDA_OK(cub::DeviceSelect::If(nullptr, t2, (PairT *) nullptr, (PairT *) nullptr, (int64_t *) nullptr, (int) bm2_max<int64_t>(n_tmpl, 1), IsEntry(), st));
    temp = bm2_max(temp, t2);
    const size_t out_bytes = bm2_max((size_t) 2 * n_tmpl * sizeof(bm2_dup_entry), (size_t) n_tmpl * sizeof(PairT)) + 8;
    if (ctx->ensure(b[DD_IN], (size_t) n + 16) || ctx->ensure(b[DD_STARTS], (size_t) n_recs * 8 + 8) ||
        ctx->ensure(b[DD_TFIRST], (size_t) (n_tmpl + 1) * 8) || ctx->ensure(b[DD_TID], (size_t) n_tmpl * 8 + 8) ||
        ctx->ensure(b[DD_PAIR], (size_t) n_tmpl * sizeof(PairT) + 8) || ctx->ensure(b[DD_FRAG], (size_t) 2 * n_tmpl * sizeof(bm2_dup_entry) + 8) ||
        ctx->ensure(b[DD_OUT], out_bytes) || ctx->ensure(b[DD_CNT], 32) || ctx->ensure(b[DD_TEMP], temp + 16) ||
        ensure_events(ctx)) return 1;
    int64_t cnt[2] = { 0, 0 };
    unsigned long long tallies[2] = { 0, 0 };
    ctx->dup_sig_ms = 0;
    if (n_tmpl) {
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_IN].p, recs, (size_t) n, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_STARTS].p, starts, (size_t) n_recs * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_TFIRST].p, tmpl_first, (size_t) (n_tmpl + 1) * 8, cudaMemcpyHostToDevice, st));
        BM2_CUDA_OK(cudaMemcpyAsync(b[DD_TID].p, tmpl_id, (size_t) n_tmpl * 8, cudaMemcpyHostToDevice, st));
        unsigned long long *tally = (unsigned long long *) ((uint8_t *) b[DD_CNT].p + 16);
        if (EX) BM2_CUDA_OK(cudaMemsetAsync(tally, 0, 16, st));
        BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[0], st));
        dup_sig_kernel<EX><<<(unsigned) ((n_tmpl * 32 + 255) / 256), 256, 0, st>>>((const uint8_t *) b[DD_IN].p, (const int64_t *) b[DD_STARTS].p,
                                                                                  (const int64_t *) b[DD_TFIRST].p, (const int64_t *) b[DD_TID].p, n_tmpl,
                                                                                  (bm2_dup_entry *) b[DD_PAIR].p, (bm2_dup_entry *) b[DD_FRAG].p,
                                                                                  (bm2_dup_loc_entry *) b[DD_PAIR].p, tally);
        BM2_CUDA_OK(cudaGetLastError());
        bm2_dup_entry *outp = (bm2_dup_entry *) b[DD_OUT].p;
        size_t tb = b[DD_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceSelect::If(b[DD_TEMP].p, tb, (const PairT *) b[DD_PAIR].p, (PairT *) outp, (int64_t *) b[DD_CNT].p, (int) n_tmpl, IsEntry(), st));
        BM2_CUDA_OK(cudaMemcpyAsync(&cnt[0], b[DD_CNT].p, 8, cudaMemcpyDeviceToHost, st));
        if (EX) BM2_CUDA_OK(cudaMemcpyAsync(tallies, tally, 16, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        std::vector<PairT> &hp = *(std::vector<PairT> *) (EX ? (void *) &ctx->dup_lpairs : (void *) &ctx->dup_pairs);
        hp.resize((size_t) cnt[0]);
        if (cnt[0]) BM2_CUDA_OK(cudaMemcpyAsync(hp.data(), outp, (size_t) cnt[0] * sizeof(PairT), cudaMemcpyDeviceToHost, st));
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
    } else { ctx->dup_pairs.clear(); ctx->dup_lpairs.clear(); ctx->dup_frags.clear(); }
    if (EX) { *lpairs = ctx->dup_lpairs.data(); counts[0] = (int64_t) tallies[0]; counts[1] = (int64_t) tallies[1]; }
    else *pairs = ctx->dup_pairs.data();
    *n_pairs = cnt[0];
    *frags = ctx->dup_frags.data(); *n_frags = cnt[1];
    return 0;
}

// the optical pass over the sorted located entries S (n of them, groups numbered by seg, started where head is set, `groups` of them):
// the small groups one warp each, then the exact cell pass over the located members of the larger ones.  Returns the optical count in *out.
// Work: the small kernel O(32 x 32) per group of 2 .. 32; the exact pass three radix-sort passes over its m members, a binary search per
// member and neighbour cell per round, the suffix walk of the largest cell, and rounds until no root moves (each round with a change leaves
// fewer components: at most as many rounds as cells, a few in practice; none for a dense group, which is one cell per class and tile).
int optical_pass(bm2_ctx *ctx, const bm2_dup_loc_entry *S, const int32_t *head, const int32_t *seg, int64_t n, int64_t groups, int64_t d, int64_t *out) {
    bm2_ctx *ctx_for_error = ctx;
    cudaStream_t st = ctx->stream;
    DevBuf *b = ctx->dup_d;
    const unsigned g = (unsigned) ((n + 255) / 256);
    int32_t *gstart = (int32_t *) b[DD_GSTART].p;
    unsigned long long *cnt = (unsigned long long *) ((uint8_t *) b[DD_CNT].p + 16);   // [0] small-group count, [1] roots of the exact pass
    unsigned *rg_or = (unsigned *) ((uint8_t *) b[DD_CNT].p + 12);
    BM2_CUDA_OK(cudaMemsetAsync(rg_or, 0, 20, st));
    dup_gstart_kernel<<<g, 256, 0, st>>>(head, seg, n, gstart);
    BM2_CUDA_OK(cudaGetLastError());
    dup_optical_small_kernel<<<(unsigned) ((groups * 32 + 255) / 256), 256, 0, st>>>(S, gstart, groups, d, cnt);
    BM2_CUDA_OK(cudaGetLastError());
    uint8_t *flag = (uint8_t *) b[DD_OPT_FLAG].p;
    dup_optical_flag_kernel<<<g, 256, 0, st>>>(S, seg, gstart, n, flag);
    BM2_CUDA_OK(cudaGetLastError());
    dup_cell_rg_or_kernel<<<g, 256, 0, st>>>(S, flag, n, rg_or);
    BM2_CUDA_OK(cudaGetLastError());
    uint32_t *ord0 = (uint32_t *) b[DD_ORD0].p;
    size_t tb = b[DD_TEMP].cap;
    BM2_CUDA_OK(cub::DeviceSelect::Flagged(b[DD_TEMP].p, tb, cub::CountingInputIterator<uint32_t>(0), flag, ord0, (int64_t *) b[DD_CNT].p, (int) n, st));
    int64_t m = 0;
    unsigned rgs = 0;
    BM2_CUDA_OK(cudaMemcpyAsync(&m, b[DD_CNT].p, 8, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaMemcpyAsync(&rgs, rg_or, 4, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    unsigned long long small = 0, roots = 0;
    if (m) {
        const unsigned gm = (unsigned) ((m + 255) / 256);
        cub::DoubleBuffer<uint64_t> kb((uint64_t *) b[DD_KEYS0].p, (uint64_t *) b[DD_KEYS1].p);
        cub::DoubleBuffer<uint32_t> vb(ord0, (uint32_t *) b[DD_ORD1].p);
        for (int f : { 0, 1, 3, 2 }) {                   // x, (cx, cy), read group, (group, class, tile): each pass stable
            if (f == 3 && !rgs) continue;
            dup_cell_field_kernel<<<gm, 256, 0, st>>>(S, seg, vb.Current(), m, f, d, kb.Current());
            BM2_CUDA_OK(cudaGetLastError());
            tb = b[DD_TEMP].cap;
            BM2_CUDA_OK(cub::DeviceRadixSort::SortPairs(b[DD_TEMP].p, tb, kb, vb, (int) m, 0, f == 0 ? 32 : f == 3 ? bits_of(rgs) : 64, st));
        }
        const uint32_t *idx = vb.Current();
        int32_t *mx = (int32_t *) b[DD_MXY].p, *my = mx + m, *cell = (int32_t *) b[DD_CELL].p, *cstart = (int32_t *) b[DD_CSTART].p;
        int32_t *parent = (int32_t *) b[DD_PARENT].p, *cy = (int32_t *) b[DD_CY].p, *suf = (int32_t *) b[DD_SUF].p;
        uint64_t *ckey = (uint64_t *) b[DD_CKEY].p;
        uint32_t *crg = (uint32_t *) b[DD_CRG].p;
        dup_cell_head_kernel<<<gm, 256, 0, st>>>(S, seg, idx, m, d, parent, mx, my);    // the heads in parent, for the scan
        BM2_CUDA_OK(cudaGetLastError());
        tb = b[DD_TEMP].cap;
        BM2_CUDA_OK(cub::DeviceScan::InclusiveSum(b[DD_TEMP].p, tb, (const int32_t *) parent, cell, (int) m, st));
        int32_t nc32 = 0;
        BM2_CUDA_OK(cudaMemcpyAsync(&nc32, cell + m - 1, 4, cudaMemcpyDeviceToHost, st));
        dup_cell_init_kernel<<<gm, 256, 0, st>>>(S, seg, idx, cell, m, d, cstart, ckey, crg, parent, cy);
        BM2_CUDA_OK(cudaGetLastError());
        dup_cell_y_kernel<<<gm, 256, 0, st>>>(cell, my, m, cy);
        BM2_CUDA_OK(cudaGetLastError());
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        const int64_t nc = nc32;
        const unsigned gc = (unsigned) ((nc + 255) / 256);
        dup_cell_suffix_kernel<<<gc, 256, 0, st>>>(cstart, nc, my, m, suf);
        BM2_CUDA_OK(cudaGetLastError());
        int32_t *changed = (int32_t *) ((uint8_t *) b[DD_CNT].p + 8);
        for (int32_t ch = 1; ch;) {
            BM2_CUDA_OK(cudaMemsetAsync(changed, 0, 4, st));
            dup_cell_link_kernel<<<gm, 256, 0, st>>>(cell, cstart, ckey, crg, cy, mx, my, suf, m, nc, d, parent, changed);
            BM2_CUDA_OK(cudaGetLastError());
            dup_cell_jump_kernel<<<gc, 256, 0, st>>>(parent, nc);
            BM2_CUDA_OK(cudaGetLastError());
            BM2_CUDA_OK(cudaMemcpyAsync(&ch, changed, 4, cudaMemcpyDeviceToHost, st));
            BM2_CUDA_OK(cudaStreamSynchronize(st));
        }
        dup_cell_roots_kernel<<<gc, 256, 0, st>>>(parent, nc, cnt + 1);
        BM2_CUDA_OK(cudaGetLastError());
    }
    unsigned long long c2[2] = { 0, 0 };
    BM2_CUDA_OK(cudaMemcpyAsync(c2, cnt, 16, cudaMemcpyDeviceToHost, st));
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    small = c2[0]; roots = c2[1];
    *out = (int64_t) small + (m - (int64_t) roots);
    return 0;
}

// bm2_dup_resolve (le null: e) and bm2_dup_resolve_ex (le, its sorted located entries in *lsorted and the optical count in *n_optical)
int dup_resolve(bm2_ctx *ctx, const bm2_dup_entry *entries, const bm2_dup_loc_entry *le, int64_t n, int resolve, int64_t d, const bm2_dup_entry **sorted,
                const bm2_dup_loc_entry **lsorted, const int64_t **dups, int64_t *n_dups, int64_t *n_optical) {
    bm2_ctx *ctx_for_error = ctx;
    const bool ex = lsorted != nullptr || n_optical != nullptr || le != nullptr;
    const std::string fn = ex ? "bm2_dup_resolve_ex" : "bm2_dup_resolve";
    if (!ctx || n < 0 || (n && !(ex ? (const void *) le : (const void *) entries)) || (!resolve && !(ex ? (void *) lsorted : (void *) sorted)) ||
        (resolve && (!dups || !n_dups)) || (ex && (d < 0 || d > INT32_MAX))) {
        if (ctx) bm2_set_error(ctx, fn + ": bad arguments");
        return 1;
    }
    if (n >= (1LL << 31) - 1) { bm2_set_error(ctx, fn + ": 2^31-1 entries or more in one call"); return 1; }
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
        if (ex) {
            BM2_CUDA_OK(cub::DeviceSelect::Flagged(nullptr, t2, cub::CountingInputIterator<uint32_t>(0), (const uint8_t *) nullptr, (uint32_t *) nullptr,
                                                   (int64_t *) nullptr, ni, st));
            temp = bm2_max(temp, t2);
        }
    }
    const size_t ne = (size_t) n * sizeof(bm2_dup_entry) + 8;
    if (ctx->ensure(b[DD_PAIR], ne) || ctx->ensure(b[DD_SORTED], ne) || ctx->ensure(b[DD_KEYS0], (size_t) n * 8 + 8) ||
        ctx->ensure(b[DD_KEYS1], (size_t) n * 8 + 8) || ctx->ensure(b[DD_ORD0], (size_t) n * 4 + 8) || ctx->ensure(b[DD_ORD1], (size_t) n * 4 + 8) ||
        ctx->ensure(b[DD_CNT], 32) || ctx->ensure(b[DD_TEMP], temp + 16) || ensure_events(ctx)) return 1;
    if (resolve && (ctx->ensure(b[DD_IN], (size_t) n * 4 + 8) || ctx->ensure(b[DD_STARTS], (size_t) n * 4 + 8) ||
                    ctx->ensure(b[DD_TFIRST], (size_t) n * 4 + 8) || ctx->ensure(b[DD_TID], (size_t) n * 4 + 8) ||
                    ctx->ensure(b[DD_FRAG], (size_t) n * 9 + 32) || ctx->ensure(b[DD_OUT], (size_t) n * 8 + 8))) return 1;
    const size_t nl = (size_t) n * sizeof(bm2_dup_loc_entry) + 8;
    if (ex && (ctx->ensure(b[DD_LOC_IN], nl) || ctx->ensure(b[DD_LOC_SORTED], nl))) return 1;
    if (ex && resolve && (ctx->ensure(b[DD_GSTART], (size_t) n * 4 + 8) || ctx->ensure(b[DD_OPT_FLAG], (size_t) n + 8) ||
                          ctx->ensure(b[DD_MXY], (size_t) n * 8 + 8) || ctx->ensure(b[DD_SUF], (size_t) n * 8 + 8) ||
                          ctx->ensure(b[DD_CELL], (size_t) n * 4 + 8) || ctx->ensure(b[DD_CSTART], (size_t) n * 4 + 8) ||
                          ctx->ensure(b[DD_CKEY], (size_t) n * 16 + 8) || ctx->ensure(b[DD_CY], (size_t) n * 8 + 8) ||
                          ctx->ensure(b[DD_PARENT], (size_t) n * 4 + 8) || ctx->ensure(b[DD_CRG], (size_t) n * 4 + 8))) return 1;
    ctx->dup_resolve_ms = 0;
    ctx->dup_sorted.clear(); ctx->dup_lsorted.clear(); ctx->dup_ids.clear();
    if (n_optical) *n_optical = 0;
    if (n == 0) {
        if (sorted) *sorted = ctx->dup_sorted.data();
        if (lsorted) *lsorted = ctx->dup_lsorted.data();
        if (resolve) { *dups = ctx->dup_ids.data(); *n_dups = 0; }
        return 0;
    }
    const unsigned g = (unsigned) ((n + 255) / 256);
    bm2_dup_entry *E = (bm2_dup_entry *) b[DD_PAIR].p, *S = (bm2_dup_entry *) b[DD_SORTED].p;
    if (ex) BM2_CUDA_OK(cudaMemcpyAsync(b[DD_LOC_IN].p, le, (size_t) n * sizeof(bm2_dup_loc_entry), cudaMemcpyHostToDevice, st));
    else BM2_CUDA_OK(cudaMemcpyAsync(E, entries, (size_t) n * sizeof(bm2_dup_entry), cudaMemcpyHostToDevice, st));
    BM2_CUDA_OK(cudaMemsetAsync(b[DD_CNT].p, 0, 24, st));
    BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[0], st));
    if (ex) {
        dup_loc_split_kernel<<<g, 256, 0, st>>>((const bm2_dup_loc_entry *) b[DD_LOC_IN].p, n, E);
        BM2_CUDA_OK(cudaGetLastError());
    }
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
    bm2_dup_loc_entry *SL = (bm2_dup_loc_entry *) b[DD_LOC_SORTED].p;
    if (ex) {
        dup_loc_permute_kernel<<<g, 256, 0, st>>>((const bm2_dup_loc_entry *) b[DD_LOC_IN].p, vb.Current(), n, SL);
        BM2_CUDA_OK(cudaGetLastError());
    }
    int64_t nd = 0;
    if (!resolve) {
        BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[3], st));
        if (ex) {
            ctx->dup_lsorted.resize((size_t) n);
            BM2_CUDA_OK(cudaMemcpyAsync(ctx->dup_lsorted.data(), SL, (size_t) n * sizeof(bm2_dup_loc_entry), cudaMemcpyDeviceToHost, st));
        } else {
            ctx->dup_sorted.resize((size_t) n);
            BM2_CUDA_OK(cudaMemcpyAsync(ctx->dup_sorted.data(), S, (size_t) n * sizeof(bm2_dup_entry), cudaMemcpyDeviceToHost, st));
        }
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
        if (!ex) BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[3], st));
        int32_t groups = 0;
        BM2_CUDA_OK(cudaMemcpyAsync(&nd, b[DD_CNT].p, 8, cudaMemcpyDeviceToHost, st));
        if (ex) BM2_CUDA_OK(cudaMemcpyAsync(&groups, seg + n - 1, 4, cudaMemcpyDeviceToHost, st));
        BM2_CUDA_OK(cudaStreamSynchronize(st));
        ctx->dup_ids.resize((size_t) nd);
        if (nd) BM2_CUDA_OK(cudaMemcpyAsync(ctx->dup_ids.data(), b[DD_OUT].p, (size_t) nd * 8, cudaMemcpyDeviceToHost, st));
        if (ex) {
            int64_t opt = 0;
            if (optical_pass(ctx, SL, head, seg, n, groups, d, &opt)) return 1;
            BM2_CUDA_OK(cudaEventRecord(ctx->dup_ev[3], st));
            // every group's count is at most its duplicates (size - 1), so the sum is at most the duplicates of the pair groups
            if (opt < 0 || opt > nd) { bm2_set_error(ctx, fn + ": " + std::to_string(opt) + " optical duplicates, more than the " + std::to_string(nd) + " duplicates"); return 1; }
            if (n_optical) *n_optical = opt;
        }
    }
    BM2_CUDA_OK(cudaStreamSynchronize(st));
    float ms[2] = { 0, 0 };
    BM2_CUDA_OK(cudaEventElapsedTime(&ms[0], ctx->dup_ev[0], ctx->dup_ev[1]));
    BM2_CUDA_OK(cudaEventElapsedTime(&ms[1], ctx->dup_ev[2], ctx->dup_ev[3]));
    ctx->dup_resolve_ms = (double) ms[0] + ms[1];
    if (sorted) *sorted = ctx->dup_sorted.data();
    if (lsorted) *lsorted = ctx->dup_lsorted.data();
    if (resolve) { *dups = ctx->dup_ids.data(); *n_dups = nd; }
    return 0;
}

}  // namespace

extern "C" int bm2_dup_signatures(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tmpl_first,
                                  const int64_t *tmpl_id, int64_t n_tmpl, const bm2_dup_entry **pairs, int64_t *n_pairs, const bm2_dup_entry **frags,
                                  int64_t *n_frags) {
    return dup_signatures<false>(ctx, recs, n, starts, n_recs, tmpl_first, tmpl_id, n_tmpl, pairs, nullptr, n_pairs, frags, n_frags, nullptr);
}

extern "C" int bm2_dup_signatures_ex(bm2_ctx *ctx, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tmpl_first,
                                     const int64_t *tmpl_id, int64_t n_tmpl, const bm2_dup_loc_entry **pairs, int64_t *n_pairs, const bm2_dup_entry **frags,
                                     int64_t *n_frags, int64_t counts[2]) {
    return dup_signatures<true>(ctx, recs, n, starts, n_recs, tmpl_first, tmpl_id, n_tmpl, nullptr, pairs, n_pairs, frags, n_frags, counts);
}

extern "C" int bm2_dup_resolve(bm2_ctx *ctx, const bm2_dup_entry *entries, int64_t n, int resolve, const bm2_dup_entry **sorted, const int64_t **dups,
                               int64_t *n_dups) {
    return dup_resolve(ctx, entries, nullptr, n, resolve, 0, sorted, nullptr, dups, n_dups, nullptr);
}

extern "C" int bm2_dup_resolve_ex(bm2_ctx *ctx, const bm2_dup_loc_entry *entries, int64_t n, int resolve, int64_t distance, const bm2_dup_loc_entry **sorted,
                                  const int64_t **dups, int64_t *n_dups, int64_t *n_optical) {
    if (ctx && !resolve && !sorted) { bm2_set_error(ctx, "bm2_dup_resolve_ex: bad arguments"); return 1; }
    int64_t unused = 0;
    return dup_resolve(ctx, nullptr, entries, n, resolve, distance, nullptr, sorted, dups, n_dups, n_optical ? n_optical : &unused);
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

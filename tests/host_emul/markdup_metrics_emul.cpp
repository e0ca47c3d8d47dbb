// markdup_metrics_emul.cpp — TEST ONLY: bm2_mem --markdup-metrics on the CPU.  The location, class and link logic is markdup_device.cuh's,
// compiled here; bm2_dup_signatures_ex is restated per template over markdup_emul.cpp's bm2_dup_signatures restatement, and
// bm2_dup_resolve_ex as markdup_emul.cpp's resolve with the located entries sorted by the same stable order, then the optical pass: groups of
// up to 32 members by the warp kernel's rows closed under OR (a loop over the lanes), larger ones by the cell pass restated sequentially
// (one sort, cells, the same neighbour tests, a plain union-find).  The metrics file is markdup_metrics.h's.  The GPU must give these
// entries, counters and optical counts exactly.
#include "markdup_device.cuh"
#include "markdup_metrics.h"
#include <algorithm>
#include <cstring>
#include <numeric>
#include <vector>

extern "C" void markdup_emul_signatures(const uint8_t *recs, const int64_t *starts, const int64_t *tmpl_first, const int64_t *tmpl_id, int64_t n_tmpl,
                                        bm2_dup_entry *pairs_out, int64_t *n_pairs, bm2_dup_entry *frags_out, int64_t *n_frags);
extern "C" void markdup_emul_resolve(const bm2_dup_entry *e, int64_t n, int res, bm2_dup_entry *sorted_out, int64_t *dups_out, int64_t *n_dups);

namespace {

// dup_optical_small_kernel, one lane at a time
int64_t optical_small(const bm2_dup_loc_entry *g, int sz, int64_t d) {
    uint32_t row[32];
    for (int i = 0; i < sz; ++i) {
        row[i] = 1u << i;
        for (int j = 0; j < sz; ++j) if (dup_optical_linked(g[i], g[j], d)) row[i] |= 1u << j;
    }
    for (int r = 0; r < 5; ++r) {
        uint32_t nr[32];
        bool changed = false;
        for (int i = 0; i < sz; ++i) {
            nr[i] = row[i];
            for (int j = 0; j < sz; ++j) if ((row[i] >> j) & 1) nr[i] |= row[j];
            changed |= nr[i] != row[i];
        }
        if (!changed) break;
        std::copy(nr, nr + sz, row);
    }
    int comps = 0;
    for (int i = 0; i < sz; ++i) comps += __builtin_ctz(row[i]) == i;
    return sz - comps;
}

int32_t root(std::vector<int32_t> &p, int32_t c) { while (p[(size_t) c] != c) c = p[(size_t) c] = p[(size_t) p[(size_t) c]]; return c; }

// the exact cell pass of one group (dup_cell_*_kernel), sequential: located members - components
int64_t optical_cells(const bm2_dup_loc_entry *g, int64_t sz, int64_t d) {
    std::vector<int64_t> idx;
    for (int64_t i = 0; i < sz; ++i) if (g[i].loc & DUP_LOC_HAS) idx.push_back(i);
    const int64_t m = (int64_t) idx.size();
    if (!m) return 0;
    auto hi = [&](int64_t i) { return dup_cell_hi(0, g[i]); };
    auto lo = [&](int64_t i) { return dup_cell_lo(g[i], d); };
    std::stable_sort(idx.begin(), idx.end(), [&](int64_t a, int64_t b) {
        if (hi(a) != hi(b)) return hi(a) < hi(b);
        if (lo(a) != lo(b)) return lo(a) < lo(b);
        return g[a].x < g[b].x;
    });
    std::vector<int32_t> mx((size_t) m), my((size_t) m), cell((size_t) m), cstart, sufmax((size_t) m), sufmin((size_t) m), cymin, cymax;
    std::vector<std::pair<uint64_t, uint64_t>> ckey;
    for (int64_t p = 0; p < m; ++p) {
        mx[(size_t) p] = g[idx[(size_t) p]].x; my[(size_t) p] = g[idx[(size_t) p]].y;
        if (p == 0 || hi(idx[(size_t) p]) != hi(idx[(size_t) p - 1]) || lo(idx[(size_t) p]) != lo(idx[(size_t) p - 1])) {
            cstart.push_back((int32_t) p); ckey.push_back({hi(idx[(size_t) p]), lo(idx[(size_t) p])}); cymin.push_back(INT32_MAX); cymax.push_back(INT32_MIN);
        }
        cell[(size_t) p] = (int32_t) cstart.size() - 1;
        cymin.back() = std::min(cymin.back(), my[(size_t) p]); cymax.back() = std::max(cymax.back(), my[(size_t) p]);
    }
    const int64_t nc = (int64_t) cstart.size();
    cstart.push_back((int32_t) m);
    for (int64_t c = 0; c < nc; ++c) {
        int32_t h = INT32_MIN, l = INT32_MAX;
        for (int64_t p = cstart[(size_t) c + 1] - 1; p >= cstart[(size_t) c]; --p) {
            h = std::max(h, my[(size_t) p]); l = std::min(l, my[(size_t) p]); sufmax[(size_t) p] = h; sufmin[(size_t) p] = l;
        }
    }
    auto find = [&](uint64_t h, uint64_t l) -> int64_t {
        auto it = std::lower_bound(ckey.begin(), ckey.end(), std::make_pair(h, l));
        return it != ckey.end() && *it == std::make_pair(h, l) ? it - ckey.begin() : -1;
    };
    std::vector<int32_t> parent((size_t) nc);
    std::iota(parent.begin(), parent.end(), 0);
    auto unite = [&](int64_t a, int64_t b) { const int32_t ra = root(parent, (int32_t) a), rb = root(parent, (int32_t) b); if (ra != rb) parent[(size_t) std::max(ra, rb)] = std::min(ra, rb); };
    for (int64_t p = 0; p < m; ++p) {
        const int32_t c = cell[(size_t) p];
        const uint64_t h = ckey[(size_t) c].first, l = ckey[(size_t) c].second;
        const uint32_t x = (uint32_t) (l >> 32), y = (uint32_t) l;
        if (p == cstart[(size_t) c]) {
            const int64_t a = x ? find(h, (uint64_t) (x - 1) << 32 | y) : -1;
            if (a >= 0 && (int64_t) mx[(size_t) cstart[(size_t) a + 1] - 1] >= (int64_t) mx[(size_t) p] - d) unite(a, c);
            const int64_t b = y ? find(h, (uint64_t) x << 32 | (y - 1)) : -1;
            if (b >= 0 && (int64_t) cymax[(size_t) b] >= (int64_t) cymin[(size_t) c] - d) unite(b, c);
        }
        for (int k = 0; k < 2 && x; ++k) {
            const bool below = k == 0;
            if (below ? y == 0 : y == 0xFFFFFFFFu) continue;
            const int64_t a = find(h, (uint64_t) (x - 1) << 32 | (below ? y - 1 : y + 1));
            if (a < 0) continue;
            const int32_t s0 = cstart[(size_t) a];
            if (dup_cell_diag_linked(mx.data() + s0, (below ? sufmax : sufmin).data() + s0, cstart[(size_t) a + 1] - s0, mx[(size_t) p], my[(size_t) p], d, below))
                unite(a, c);
        }
    }
    int64_t roots = 0;
    for (int64_t c = 0; c < nc; ++c) roots += root(parent, (int32_t) c) == c;
    return m - roots;
}

}  // namespace

// the optical count of one pair group's members (any order), as bm2_dup_resolve_ex counts it
extern "C" int64_t mm_optical_group(const bm2_dup_loc_entry *g, int64_t sz, int64_t d) {
    if (sz < 2 || sz > DUP_OPTICAL_MAX_SET) return 0;
    return sz <= 32 ? optical_small(g, (int) sz, d) : optical_cells(g, sz, d);
}

// dup_name_location: out = {loc, tile, x, y}
extern "C" void mm_name_location(const uint8_t *name, int len, int32_t *out) { out[0] = dup_name_location(name, len, out + 1, out + 2, out + 3); }

// bm2_dup_signatures_ex restated: pairs_out / frags_out have room for n_tmpl / 2 n_tmpl entries
extern "C" void mm_signatures_ex(const uint8_t *recs, const int64_t *starts, const int64_t *tmpl_first, const int64_t *tmpl_id, int64_t n_tmpl,
                                 bm2_dup_loc_entry *pairs_out, int64_t *n_pairs, bm2_dup_entry *frags_out, int64_t *n_frags, int64_t *counts) {
    *n_pairs = *n_frags = 0; counts[0] = counts[1] = 0;
    for (int64_t t = 0; t < n_tmpl; ++t) {
        bm2_dup_entry pe, fe[2]; int64_t np = 0, nf = 0;
        markdup_emul_signatures(recs, starts, tmpl_first + t, tmpl_id + t, 1, &pe, &np, fe, &nf);
        int32_t pflag[2] = { 0, 0 }; int n_prim = 0;
        for (int64_t i = tmpl_first[t]; i < tmpl_first[t + 1]; ++i) {
            const int32_t f = (int32_t) bam_le16(recs + starts[i] + 18);
            counts[0] += (f & 0x900) != 0;
            counts[1] += (f & 0x900) == 0 && (f & 4);
            if (dup_is_primary(f) && n_prim < 2) pflag[n_prim++] = f;
        }
        if (np) {
            bm2_dup_loc_entry &l = pairs_out[(*n_pairs)++];
            l.e = pe;
            const uint8_t *r = recs + starts[tmpl_first[t]];
            l.loc = dup_name_location(r + 36, std::max<int>((int) r[12] - 1, 0), &l.tile, &l.x, &l.y) | dup_pair_class(pflag[0], pflag[1]);
        }
        for (int64_t k = 0; k < nf; ++k) frags_out[(*n_frags)++] = fe[k];
    }
}

// bm2_dup_resolve_ex restated: sorted_out (n entries) when !res, else dups_out (room for n ids), *n_dups and *n_optical
extern "C" void mm_resolve_ex(const bm2_dup_loc_entry *e, int64_t n, int res, int64_t d, bm2_dup_loc_entry *sorted_out, int64_t *dups_out, int64_t *n_dups,
                              int64_t *n_optical) {
    std::vector<bm2_dup_loc_entry> s(e, e + n);
    std::stable_sort(s.begin(), s.end(), [](const bm2_dup_loc_entry &a, const bm2_dup_loc_entry &b) { return dup_less(a.e, b.e); });
    if (!res) { std::copy(s.begin(), s.end(), sorted_out); return; }
    std::vector<bm2_dup_entry> base((size_t) n);
    for (int64_t i = 0; i < n; ++i) base[(size_t) i] = e[i].e;
    markdup_emul_resolve(base.data(), n, 1, nullptr, dups_out, n_dups);
    int64_t opt = 0;
    for (int64_t g0 = 0; g0 < n;) {
        int64_t g1 = g0 + 1;
        while (g1 < n && dup_same_key(s[(size_t) g1].e, s[(size_t) g0].e)) ++g1;
        if (s[(size_t) g0].e.kind == DUP_KIND_PAIR) opt += mm_optical_group(s.data() + g0, g1 - g0, d);
        g0 = g1;
    }
    *n_optical = opt;
}

// markdup_metrics.h: v = {unpaired reads, read pairs, secondary or supplementary, unmapped, unpaired dups, pair dups, optical pairs}
extern "C" int64_t mm_metrics_text(const int64_t *v, const char *library, const char *args, char *out, int64_t cap) {
    DupMetrics m;
    if (library) m.library = library;
    m.unpaired_reads = v[0]; m.read_pairs = v[1]; m.secondary_or_supplementary = v[2]; m.unmapped = v[3];
    m.unpaired_dups = v[4]; m.pair_dups = v[5]; m.optical_pairs = v[6];
    const std::string t = dup_metrics_text(m, args);
    if ((int64_t) t.size() < cap) memcpy(out, t.c_str(), t.size() + 1);
    return (int64_t) t.size();
}

extern "C" int64_t mm_library_size(int64_t pairs, int64_t unique) { return dup_library_size(pairs, unique); }

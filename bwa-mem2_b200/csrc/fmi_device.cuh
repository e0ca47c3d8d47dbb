// fmi_device.cuh — the per-element logic of bm2_index_build (fmi_build.cu) as BM2_HD functions: the 31-mer key, the second key of a
// doubling round, the 40-bit inverse suffix array and a 64-row block to a CP_OCC entry.  tests/host_emul/fmi_emul.cpp runs the same functions
// in the same pass and round structure with g++.
#pragma once
#include "hd.h"

constexpr int FMI_K = 31;                       // bases per first-pass sort key (62 bits)

// The text: 2 bits per base, 32 bases per word, the first base in the top bits.  The bits past base n are zero and one zero word follows
// the last, so that a key at any position reads two words.
BM2_HD uint32_t fmi_base(const uint64_t *w, int64_t i) { return (uint32_t) (w[i >> 5] >> (62 - 2 * (i & 31))) & 3u; }

// the 31-mer key of the suffix at p, first base most significant.  Bases past the end count as A, so a suffix shorter than 31 ties with
// the suffixes it prefixes until fmi_key2's beyond-the-end rule puts it first.
BM2_HD uint64_t fmi_kmer(const uint64_t *w, int64_t p) {
    const int64_t q = p >> 5; const int s = (int) (p & 31) * 2;
    uint64_t v = w[q] << s;
    if (s) v |= w[q + 1] >> (64 - s);
    return v >> 2;
}
// the first-pass bucket of the suffix at p: its first b bases, the top 2b bits of its key, so that bucket order is key order
BM2_HD uint32_t fmi_bucket(const uint64_t *w, int64_t p, int b) { return (uint32_t) (fmi_kmer(w, p) >> (62 - 2 * b)); }

// the inverse suffix array: 40-bit ranks kept as a uint32 low word and a uint8 high byte, as the index file splits its sampled SA
BM2_HD uint64_t fmi_get40(const uint32_t *lo, const uint8_t *hi, int64_t i) { return (uint64_t) hi[i] << 32 | lo[i]; }
BM2_HD void fmi_put40(uint32_t *lo, uint8_t *hi, int64_t i, uint64_t v) { lo[i] = (uint32_t) v; hi[i] = (uint8_t) (v >> 32); }

// The second key of the suffix at p in the doubling round of step h (Larsson-Sadakane, as index_build.py): the rank of the suffix at p + h,
// offset past n.  A suffix that ends within h bases gets its length n - p instead: it sorts before every suffix it prefixes, and shorter
// before longer (index_build.py's negative -(p + h - n) - 1, made non-negative).  Values lie in [1, 2n].
BM2_HD uint64_t fmi_key2(const uint32_t *lo, const uint8_t *hi, int64_t n, int64_t p, int64_t h) {
    return p + h < n ? (uint64_t) n + 1 + fmi_get40(lo, hi, p + h) : (uint64_t) (n - p);
}

// bm2_cp_occ's layout (CP_OCC, src/FMI_search.h:54-58)
struct FmiCpOcc { int64_t cp_count[4]; uint64_t one_hot[4]; };

// The BWT character of a row whose suffix starts at s: the base before it, 4 for the row of the suffix at 0.
BM2_HD uint8_t fmi_bwt_char(const uint64_t *w, uint64_t s) { return s == 0 ? 4 : (uint8_t) fmi_base(w, (int64_t) s - 1); }

// One 64-row block of the BWT (codes 0-3; the sentinel's 4 and the padding rows' 6 count nothing) -> its CP_OCC entry, given the counts of
// the rows before it; row j of the block is bit 63 - j (build_fm_index, src/FMI_search.cpp:218-251).  Returns the block's counts in add.
BM2_HD void fmi_cp_entry(const uint8_t *c, const int64_t *run, FmiCpOcc *e, int64_t *add) {
    uint64_t oh[4] = { 0, 0, 0, 0 };
    for (int j = 0; j < 64; ++j) if (c[j] < 4) oh[c[j]] |= 1ull << (63 - j);
    for (int k = 0; k < 4; ++k) { e->cp_count[k] = run[k]; e->one_hot[k] = oh[k]; add[k] = BM2_POPC64(oh[k]); }
}

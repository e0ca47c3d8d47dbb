// fmi_emul.cpp — TEST ONLY: bm2_index_build's pass and round structure (bwa-mem2_b200/csrc/fmi_build.cu) run sequentially with g++ over the
// same BM2_HD functions (fmi_device.cuh), so that the CPU suite checks the algorithm - bucket groups, pieces that end at tie-group boundaries,
// in-place refinement across pieces, windowed emit - against a naive sort and index_build.py at sizes where every stage runs several times.
//   cap   slots per group / piece (raised to the largest bucket + 1, as the builder does);  win   rows per emit window (a multiple of 64)
#include "fmi_device.cuh"
#include <algorithm>
#include <cstring>
#include <utility>
#include <vector>

extern "C" int fmi_emul(const uint8_t *T, int64_t n, int64_t cap, int64_t win, int64_t *sa_out, int64_t *cp_out, int8_t *ms_out,
                        uint32_t *ls_out, int64_t *info) {
    std::vector<uint64_t> w((size_t) (n / 32 + 2), 0);
    for (int64_t i = 0; i < n; ++i) w[(size_t) (i >> 5)] |= (uint64_t) T[i] << (62 - 2 * (i & 31));
    std::vector<uint32_t> lo((size_t) n); std::vector<uint8_t> hi((size_t) n);
    int b = 1;
    while (b < 12 && (n >> (2 * b)) * 16 > cap) ++b;
    std::vector<int64_t> hist((size_t) 1 << (2 * b), 0);
    for (int64_t p = 0; p < n; ++p) ++hist[fmi_bucket(w.data(), p, b)];
    cap = std::max<int64_t>(cap, *std::max_element(hist.begin(), hist.end()) + 1);
    int64_t groups = 0, pieces = 0, rounds = 0, windows = 0;
    std::vector<uint64_t> U;
    // pass 1
    uint64_t base = 0;
    for (size_t blo = 0; blo < hist.size();) {
        size_t bhi = blo; int64_t m = 0;
        while (bhi < hist.size() && m + hist[bhi] <= cap) m += hist[bhi++];
        if (m > 0) {
            ++groups;
            std::vector<std::pair<uint64_t, uint64_t>> kp;
            for (int64_t p = 0; p < n; ++p) { const uint32_t bk = fmi_bucket(w.data(), p, b); if (bk >= blo && bk < bhi) kp.push_back({ fmi_kmer(w.data(), p), (uint64_t) p }); }
            std::sort(kp.begin(), kp.end(), [](const auto &x, const auto &y) { return x.first < y.first; });
            int64_t start = 0;
            for (int64_t j = 0; j < m; ++j) {
                if (j == 0 || kp[j].first != kp[j - 1].first) start = j;
                fmi_put40(lo.data(), hi.data(), (int64_t) kp[j].second, base + (uint64_t) start);
                const bool single = start == j && (j + 1 == m || kp[j + 1].first != kp[j].first);
                if (!single) U.push_back(kp[j].second);
            }
        }
        base += (uint64_t) m;
        blo = bhi;
    }
    const int k2bits = [&] { int x = 0; while ((uint64_t) 2 * n >> x) ++x; return x; }();
    // refinement rounds: pieces that end before the last group of a load that does not reach the end of the list
    for (int64_t h = FMI_K; !U.empty(); h *= 2) {
        if (++rounds > 40) return -3;
        const size_t nU = U.size();
        size_t u0 = 0, wcur = 0;
        while (u0 < nU) {
            const int64_t L = std::min<int64_t>(cap, (int64_t) (nU - u0));
            std::vector<uint64_t> g((size_t) L); std::vector<int> flag((size_t) L);
            int64_t last = 0;
            for (int64_t j = 0; j < L; ++j) {
                g[j] = fmi_get40(lo.data(), hi.data(), (int64_t) U[u0 + j]);
                flag[j] = j == 0 || g[j] != fmi_get40(lo.data(), hi.data(), (int64_t) U[u0 + j - 1]);
                if (flag[j]) last = j;
            }
            const int64_t P = u0 + (size_t) L < nU ? last : L;
            std::vector<std::pair<uint64_t, uint64_t>> kp((size_t) P);
            std::vector<uint64_t> gval; std::vector<int64_t> gfirst;
            for (int64_t j = 0, o = -1; j < P; ++j) {
                if (flag[j]) { ++o; gval.push_back(g[j]); gfirst.push_back(j); }
                kp[j] = { (uint64_t) o << k2bits | fmi_key2(lo.data(), hi.data(), n, (int64_t) U[u0 + j], h), U[u0 + j] };
            }
            std::stable_sort(kp.begin(), kp.end(), [](const auto &x, const auto &y) { return x.first < y.first; });
            int64_t start = 0;
            std::vector<uint64_t> kept;
            for (int64_t j = 0; j < P; ++j) {
                if (j == 0 || kp[j].first != kp[j - 1].first) start = j;
                const int64_t o = (int64_t) (kp[j].first >> k2bits);
                fmi_put40(lo.data(), hi.data(), (int64_t) kp[j].second, gval[o] + (uint64_t) (start - gfirst[o]));
                const bool single = start == j && (j + 1 == P || kp[j + 1].first != kp[j].first);
                if (!single) kept.push_back(kp[j].second);
            }
            std::copy(kept.begin(), kept.end(), U.begin() + wcur);
            wcur += kept.size(); u0 += (size_t) P; ++pieces;
        }
        U.resize(wcur);
    }
    // emit, one window of rows at a time
    const int64_t n_rows = n + 1, nb_all = (n_rows + 63) / 64;
    int64_t run[4] = { 0, 0, 0, 0 }, sentinel = -1;
    for (int64_t r0 = 0; r0 < nb_all * 64; r0 += win) {
        ++windows;
        const int64_t m = std::min(win, nb_all * 64 - r0);
        std::vector<uint64_t> sa((size_t) m, ~0ull);
        if (r0 == 0) sa[0] = (uint64_t) n;
        for (int64_t p = 0; p < n; ++p) {
            const int64_t r = (int64_t) fmi_get40(lo.data(), hi.data(), p) + 1;
            if (r >= r0 && r < r0 + m) { if (sa[r - r0] != ~0ull) return -1; sa[r - r0] = (uint64_t) p; }
        }
        std::vector<uint8_t> bw((size_t) m, 6);
        for (int64_t j = 0; j < m && r0 + j < n_rows; ++j) {
            if (sa[j] == ~0ull) return -2;
            bw[j] = fmi_bwt_char(w.data(), sa[j]);
            if (sa[j] == 0) sentinel = r0 + j;
            if (r0 + j > 0) sa_out[r0 + j - 1] = (int64_t) sa[j];
            if (((r0 + j) & 7) == 0) { ms_out[(r0 + j) >> 3] = (int8_t) (sa[j] >> 32 & 0xff); ls_out[(r0 + j) >> 3] = (uint32_t) sa[j]; }
        }
        for (int64_t k = 0; k < m / 64; ++k) {
            FmiCpOcc e; int64_t add[4];
            fmi_cp_entry(bw.data() + 64 * k, run, &e, add);
            memcpy(cp_out + 8 * ((r0 >> 6) + k), &e, sizeof e);
            for (int c = 0; c < 4; ++c) run[c] += add[c];
        }
    }
    info[0] = groups; info[1] = pieces; info[2] = rounds; info[3] = windows; info[4] = sentinel; info[5] = cap;
    return 0;
}

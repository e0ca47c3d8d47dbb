// bgzf_emul.cpp — TEST ONLY: bm2_bgzf_compress (bwa-mem2_b200/csrc/bgzf.cu) with plain loops over the same BM2_HD functions
// (bgzf_device.cuh), compiled with g++: the hash chain by its sequential definition, the segments parsed one after the other, the bits
// written in order.  The kernel must give these bytes exactly.
#include "bgzf_device.cuh"
#include <cstring>
#include <vector>

// one member of n <= BGZF_BLOCK bytes into o (room for BGZF_MAX_MEMBER); returns its size
extern "C" int bgzf_emul_block(const uint8_t *d, int n, uint8_t *o) {
    const int np = n >= 3 ? n - 2 : 0;
    std::vector<uint16_t> prev((size_t) n + 1, BGZF_NONE), head((size_t) 1 << BGZF_HASH_BITS, BGZF_NONE);
    for (int i = 0; i < np; ++i) { const uint32_t h = bgzf_hash3(d + i); prev[i] = head[h]; head[h] = (uint16_t) i; }
    uint32_t fll[288] = { 0 }, fd[32] = { 0 };
    fll[256] = 1;
    std::vector<uint16_t> items(BGZF_BLOCK + 1);
    std::vector<int> seg_n;
    const int nseg = (n + BGZF_SEG - 1) / BGZF_SEG;
    for (int t = 0; t < nseg; ++t)
        seg_n.push_back(bgzf_parse_segment(d, n, prev.data(), t * BGZF_SEG, bm2_min(n, (t + 1) * BGZF_SEG), items.data() + t * BGZF_SEG, fll, fd));
    static BgzfCodes c; static BgzfHuffTmp tmp; static BgzfHeaderTmp h;
    bgzf_huff_lengths(fll, 286, 15, c.ll_len, tmp);
    bgzf_huff_lengths(fd, 30, 15, c.d_len, tmp);
    std::vector<uint32_t> w((size_t) (n + 5) / 4 + 160, 0);
    const uint64_t hb = bgzf_write_header(c, h, tmp, w.data());
    uint64_t bits = hb;
    for (int t = 0; t < nseg; ++t) bits += bgzf_segment_bits(items.data() + t * BGZF_SEG, seg_n[t], c);
    const uint64_t eob = bits;
    bits += c.ll_len[256];
    const bool stored = (int64_t) ((bits + 7) / 8) >= (int64_t) n + 5;
    int body;
    if (stored) { bgzf_stored_head(o + 18, n); memcpy(o + 23, d, (size_t) n); body = n + 5; }
    else {
        uint64_t pos = hb;
        for (int t = 0; t < nseg; ++t) pos = bgzf_emit_segment(items.data() + t * BGZF_SEG, seg_n[t], c, w.data(), pos);
        if (pos != eob) return -1;
        bgzf_put(w.data(), eob, c.ll_code[256], c.ll_len[256]);
        body = (int) ((bits + 7) / 8);
        memcpy(o + 18, w.data(), (size_t) body);
    }
    const int member = 18 + body + 8;
    bgzf_member_head(o, member);
    bgzf_put32(o + 18 + body, ~bgzf_crc_raw(d, n, 0xFFFFFFFFu));
    bgzf_put32(o + 22 + body, (uint32_t) n);
    return member;
}

// the block starts of bm2_bgzf_compress (n_blocks + 1 values into starts, room for cap); returns n_blocks or -1
extern "C" int64_t bgzf_emul_cuts(int64_t n, const int64_t *cut, int64_t n_cut, int64_t *starts, int64_t cap) {
    std::vector<int64_t> s;
    const int64_t nb = bgzf_cut_blocks(n, cut, n_cut, s);
    if ((int64_t) s.size() > cap) return -1;
    memcpy(starts, s.data(), s.size() * sizeof(int64_t));
    return nb;
}

// the whole stream: the members of every block, concatenated; returns the byte count or -1 when out (cap bytes) is too small
extern "C" int64_t bgzf_emul(const uint8_t *in, int64_t n, const int64_t *cut, int64_t n_cut, uint8_t *out, int64_t cap) {
    std::vector<int64_t> s;
    const int64_t nb = bgzf_cut_blocks(n, cut, n_cut, s);
    std::vector<uint8_t> m(BGZF_MAX_MEMBER);
    int64_t at = 0;
    for (int64_t b = 0; b < nb; ++b) {
        const int k = bgzf_emul_block(in + s[b], (int) (s[b + 1] - s[b]), m.data());
        if (k < 0 || at + k > cap) return -1;
        memcpy(out + at, m.data(), (size_t) k); at += k;
    }
    return at;
}

// bgzf_device.cuh — the per-block logic of bm2_bgzf_compress (bgzf.cu): one BGZF member (SAMv1 §4.1) of up to 65280 input bytes, its raw
// DEFLATE data (RFC 1951) one dynamic Huffman block, or a stored block when that would not be smaller.
//
// The compressed bytes are a function of the block's bytes alone.  Each step is defined by a sequential rule; the kernel computes the same
// result in parallel and tests/host_emul/bgzf_emul.cpp computes it with plain loops over these BM2_HD functions:
//   chain      prev[i] = the largest j < i whose 3-byte hash equals that of i (a hash chain over the whole block)
//   parse      the block is cut into 256-byte segments; each is parsed greedily on its own: at p, the longest match among the first
//              BGZF_CHAIN candidates of the chain within 32 KiB (the nearest on ties, length 3..258, not past the segment's end), else a literal
//   codes      lit/len and distance code lengths from the symbol counts by Huffman's rule, counts halved until no code is longer than 15
//              bits (7 for the code-length code); canonical codes as RFC 1951 §3.2.2
//   packing    header, then the segments' symbols in order, then end-of-block: each segment's bits start at the sum of the bit lengths
//              of the ones before it
#pragma once
#include "hd.h"

#define BGZF_BLOCK 65280              // input bytes per member at most (htslib's BGZF_BLOCK_SIZE, 0xff00)
#define BGZF_MAX_MEMBER 65536         // bytes per member at most (BSIZE is 16 bits)
#define BGZF_SEG 256                  // input bytes per parse segment (one thread each)
#define BGZF_NSEG (BGZF_BLOCK / BGZF_SEG)
#define BGZF_HASH_BITS 12
#define BGZF_CHAIN 16                 // chain candidates tried per position
#define BGZF_NICE 128                 // a match this long ends the search
#define BGZF_NONE 0xFFFFu
#define BGZF_WINDOW 32768
#define BGZF_POLY 0xEDB88320u

BM2_HD uint32_t bgzf_hash3(const uint8_t *d) { return ((uint32_t) d[0] << 16 | (uint32_t) d[1] << 8 | d[2]) * 2654435761u >> (32 - BGZF_HASH_BITS); }

// ---- counts and bit writes: atomic on the device (several threads share a word), plain on the host ----
BM2_HD void bgzf_inc(uint32_t *p) {
#if defined(__CUDA_ARCH__)
    atomicAdd(p, 1u);
#else
    ++*p;
#endif
}
BM2_HD void bgzf_or(uint32_t *p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
// nb <= 32 bits of v at bit position pos of the LSB-first stream w (zeroed beforehand)
BM2_HD void bgzf_put(uint32_t *w, uint64_t pos, uint32_t v, int nb) {
    if (!nb) return;
    const int s = (int) (pos & 31);
    const uint64_t k = pos >> 5;
    bgzf_or(w + k, v << s);
    if (s + nb > 32) bgzf_or(w + k + 1, v >> (32 - s));
}

// ---- DEFLATE's length and distance codes (RFC 1951 §3.2.5) ----
BM2_HD int bgzf_log2(uint32_t x) { int b = 0; while (x >> (b + 1)) ++b; return b; }
// length 3..258 -> symbol 257..285, extra bits and their value
BM2_HD void bgzf_len_code(int len, int &sym, int &nx, int &xv) {
    const int x = len - 3;
    if (len == 258) { sym = 285; nx = 0; xv = 0; }
    else if (x < 8) { sym = 257 + x; nx = 0; xv = 0; }
    else { const int b = bgzf_log2((uint32_t) x); sym = 257 + 4 * (b - 1) + ((x >> (b - 2)) & 3); nx = b - 2; xv = x & ((1 << (b - 2)) - 1); }
}
// distance 1..32768 -> symbol 0..29, extra bits and their value
BM2_HD void bgzf_dist_code(int dist, int &sym, int &nx, int &xv) {
    const int x = dist - 1;
    if (x < 4) { sym = x; nx = 0; xv = 0; }
    else { const int b = bgzf_log2((uint32_t) x); sym = 2 * b + ((x >> (b - 1)) & 1); nx = b - 1; xv = x & ((1 << (b - 1)) - 1); }
}

// ---- CRC-32 (the gzip polynomial, reflected) as polynomial arithmetic modulo P, so that pieces computed apart combine ----
BM2_HD uint32_t bgzf_multmodp(uint32_t a, uint32_t b) {      // a * b mod P; a != 0
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ BGZF_POLY : b >> 1;
    }
    return p;
}
struct BgzfX2n { uint32_t p[32]; };                          // x^(2^k) mod P
BM2_HD BgzfX2n bgzf_x2n() {
    BgzfX2n t; t.p[0] = 1u << 30;
    for (int k = 1; k < 32; ++k) t.p[k] = bgzf_multmodp(t.p[k - 1], t.p[k - 1]);
    return t;
}
BM2_HD uint32_t bgzf_xpow(const BgzfX2n &t, uint64_t e) {    // x^e mod P
    uint32_t p = 1u << 31;
    for (int k = 0; e; ++k, e >>= 1) if (e & 1) p = bgzf_multmodp(t.p[k], p);
    return p;
}
BM2_HD uint32_t bgzf_crc_raw(const uint8_t *d, int n, uint32_t c) {     // no pre- or post-inversion
    for (int i = 0; i < n; ++i) { c ^= d[i]; for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ BGZF_POLY : c >> 1; }
    return c;
}

// ---- the chain walk and greedy parse of one segment [s, e) ----
// items: a literal is its byte (< 256); a match is 256 + len - 3, then dist - 1.  Returns the item count (<= e - s).
// fll[286] / fd[30]: symbol counts, incremented
BM2_HD int bgzf_parse_segment(const uint8_t *d, int n, const uint16_t *prev, int s, int e, uint16_t *items, uint32_t *fll, uint32_t *fd) {
    int p = s, k = 0;
    while (p < e) {
        int best = 0, bd = 0;
        const int maxl = bm2_min(258, e - p);
        if (maxl >= 3 && p + 3 <= n) {
            uint32_t j = prev[p];
            for (int c = 0; c < BGZF_CHAIN && j != BGZF_NONE && p - (int) j <= BGZF_WINDOW; ++c, j = prev[j]) {
                if (d[j + best] != d[p + best]) continue;
                int l = 0;
                while (l < maxl && d[j + l] == d[p + l]) ++l;
                if (l > best) { best = l; bd = p - (int) j; if (l >= BGZF_NICE || l == maxl) break; }
            }
        }
        if (best >= 3) {
            int sym, nx, xv;
            items[k++] = (uint16_t) (256 + best - 3); items[k++] = (uint16_t) (bd - 1);
            bgzf_len_code(best, sym, nx, xv); bgzf_inc(fll + sym);
            bgzf_dist_code(bd, sym, nx, xv); bgzf_inc(fd + sym);
            p += best;
        } else { items[k++] = d[p]; bgzf_inc(fll + d[p]); ++p; }
    }
    return k;
}

// ---- Huffman code lengths ----
struct BgzfHuffTmp {
    uint64_t key[288];                // (count << 16 | symbol) of the used symbols, sorted
    uint32_t f[288];                  // working counts
    uint32_t w[288];                  // weights of the internal nodes
    int16_t parent[576];              // leaves 0..m-1 (sorted order), internal nodes m..
    uint8_t depth[576];
};
// lengths of nsym symbols (<= 286) from their counts, none longer than limit; at least two codes, as zlib's build_tree makes them
BM2_HD void bgzf_huff_lengths(const uint32_t *freq, int nsym, int limit, uint8_t *len, BgzfHuffTmp &t) {
    int m = 0;
    for (int i = 0; i < nsym; ++i) { len[i] = 0; t.f[i] = freq[i]; if (freq[i]) ++m; }
    if (m < 2) {
        int got = 0;
        for (int i = 0; i < nsym && got < 2; ++i) if (freq[i]) { len[i] = 1; ++got; }
        for (int i = 0; i < nsym && got < 2; ++i) if (!len[i]) { len[i] = 1; ++got; }
        return;
    }
    for (;;) {
        int k = 0;
        for (int i = 0; i < nsym; ++i) if (t.f[i]) t.key[k++] = (uint64_t) t.f[i] << 16 | (uint64_t) i;
        for (int gap = m / 2; gap > 0; gap /= 2)                 // shell sort, ascending
            for (int i = gap; i < m; ++i) {
                const uint64_t v = t.key[i]; int j = i;
                while (j >= gap && t.key[j - gap] > v) { t.key[j] = t.key[j - gap]; j -= gap; }
                t.key[j] = v;
            }
        // two queues: leaves in order, internal nodes in creation order (their weights never decrease); a leaf wins ties
        int li = 0, ii = 0, ni = 0;
        for (int c = 0; c < m - 1; ++c) {
            uint32_t wsum = 0;
            for (int h = 0; h < 2; ++h) {
                const bool leaf = li < m && (ii >= ni || (uint32_t) (t.key[li] >> 16) <= t.w[ii]);
                if (leaf) { wsum += (uint32_t) (t.key[li] >> 16); t.parent[li++] = (int16_t) (m + ni); }
                else { wsum += t.w[ii]; t.parent[m + ii++] = (int16_t) (m + ni); }
            }
            t.w[ni++] = wsum;
        }
        int maxd = 0;
        t.depth[m + ni - 1] = 0;
        for (int x = m + ni - 2; x >= 0; --x) { t.depth[x] = (uint8_t) (t.depth[t.parent[x]] + 1); if (x < m && t.depth[x] > maxd) maxd = t.depth[x]; }
        if (maxd <= limit) {
            for (int x = 0; x < m; ++x) len[t.key[x] & 0xFFFF] = t.depth[x];
            return;
        }
        for (int i = 0; i < nsym; ++i) if (t.f[i]) t.f[i] = (t.f[i] + 1) >> 1;
    }
}
// canonical codes (RFC 1951 §3.2.2), bit-reversed for the LSB-first stream
BM2_HD void bgzf_huff_codes(const uint8_t *len, int nsym, uint16_t *code) {
    int count[16] = { 0 }, next[16] = { 0 };
    for (int i = 0; i < nsym; ++i) ++count[len[i]];
    count[0] = 0;
    for (int b = 1, c = 0; b < 16; ++b) { c = (c + count[b - 1]) << 1; next[b] = c; }
    for (int i = 0; i < nsym; ++i) {
        if (!len[i]) { code[i] = 0; continue; }
        const uint32_t c = (uint32_t) next[len[i]]++;
        uint32_t r = 0;
        for (int b = 0; b < len[i]; ++b) r |= ((c >> b) & 1) << (len[i] - 1 - b);
        code[i] = (uint16_t) r;
    }
}

struct BgzfCodes {
    uint16_t ll_code[288], d_code[32];
    uint8_t ll_len[288], d_len[32];
};

// bit length of a segment's items
BM2_HD uint64_t bgzf_segment_bits(const uint16_t *items, int k, const BgzfCodes &c) {
    uint64_t b = 0;
    for (int i = 0; i < k; ++i) {
        const int v = items[i];
        if (v < 256) { b += c.ll_len[v]; continue; }
        int sym, nx, xv;
        bgzf_len_code(v - 256 + 3, sym, nx, xv); b += c.ll_len[sym] + nx;
        bgzf_dist_code(items[++i] + 1, sym, nx, xv); b += c.d_len[sym] + nx;
    }
    return b;
}
BM2_HD uint64_t bgzf_emit_segment(const uint16_t *items, int k, const BgzfCodes &c, uint32_t *w, uint64_t pos) {
    for (int i = 0; i < k; ++i) {
        const int v = items[i];
        if (v < 256) { bgzf_put(w, pos, c.ll_code[v], c.ll_len[v]); pos += c.ll_len[v]; continue; }
        int sym, nx, xv;
        bgzf_len_code(v - 256 + 3, sym, nx, xv);
        bgzf_put(w, pos, c.ll_code[sym], c.ll_len[sym]); pos += c.ll_len[sym];
        bgzf_put(w, pos, (uint32_t) xv, nx); pos += nx;
        bgzf_dist_code(items[++i] + 1, sym, nx, xv);
        bgzf_put(w, pos, c.d_code[sym], c.d_len[sym]); pos += c.d_len[sym];
        bgzf_put(w, pos, (uint32_t) xv, nx); pos += nx;
    }
    return pos;
}

// ---- the dynamic block's header (RFC 1951 §3.2.7): codes from the counts (fll[256] must already count the end-of-block), header bits written
// at bit 0 of w; returns the header's bit length ----
struct BgzfHeaderTmp {
    uint8_t all[320];                 // lit/len then distance code lengths
    uint8_t rle[320], rle_x[320];     // code-length symbols and their extra values
    uint32_t fcl[19];
    uint8_t cl_len[19];
    uint16_t cl_code[19];
};
BM2_HD uint64_t bgzf_write_header(BgzfCodes &c, BgzfHeaderTmp &h, BgzfHuffTmp &t, uint32_t *w) {
    const unsigned char *order = (const unsigned char *) "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f";     // RFC 1951 §3.2.7
    bgzf_huff_codes(c.ll_len, 286, c.ll_code);
    bgzf_huff_codes(c.d_len, 30, c.d_code);
    int hlit = 286, hdist = 30;
    while (hlit > 257 && !c.ll_len[hlit - 1]) --hlit;
    while (hdist > 1 && !c.d_len[hdist - 1]) --hdist;
    const int na = hlit + hdist;
    for (int i = 0; i < hlit; ++i) h.all[i] = c.ll_len[i];
    for (int i = 0; i < hdist; ++i) h.all[hlit + i] = c.d_len[i];
    int nr = 0;
    for (int i = 0; i < 19; ++i) h.fcl[i] = 0;
    for (int i = 0; i < na;) {
        const int v = h.all[i];
        int r = 1;
        while (i + r < na && h.all[i + r] == v) ++r;
        i += r;
        if (v == 0) {
            while (r >= 11) { const int q = bm2_min(r, 138); h.rle[nr] = 18; h.rle_x[nr++] = (uint8_t) (q - 11); r -= q; }
            if (r >= 3) { h.rle[nr] = 17; h.rle_x[nr++] = (uint8_t) (r - 3); r = 0; }
        } else {
            h.rle[nr] = (uint8_t) v; h.rle_x[nr++] = 0; --r;
            while (r >= 3) { const int q = bm2_min(r, 6); h.rle[nr] = 16; h.rle_x[nr++] = (uint8_t) (q - 3); r -= q; }
        }
        while (r-- > 0) { h.rle[nr] = (uint8_t) v; h.rle_x[nr++] = 0; }
    }
    for (int i = 0; i < nr; ++i) ++h.fcl[h.rle[i]];
    bgzf_huff_lengths(h.fcl, 19, 7, h.cl_len, t);
    bgzf_huff_codes(h.cl_len, 19, h.cl_code);
    int hclen = 19;
    while (hclen > 4 && !h.cl_len[order[hclen - 1]]) --hclen;
    uint64_t pos = 0;
    bgzf_put(w, pos, 1 | 2 << 1, 3); pos += 3;                     // BFINAL, BTYPE = 10 (dynamic)
    bgzf_put(w, pos, (uint32_t) (hlit - 257), 5); pos += 5;
    bgzf_put(w, pos, (uint32_t) (hdist - 1), 5); pos += 5;
    bgzf_put(w, pos, (uint32_t) (hclen - 4), 4); pos += 4;
    for (int i = 0; i < hclen; ++i) { bgzf_put(w, pos, h.cl_len[order[i]], 3); pos += 3; }
    for (int i = 0; i < nr; ++i) {
        const int s = h.rle[i];
        bgzf_put(w, pos, h.cl_code[s], h.cl_len[s]); pos += h.cl_len[s];
        const int nx = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
        bgzf_put(w, pos, h.rle_x[i], nx); pos += nx;
    }
    return pos;
}

// ---- the member around the DEFLATE data: gzip header with the BC subfield (18 bytes), then CRC32 and ISIZE (8 bytes) ----
BM2_HD void bgzf_member_head(uint8_t *o, int member_bytes) {
    const uint8_t h[16] = { 0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0 };
    for (int i = 0; i < 16; ++i) o[i] = h[i];
    o[16] = (uint8_t) ((member_bytes - 1) & 0xff); o[17] = (uint8_t) ((member_bytes - 1) >> 8);
}
BM2_HD void bgzf_put32(uint8_t *o, uint32_t v) { o[0] = (uint8_t) v; o[1] = (uint8_t) (v >> 8); o[2] = (uint8_t) (v >> 16); o[3] = (uint8_t) (v >> 24); }
// the stored block of n bytes: BFINAL = 1, BTYPE = 00, LEN, NLEN (then the n bytes)
BM2_HD void bgzf_stored_head(uint8_t *o, int n) { o[0] = 1; o[1] = (uint8_t) n; o[2] = (uint8_t) (n >> 8); o[3] = (uint8_t) ~n; o[4] = (uint8_t) (~n >> 8); }

// ---- block cuts, as htslib's writer cuts them (bam_write1 -> bgzf_flush_try, bgzf_write): a record that would overflow a non-empty block
// starts a new one; a block that reaches BGZF_BLOCK bytes is closed there, so a record larger than a block spans blocks.  The records are
// [cut[i], cut[i+1]) with cut ascending; bytes before cut[0] form a record of their own, the last record ends at n.  starts gets the block
// starts and n; returns the block count ----
template <class V> inline int64_t bgzf_cut_blocks(int64_t n, const int64_t *cut, int64_t n_cut, V &starts) {
    int64_t off = 0, b0 = 0, nb = 0;
    auto close = [&](int64_t at) { starts.push_back(b0); b0 = at; off = 0; ++nb; };
    for (int64_t i = -1; i < n_cut; ++i) {
        const int64_t s = i < 0 ? 0 : cut[i], e = i + 1 < n_cut ? cut[i + 1] : n;
        if (e <= s) continue;
        if (off > 0 && off + (e - s) > BGZF_BLOCK) close(s);
        for (int64_t p = s; p < e;) {
            const int64_t take = bm2_min<int64_t>(BGZF_BLOCK - off, e - p);
            off += take; p += take;
            if (off == BGZF_BLOCK) close(p);
        }
    }
    if (off > 0) close(n);
    starts.push_back(n);
    return nb;
}

// read_input.h — a whole input file into memory, plain or gzip, as the reference reads its inputs through zlib.  Shared by bm2_mem (reads)
// and bm2_fasta_pack (the FASTA of bm2_index), so that both accept the same inputs.
#pragma once
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>
#include <zlib.h>

// gzip bytes in memory (every member of a multi-member file, as gzread reads them) -> out
static inline bool gunzip_mem(const std::vector<char> &in, std::vector<char> &out) {
    z_stream zs; memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, 15 + 16) != Z_OK) return false;
    out.resize(in.size() * 4 + ((size_t) 1 << 20));
    size_t at = 0, n = 0;
    for (;;) {
        zs.next_in = (Bytef *) in.data() + at; zs.avail_in = (uInt) std::min<size_t>(in.size() - at, (size_t) 1 << 30);
        zs.next_out = (Bytef *) out.data() + n; zs.avail_out = (uInt) std::min<size_t>(out.size() - n, (size_t) 1 << 30);
        const size_t in0 = zs.avail_in, out0 = zs.avail_out;
        const int r = inflate(&zs, Z_NO_FLUSH);
        at += in0 - zs.avail_in; n += out0 - zs.avail_out;
        if (r == Z_STREAM_END) {
            if (at + 2 <= in.size() && (unsigned char) in[at] == 0x1f && (unsigned char) in[at + 1] == 0x8b) { inflateReset(&zs); continue; }
            break;
        }
        if (r != Z_OK && r != Z_BUF_ERROR) { inflateEnd(&zs); return false; }
        if (r == Z_BUF_ERROR && zs.avail_in == 0 && at >= in.size()) { inflateEnd(&zs); return false; }     // truncated
        if (out.size() - n < ((size_t) 16 << 20)) out.resize(out.size() * 2);
    }
    inflateEnd(&zs);
    out.resize(n);
    return true;
}

// the whole file into memory; gzip files (magic 1f 8b) through zlib, as the reference reads its input through zlib (gzdopen + kseq, src/fastmap.cpp:
// 905-907, :933-935) - gzread also passes plain files through, but the plain path below needs no copy loop.  "-" is standard input (kopen,
// src/kopen.c), plain or gzip by the same magic bytes, inflated in memory.
static inline bool read_file(const char *path, std::vector<char> &buf) {
    if (!strcmp(path, "-")) {
        std::vector<char> raw((size_t) 64 << 20);
        size_t n = 0;
        for (;;) {
            if (raw.size() - n < ((size_t) 16 << 20)) raw.resize(raw.size() * 2);
            const size_t r = fread(raw.data() + n, 1, raw.size() - n, stdin);
            n += r;
            if (r == 0) { if (ferror(stdin)) return false; break; }
        }
        raw.resize(n);
        if (n >= 2 && (unsigned char) raw[0] == 0x1f && (unsigned char) raw[1] == 0x8b) return gunzip_mem(raw, buf);
        buf.swap(raw);
        return true;
    }
    FILE *f = fopen(path, "rb");
    if (!f) return false;
    unsigned char magic[2] = {0, 0};
    const size_t got = fread(magic, 1, 2, f);
    if (got == 2 && magic[0] == 0x1f && magic[1] == 0x8b) {
        fclose(f);
        gzFile g = gzopen(path, "rb");
        if (!g) return false;
        gzbuffer(g, 1 << 20);
        size_t n = 0;
        buf.resize((size_t) 64 << 20);
        for (;;) {
            if (buf.size() - n < ((size_t) 16 << 20)) buf.resize(buf.size() * 2);
            const size_t want = buf.size() - n < ((size_t) 1 << 30) ? buf.size() - n : ((size_t) 1 << 30);
            const int r = gzread(g, buf.data() + n, (unsigned) want);
            if (r < 0) { gzclose(g); return false; }
            if (r == 0) break;
            n += (size_t) r;
        }
        gzclose(g);
        buf.resize(n);
        return true;
    }
    fseek(f, 0, SEEK_END); const long n = ftell(f); fseek(f, 0, SEEK_SET);
    buf.resize((size_t) n);
    const bool ok = n == 0 || fread(buf.data(), 1, (size_t) n, f) == (size_t) n;
    fclose(f);
    return ok;
}

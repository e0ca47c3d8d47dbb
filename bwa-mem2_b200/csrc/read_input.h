// read_input.h — the inputs of bm2_mem (reads) and of bm2_fasta_pack (the FASTA of bm2_index), read as the reference reads them through zlib
// (gzdopen + kseq, src/fastmap.cpp:905-907, :933-935; kopen for "-", src/kopen.c): plain or gzip by the magic bytes 1f 8b, every member of a
// multi-member file (BGZF included), bytes after the last member ignored, and an input cut inside a member read up to the cut (gzread's
// rules; a corrupt member is an error).
//
// One mechanism for every source: InputStream reads its file descriptor (a file, or standard input for "-") with read() and hands out the
// decompressed bytes piece by piece, so that its memory does not depend on the input's size (plain files are not mapped: mapped pages would
// count as resident memory too).
//
// chunk_stream is bm2_mem's chunker over such a source: it walks records with seq_record (seq_grammar.cuh) over a window of the stream
// refilled by read(), and cuts exactly the chunks that the whole input in memory gives.  tests/host_emul/stream_emul.cpp compiles it against
// a fake source.
#pragma once
#include "seq_grammar.cuh"
#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <fcntl.h>
#include <functional>
#include <string>
#include <unistd.h>
#include <vector>
#include <zlib.h>

// bytes in pieces: read() gives at least one byte, 0 at the end of the input, -1 on an error
struct ByteSource {
    virtual ~ByteSource() {}
    virtual int64_t read(char *dst, size_t cap) = 0;
};

class InputStream : public ByteSource {
public:
    std::string error_msg;
    int64_t gzip_members = 0;
    bool truncated = false;                                         // the input ended inside a gzip member
    size_t peak_bytes() const { return in_.capacity(); }
    const char *path() const { return path_; }

    InputStream() { memset(&zs_, 0, sizeof zs_); }
    ~InputStream() { if (zinit_) inflateEnd(&zs_); if (fd_ > 0) close(fd_); }
    InputStream(const InputStream &) = delete;
    InputStream &operator=(const InputStream &) = delete;

    // "-" is standard input; the format is decided by the first two bytes
    bool open(const char *path) {
        path_ = path;
        fd_ = strcmp(path, "-") ? ::open(path, O_RDONLY) : 0;
        if (fd_ < 0) return fail("cannot open");
        in_.resize((size_t) 1 << 20);
        while (len_ < 2 && !raw_eof_) if (!fill()) return false;
        gz_ = len_ >= 2 && (unsigned char) in_[0] == 0x1f && (unsigned char) in_[1] == 0x8b;
        if (gz_) {
            if (inflateInit2(&zs_, 15 + 16) != Z_OK) return fail("zlib initialisation failed");
            zinit_ = true;
        }
        return true;
    }

    int64_t read(char *dst, size_t cap) override {
        if (cap == 0) return 0;
        if (!gz_) {
            if (at_ < len_) { const size_t k = std::min(cap, len_ - at_); memcpy(dst, in_.data() + at_, k); at_ += k; return (int64_t) k; }
            if (raw_eof_) return 0;
            for (;;) {
                const ssize_t r = ::read(fd_, dst, cap);
                if (r < 0 && errno == EINTR) continue;
                if (r < 0) { fail("read error"); return -1; }
                if (r == 0) raw_eof_ = true;
                return (int64_t) r;
            }
        }
        for (;;) {
            if (!in_member_) {                                      // a member boundary
                if (len_ - at_ < 2 && !raw_eof_) { if (!fill()) return -1; continue; }
                if (len_ - at_ < 2 || (unsigned char) in_[at_] != 0x1f || (unsigned char) in_[at_ + 1] != 0x8b) return 0;   // end; trailing bytes ignored
                inflateReset(&zs_); in_member_ = true; ++gzip_members;
            }
            if (at_ == len_ && !raw_eof_) { if (!fill()) return -1; continue; }
            zs_.next_in = (Bytef *) in_.data() + at_; zs_.avail_in = (uInt) (len_ - at_);
            zs_.next_out = (Bytef *) dst; zs_.avail_out = (uInt) std::min(cap, (size_t) 1 << 30);
            const uInt out0 = zs_.avail_out;
            const int r = inflate(&zs_, Z_NO_FLUSH);      // with no input left it still gives what it holds (the rest of a match)
            at_ = len_ - zs_.avail_in;
            if (r == Z_STREAM_END) in_member_ = false;
            else if (r != Z_OK && r != Z_BUF_ERROR) { fail(zs_.msg ? zs_.msg : "corrupt gzip data"); return -1; }
            if (out0 != zs_.avail_out) return (int64_t) (out0 - zs_.avail_out);
            // the input ends inside a member: the end, after the bytes inflated so far - gzread records "unexpected end of file" there but
            // returns those bytes and then 0, so kseq (and the reference) read a truncated file as far as it goes
            if (at_ == len_ && raw_eof_) { truncated = true; return 0; }
        }
    }

private:
    const char *path_ = "";
    int fd_ = -1;
    bool gz_ = false, raw_eof_ = false, in_member_ = false, zinit_ = false;
    std::vector<char> in_; size_t at_ = 0, len_ = 0;             // compressed bytes read and not yet inflated: [at_, len_)
    z_stream zs_;

    bool fail(const char *what) { error_msg = std::string(path_) + ": " + what; return false; }

    // more raw bytes into in_: one read (it may wait for a pipe's writer, but not for more than the first bytes it sends)
    bool fill() {
        if (at_ == len_) at_ = len_ = 0;
        else if (at_ > 0) { memmove(in_.data(), in_.data() + at_, len_ - at_); len_ -= at_; at_ = 0; }
        for (;;) {
            const ssize_t r = ::read(fd_, in_.data() + len_, in_.size() - len_);
            if (r < 0 && errno == EINTR) continue;
            if (r < 0) return fail("read error");
            if (r == 0) raw_eof_ = true;
            len_ += (size_t) r;
            return true;
        }
    }
};

// the whole input into memory
static inline bool read_file(const char *path, std::vector<char> &buf) {
    InputStream s;
    if (!s.open(path)) return false;
    buf.assign((size_t) 1 << 20, 0);
    size_t n = 0;
    for (;;) {
        if (buf.size() - n < ((size_t) 1 << 19)) buf.resize(buf.size() * 2);
        const int64_t r = s.read(buf.data() + n, buf.size() - n);
        if (r < 0) return false;
        if (r == 0) break;
        n += (size_t) r;
    }
    buf.resize(n);
    return true;
}

// ---- the chunker -----------------------------------------------------------------------------------------------------------------------

// a chunk: the bytes from its first record's header character to the next chunk's (junk between records included), copied out of the
// stream (c1 / c2 point into bytes), with their absolute offsets in the input; simple: every record is a simple four-line FASTQ record
// (seq_record) that ends where the next one starts, so bm2_fastq_encode parses it as kseq does
struct Chunk {
    long long index = 0, first_read = 0;
    int64_t off1 = 0, off2 = 0;
    std::vector<char> bytes;
    const char *c1 = nullptr, *c2 = nullptr; size_t n1 = 0, n2 = 0;
    bool simple = false;
};

// the decompressed bytes [base, base + n) of a source; refill() reads once more and may drop the bytes before a given offset
struct InputWindow {
    ByteSource &src;
    std::vector<char> buf;
    int64_t base = 0, n = 0;
    bool eof = false;
    explicit InputWindow(ByteSource &s, size_t cap = (size_t) 1 << 20) : src(s), buf(cap) {}
    int64_t end() const { return base + n; }
    bool refill(int64_t keep) {
        if (eof) return true;
        if (n == (int64_t) buf.size()) {
            const int64_t drop = std::min(keep, end()) - base;
            if (drop > 0) { memmove(buf.data(), buf.data() + drop, (size_t) (n - drop)); base += drop; n -= drop; }
            if (2 * n > (int64_t) buf.size()) buf.resize(buf.size() * 2);
        }
        const int64_t r = src.read(buf.data() + n, buf.size() - (size_t) n);
        if (r < 0) return false;
        if (r == 0) eof = true;
        n += r;
        return true;
    }
    // the first header character at or after p (absolute), or the end of the input; the bytes before it are no longer needed
    bool hdr(int64_t p, int64_t &h) {
        for (;;) {
            const SeqHostSrc s = { buf.data(), n };
            const int64_t q = s.hdr(std::max(p, base) - base);
            if (q < n || eof) { h = base + q; return true; }
            p = end();
            if (!refill(p)) return false;
        }
    }
    // one seq_record walk from the header character at h (absolute) that more input cannot change: it found the next record's header
    // before the window's end, or it is malformed there, or the input is exhausted; otherwise refill and walk again from the header.
    // end and next come back absolute.  Bytes before keep may be dropped.
    bool record(int64_t keep, int64_t h, SeqRec &r) {
        for (;;) {
            const SeqHostSrc s = { buf.data(), n };
            r = seq_record(s, h - base, SeqNullSink());
            if (eof || r.next < n || (r.status == SEQ_BAD && r.end < n)) break;
            if (!refill(keep)) return false;
        }
        r.end += base; r.next += base;
        return true;
    }
};

// records (kseq_read, restated in seq_grammar.cuh) until the base count reaches the task size at an even record count (bseq_read_orig,
// src/bwa.cpp:204), mates kept together; emit() gets every chunk in order and owns it.  Returns the number of chunks, or -1 with err set.
// Memory: the two windows hold the current chunk and the record being walked; emitted chunks are the caller's.
inline long long chunk_stream(ByteSource &src1, ByteSource *src2, long long task, const std::function<void(Chunk &&)> &emit, std::string &err,
                              size_t window = (size_t) 1 << 20, size_t *window_peak = nullptr) {
    const bool paired = src2 != nullptr;
    InputWindow w1(src1, window), w2(paired ? *src2 : src1, paired ? window : 0);
    auto peak = [&] { if (window_peak) *window_peak = std::max(*window_peak, w1.buf.capacity() + w2.buf.capacity()); };
    const char *read_err = "cannot read the input files";
    int64_t h1 = 0, h2 = 0;
    if (!w1.hdr(0, h1) || (paired && !w2.hdr(0, h2))) { err = read_err; return -1; }
    long long n_chunks = 0, first_read = 0, n_file[2] = { 0, 0 };
    int64_t last_end[2] = { 0, 0 };                  // end of the last record read from each file
    // l_seq; -1: no record left; -2: an error
    auto next = [&](InputWindow &w, int64_t keep, int64_t &h, int file, bool *simple) -> int64_t {
        SeqRec r;
        if (!w.record(keep, h, r)) { err = read_err; return -2; }
        if (r.status == SEQ_NONE) return -1;          // h stays: a header character at the end of the input is not part of any chunk
        if (r.status == SEQ_BAD) {
            char m[128]; snprintf(m, sizeof m, "malformed record %lld of the %s file (a '+' line without qualities, or qualities of another length)",
                                  n_file[file], file ? "2nd" : "1st");
            err = m;
            return -2;
        }
        ++n_file[file];
        *simple = *simple && r.simple && r.next == r.end;
        last_end[file] = r.end;
        h = r.next;
        return r.l_seq;
    };
    bool more = true;
    while (more) {
        const int64_t c1 = h1, c2 = h2; long long size = 0, n_rec = 0;
        bool simple = true;
        for (;;) {
            const int64_t l1 = next(w1, c1, h1, 0, &simple);
            if (l1 == -2) return -1;
            if (l1 < 0) { more = false; break; }
            size += l1; ++n_rec;
            if (paired) {
                const int64_t l2 = next(w2, c2, h2, 1, &simple);
                if (l2 == -2) return -1;
                if (l2 < 0) { err = "the 2nd file has fewer sequences"; return -1; }
                size += l2; ++n_rec;
            }
            if (size >= task && (n_rec & 1) == 0) break;
        }
        peak();
        if (n_rec == 0) break;
        // bm2_fastq_encode takes the chunk's bytes whole: they must end where its last record ends
        if (h1 != last_end[0] || (paired && h2 != last_end[1])) simple = false;
        Chunk ck;
        ck.index = n_chunks++; ck.first_read = first_read; ck.off1 = c1; ck.off2 = c2; ck.simple = simple;
        ck.n1 = (size_t) (h1 - c1); ck.n2 = (size_t) (paired ? h2 - c2 : 0);
        ck.bytes.resize(ck.n1 + ck.n2);
        memcpy(ck.bytes.data(), w1.buf.data() + (c1 - w1.base), ck.n1);
        if (paired) memcpy(ck.bytes.data() + ck.n1, w2.buf.data() + (c2 - w2.base), ck.n2);
        ck.c1 = ck.bytes.data(); ck.c2 = paired ? ck.bytes.data() + ck.n1 : nullptr;
        first_read += n_rec;
        emit(std::move(ck));
    }
    if (paired) {
        SeqRec r;
        if (!w2.record(h2, h2, r)) { err = read_err; return -1; }
        if (r.status != SEQ_NONE) fprintf(stderr, "[W::bm2_mem] the 1st file has fewer sequences.\n");
    }
    return n_chunks;
}

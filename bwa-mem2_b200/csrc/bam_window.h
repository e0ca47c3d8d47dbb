// bam_window.h — a BAM file read in windows of whole records, in bounded host memory (bm2_applybqsr).  Host only, so that
// tests/host_emul/applybqsr_emul.cpp compiles the same reader.
//
//   members   read one after the other from the stream (a file or standard input).  Each must be a gzip member with the BC extra subfield
//             (SAMv1 §4.1); anything else is "not BGZF".  A member cut short is an error.  Empty members are skipped; when the input does
//             not end with one (the EOF block), `warning` says so, as htslib warns, and the records read stand.
//   windows   members are read until about `window` uncompressed bytes are held, then inflated by zlib on `threads` threads (bgzf_inflate,
//             shared with the sorted-run merge).  The whole records among them are the window; the bytes of an unfinished record wait for
//             the next one.  A record larger than the window makes its window larger.  The record boundaries are found here, and each
//             record's fixed fields are checked to lie inside it.  The input ending inside a record is an error.
//   header    SAMv1 §4.2: the magic BAM\1, the text, the references; otherwise "not BAM".
#pragma once
#include "bam_sort.h"
#include <cstdio>
#include <string>
#include <vector>

struct BamWindowReader {
    FILE *f = nullptr;
    std::string name;                              // for the messages
    int threads = 1;
    int64_t window = (int64_t) 256 << 20;
    // stats
    double inflate_s = 0;                          // the inflate threads' time, summed
    int64_t in_bytes = 0, members = 0, records = 0;
    std::string warning;                           // set once the input has ended without an EOF block
    // state
    std::vector<uint8_t> rest;                     // inflated bytes not handed out yet (an unfinished record)
    bool ended = false, last_empty = false;
    std::vector<std::vector<uint8_t>> z;           // the compressed members of one fill

    std::string where() const { return name + ": "; }

    // reads and inflates members until at least `want` bytes are held or the input ends
    std::string fill(size_t want) {
        while (!ended && rest.size() < want) {
            std::vector<InflateJob> jobs;
            size_t have = rest.size(), nz = 0;
            const size_t goal = std::max(want, rest.size() + (size_t) window);
            while (have < goal) {
                uint8_t h[12];
                const size_t got = fread(h, 1, 12, f);
                if (got == 0 && feof(f)) { ended = true; break; }
                if (got < 12) return where() + (members || got ? "a truncated BGZF member" : "cannot read the input");
                if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) return where() + "not BGZF (a member without the gzip magic and extra field)";
                const size_t xlen = (size_t) (h[10] | h[11] << 8);
                if (nz == z.size()) z.emplace_back();
                std::vector<uint8_t> &m = z[nz];
                m.assign(h, h + 12);
                m.resize(12 + xlen);
                if (fread(m.data() + 12, 1, xlen, f) != xlen) return where() + "a truncated BGZF member";
                int64_t bsize = -1;
                for (size_t p = 12; p + 4 <= 12 + xlen;) {
                    const size_t sl = (size_t) (m[p + 2] | m[p + 3] << 8);
                    if (m[p] == 66 && m[p + 1] == 67 && sl == 2 && p + 6 <= 12 + xlen) bsize = (int64_t) (m[p + 4] | m[p + 5] << 8) + 1;
                    p += 4 + sl;
                }
                if (bsize < 0) return where() + "not BGZF (a gzip member without the BC subfield)";
                if (bsize < (int64_t) (12 + xlen + 8)) return where() + "a BGZF member with a bad BSIZE";
                m.resize((size_t) bsize);
                if (fread(m.data() + 12 + xlen, 1, (size_t) bsize - 12 - xlen, f) != (size_t) bsize - 12 - xlen) return where() + "a truncated BGZF member";
                uint32_t crc, isize;
                memcpy(&crc, m.data() + bsize - 8, 4); memcpy(&isize, m.data() + bsize - 4, 4);
                if (isize > BGZF_MAX_MEMBER) return where() + "a BGZF member of more than 65536 bytes";
                in_bytes += bsize; ++members;
                last_empty = isize == 0;
                if (!isize) continue;
                jobs.push_back({m.data() + 12 + xlen, (size_t) bsize - 12 - xlen - 8, nullptr, isize, crc});
                have += isize; ++nz;
            }
            size_t at = rest.size();
            rest.resize(have);
            for (InflateJob &j : jobs) { j.out = rest.data() + at; at += j.isize; }
            if (!bgzf_inflate(jobs, threads, &inflate_s)) return where() + "a BGZF member does not inflate";
        }
        if (ended && !last_empty && warning.empty()) warning = where() + "no BGZF EOF block at the end: the input may be truncated";
        return "";
    }

    // the header: its text and bytes as read, the references' names and lengths
    std::string header(std::string &text, std::vector<std::pair<std::string, int32_t>> &refs) {
        std::string e;
        auto need = [&](size_t n) { if (!(e = fill(n)).empty()) return false; if (rest.size() < n) { e = where() + "the input ends inside the BAM header"; return false; } return true; };
        if (!need(4)) return e;
        if (memcmp(rest.data(), "BAM\1", 4)) return where() + "not BAM (no BAM magic)";
        if (!need(8)) return e;
        const int32_t lt = bam_le32(rest.data() + 4);
        if (lt < 0 || !need(12 + (size_t) lt)) return e.empty() ? where() + "a bad BAM header" : e;
        text.assign((const char *) rest.data() + 8, (size_t) lt);
        const int32_t nref = bam_le32(rest.data() + 8 + lt);
        if (nref < 0) return where() + "a bad BAM header";
        size_t at = 12 + (size_t) lt;
        for (int32_t r = 0; r < nref; ++r) {
            if (!need(at + 4)) return e;
            const int32_t ln = bam_le32(rest.data() + at);
            if (ln < 1 || !need(at + 8 + (size_t) ln)) return e.empty() ? where() + "a bad BAM header" : e;
            refs.push_back({std::string((const char *) rest.data() + at + 4, (size_t) ln - 1), bam_le32(rest.data() + at + 4 + ln)});
            at += 8 + (size_t) ln;
        }
        rest.erase(rest.begin(), rest.begin() + (long) at);
        return "";
    }

    // the next window's records (contiguous, whole) and their starts; both empty at the end of the input
    std::string next(std::vector<uint8_t> &recs, std::vector<int64_t> &starts) {
        recs.clear(); starts.clear();
        std::string e = fill((size_t) window);
        if (!e.empty()) return e;
        size_t q = 0;
        for (;;) {
            while (q + 4 <= rest.size()) {
                const int32_t bs = bam_le32(rest.data() + q);
                if (bs < 32) return where() + "record " + std::to_string(records) + " is malformed (block_size " + std::to_string(bs) + ")";
                if (q + 4 + (size_t) bs > rest.size()) break;
                const uint8_t *r = rest.data() + q;
                const int32_t l_seq = bam_le32(r + 20);
                if (l_seq < 0 || r[12] < 1 || 32 + (int64_t) r[12] + 4 * (int64_t) bam_le16(r + 16) + (l_seq + 1) / 2 + (int64_t) l_seq > (int64_t) bs)
                    return where() + "record " + std::to_string(records) + " is malformed (its fields overrun its block_size)";
                starts.push_back((int64_t) q);
                ++records;
                q += 4 + (size_t) bs;
            }
            if (!starts.empty() || rest.size() == q) break;
            const size_t want = q + 4 <= rest.size() ? q + 4 + (size_t) bam_le32(rest.data() + q) : q + 4;
            if (ended) return where() + "the input ends inside record " + std::to_string(records);
            if (!(e = fill(want)).empty()) return e;
        }
        if (starts.empty() && !rest.empty() && ended) return where() + "the input ends inside record " + std::to_string(records);
        std::vector<uint8_t> tail(rest.begin() + (long) q, rest.end());
        rest.resize(q);
        recs.swap(rest);
        rest.swap(tail);
        return "";
    }
};

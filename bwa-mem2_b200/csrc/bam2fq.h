// bam2fq.h — the host half of bm2_bam2fq: the reads of a BAM file in any order back to FASTQ, mates paired.  Host only; the device work
// comes in through the callbacks (bm2_bam2fq_records, bm2_markdup_pair, bm2_bam2fq_format in the tool), so that the host emulation
// tests/host_emul/bam2fq_emul.cpp runs this file unchanged over a CPU restatement of them.
//
//   streams   interleaved: one stream, a file or standard output.  Split: -1 and -2, and -0 and -s when given.  A file whose name ends in
//             .gz is BGZF; any other file and standard output are plain text.  Files are written to <name>.tmp and renamed once every
//             stream is complete, so an error leaves no file; standard output is streamed.
//   pairs     a READ1 and a READ2 of one QNAME, wherever they lie: the window's halves, after the halves carried from earlier windows in
//             input order, go through the pairing, which joins each half to the first earlier unjoined half of the same name, so the joins
//             are those of one pass over the whole input and do not depend on the windows.  A pair is written when its later record is
//             reached, READ1 first: to -1 and -2, or one after the other in the interleaved stream.  A joined pair of two READ1s or two
//             READ2s is an error that names the read.  An unjoined half is carried: its hash, name and record bytes stay on the host.
//   others    (both or neither of 0x40 and 0x80) written when reached: in place in the interleaved stream, or to -0
//   singletons  the halves still carried at the end, in input order: at the end of the interleaved stream, or to -s
//   dropped   in split mode without -0 or -s those records are counted and dropped, with one warning (our choice: samtools would write
//             them into another output, and -1 and -2 would then fall out of step)
#pragma once
#include "bm2_b200.h"
#include "bam_window.h"
#include <cstdio>
#include <functional>
#include <string>
#include <thread>
#include <unistd.h>
#include <vector>

struct Bam2fq {
    enum { S_MAIN = 0, S_R2 = 1, S_OTHER = 2, S_SINGLE = 3, S_N = 4 };
    // the run: the input ("-": standard input); split mode or not; the paths of the streams (interleaved: path[S_MAIN], empty for standard
    // output; split: -1, -2, -0, -s, the last two empty when not given); suffixes on or off
    std::string in_path;
    bool split = false;
    std::string path[S_N];
    int suffixes = 1, threads = 1;
    int64_t window = (int64_t) 256 << 20;
    // the device steps; each calls die on an error and does not return then
    std::function<void(int, const std::string &)> fail;       // does not return
    std::function<const bm2_bam2fq_rec *(const uint8_t *, int64_t, const int64_t *, int64_t)> records;
    std::function<const int32_t *(const bm2_markdup_half *, int64_t, const uint8_t *, int64_t)> pair;
    std::function<void(const int64_t *, int64_t, const uint8_t *, int64_t, const int64_t *, int64_t, const uint8_t *, int64_t, int, int,
                       bm2_bam2fq_out *)> format;
    // stats
    int64_t n_records = 0, kept = 0, pairs = 0, others = 0, singletons = 0, others_dropped = 0, singletons_dropped = 0;
    int64_t pending_max = 0, pending_bytes_max = 0, n_windows = 0, in_bytes = 0, out_bytes = 0;
    double inflate_s = 0;
    std::string warning;                                        // for the caller to print, one line each

    struct Stream { bool on = false, gz = false; std::string tmp, carry; FILE *f = nullptr; std::vector<int64_t> list; };
    struct Pending { uint64_t hash; int32_t kind; std::string name, rec; };
    Stream st[S_N];
    std::vector<Pending> pend;

    [[noreturn]] void die(int code, const std::string &m) {
        for (Stream &s : st) {
            if (s.f && s.f != stdout) fclose(s.f);
            s.f = nullptr;
            if (!s.tmp.empty()) unlink(s.tmp.c_str());
            s.tmp.clear();
        }
        fail(code, m);
        throw 0;                                                // fail does not return
    }

    static bool ends_with(const std::string &s, const char *e) { const size_t n = strlen(e); return s.size() >= n && s.compare(s.size() - n, n, e) == 0; }

    void put(Stream &s, const uint8_t *p, int64_t n) {
        if (n && fwrite(p, 1, (size_t) n, s.f) != (size_t) n) die(2, "cannot write " + (s.tmp.empty() ? std::string("standard output") : s.tmp));
        out_bytes += n;
    }

    // the stream's list, formatted against the current window and the extra records
    void emit(Stream &s, const std::string &xb, const std::vector<int64_t> &xs, int last) {
        bm2_bam2fq_out o{};
        format(s.list.data(), (int64_t) s.list.size(), (const uint8_t *) xb.data(), (int64_t) xb.size(), xs.data(), (int64_t) xs.size(),
               (const uint8_t *) s.carry.data(), (int64_t) s.carry.size(), s.gz ? 1 : 0, last, &o);
        put(s, o.data, o.len);
        if (s.gz) s.carry.assign((const char *) o.tail, (size_t) o.tail_len);
        s.list.clear();
    }

    void window_(const std::vector<uint8_t> &B, const std::vector<int64_t> &S) {
        const int64_t nr = (int64_t) S.size(), P = (int64_t) pend.size();
        const bm2_bam2fq_rec *info = records(B.data(), (int64_t) B.size(), S.data(), nr);
        std::vector<bm2_markdup_half> halves;
        std::string names;
        auto add = [&](uint64_t h, const uint8_t *nm, int32_t len) {
            halves.push_back(bm2_markdup_half{h, 0, len, (int64_t) names.size()});
            names.append((const char *) nm, (size_t) len);
        };
        for (const Pending &p : pend) add(p.hash, (const uint8_t *) p.name.data(), (int32_t) p.name.size());
        std::vector<int64_t> rec_of;                            // the window record of each of its halves
        for (int64_t i = 0; i < nr; ++i)
            if (info[i].kind == BM2_B2F_READ1 || info[i].kind == BM2_B2F_READ2) {
                const uint8_t *r = B.data() + S[i];
                add(info[i].hash, r + 36, r[12] ? r[12] - 1 : 0);
                rec_of.push_back(i);
            }
        const int32_t *partner = pair(halves.data(), (int64_t) halves.size(), (const uint8_t *) names.data(), (int64_t) names.size());
        std::string xb;                                         // the carried halves whose pairs complete in this window
        std::vector<int64_t> xs;
        std::vector<Pending> fresh;
        Stream &m = st[S_MAIN], &r2 = split ? st[S_R2] : st[S_MAIN], &oth = split ? st[S_OTHER] : st[S_MAIN];
        for (int64_t i = 0, h = P; i < nr; ++i) {
            const int k = info[i].kind;
            if (k == BM2_B2F_SKIP) continue;
            ++kept;
            if (k == BM2_B2F_OTHER) {
                ++others;
                if (oth.on) oth.list.push_back(i); else ++others_dropped;
                continue;
            }
            const uint8_t *r = B.data() + S[i];
            const int32_t q = partner[h++];
            if (q < 0) {
                fresh.push_back(Pending{info[i].hash, k, std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0),
                                        std::string((const char *) r, 4 + (size_t) bam_le32(r))});
                continue;
            }
            int64_t other;
            int ok;
            if (q >= P) {
                const int64_t j = rec_of[(size_t) (q - P)];
                if (j > i) continue;                            // the pair completes at its later record
                other = j; ok = info[j].kind;
            } else {
                xs.push_back((int64_t) xb.size());
                xb += pend[(size_t) q].rec;
                other = ~(int64_t) (xs.size() - 1); ok = pend[(size_t) q].kind;
            }
            if (ok == k)
                die(1, "read " + std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0) + ": two " + (k == BM2_B2F_READ1 ? "READ1" : "READ2") +
                           " records (0x40 and 0x80 flags) of one name");
            m.list.push_back(k == BM2_B2F_READ1 ? i : other);
            r2.list.push_back(k == BM2_B2F_READ1 ? other : i);
            ++pairs;
        }
        std::vector<Pending> keep;
        for (int64_t p = 0; p < P; ++p) if (partner[p] < 0) keep.push_back(std::move(pend[(size_t) p]));
        for (Pending &p : fresh) keep.push_back(std::move(p));
        pend.swap(keep);
        int64_t pb = 0;
        for (const Pending &p : pend) pb += (int64_t) p.rec.size();
        pending_max = std::max(pending_max, (int64_t) pend.size());
        pending_bytes_max = std::max(pending_bytes_max, pb);
        for (Stream &s : st) if (s.on && !s.list.empty()) emit(s, xb, xs, 0);
    }

    void run() {
        for (int s = 0; s < S_N; ++s) {
            Stream &x = st[s];
            x.on = s == S_MAIN || (split && (s == S_R2 || !path[s].empty()));
            if (!x.on) continue;
            x.gz = ends_with(path[s], ".gz");
        }
        BamWindowReader rd;
        rd.name = in_path == "-" ? "standard input" : in_path;
        rd.f = in_path == "-" ? stdin : fopen(in_path.c_str(), "rb");
        if (!rd.f) die(1, "cannot open " + in_path);
        rd.threads = threads; rd.window = window;
        std::string text;
        std::vector<std::pair<std::string, int32_t>> refs;
        std::string e = rd.header(text, refs);
        if (!e.empty()) die(1, e);
        for (int s = 0; s < S_N; ++s) {
            Stream &x = st[s];
            if (!x.on) continue;
            if (path[s].empty()) { x.f = stdout; continue; }
            x.tmp = path[s] + ".tmp";
            x.f = fopen(x.tmp.c_str(), "wb");
            if (!x.f) { const std::string t = x.tmp; x.tmp.clear(); die(2, "cannot open " + t); }
        }
        std::vector<uint8_t> buf[2];
        std::vector<int64_t> starts[2];
        e = rd.next(buf[0], starts[0]);
        if (!e.empty()) die(1, e);
        for (int cur = 0; !starts[cur].empty(); cur ^= 1) {
            std::string e_next;
            std::thread next([&] { e_next = rd.next(buf[cur ^ 1], starts[cur ^ 1]); });
            try {
                window_(buf[cur], starts[cur]);
            } catch (...) {
                next.join();
                throw;
            }
            n_records += (int64_t) starts[cur].size(); ++n_windows;
            next.join();
            if (!e_next.empty()) die(1, e_next);
        }
        // the singletons, in input order, then every stream's last block
        singletons = (int64_t) pend.size();
        std::string xb;
        std::vector<int64_t> xs;
        Stream &ss = split ? st[S_SINGLE] : st[S_MAIN];
        if (ss.on)
            for (const Pending &p : pend) { xs.push_back((int64_t) xb.size()); xb += p.rec; ss.list.push_back(~(int64_t) (xs.size() - 1)); }
        else singletons_dropped = singletons;
        pend.clear();
        static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (Stream &s : st) {
            if (!s.on) continue;
            if (s.gz || !s.list.empty()) emit(s, xb, xs, 1);
            if (s.gz) put(s, eof, sizeof eof);
        }
        if (!rd.warning.empty()) warning += rd.warning + "\n";
        if (rd.f != stdin) fclose(rd.f);
        in_bytes = rd.in_bytes; inflate_s = rd.inflate_s;
        for (Stream &s : st) {
            if (!s.on) continue;
            if (s.f == stdout) { if (fflush(stdout)) die(2, "cannot write standard output"); continue; }
            const int bad = fclose(s.f);
            s.f = nullptr;
            if (bad) die(2, "cannot write " + s.tmp);
        }
        for (int k = 0; k < S_N; ++k) {
            Stream &s = st[k];
            if (s.tmp.empty()) continue;
            if (rename(s.tmp.c_str(), path[k].c_str())) die(2, "cannot write " + path[k]);
            s.tmp.clear();
        }
        if (others_dropped || singletons_dropped)
            warning += std::to_string(others_dropped) + " records with both or neither of 0x40 and 0x80 and " + std::to_string(singletons_dropped) +
                       " READ1 or READ2 records without their mate were not written: give -0 and -s to keep them\n";
    }
};

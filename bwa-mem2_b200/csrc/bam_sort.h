// bam_sort.h — the host side of bm2_mem --sort: coordinate-sorted BAM, and its BAI index, in bounded host memory.
//
//   runs    the records arrive in output order (add) and fill a run of at most run_bytes (a record larger than that is a run of its own).
//           A full run goes to a sorter thread, which sorts and compresses it with the device call and writes it to a temporary file
//           (opened, then unlinked at once, so that nothing is left behind whatever happens), while the next run fills: host memory is two
//           runs.  When the whole output fits in one run, that run, sorted, is the output and no file is written.
//   merge   window by window: every unfinished run loads its next members (inflated by zlib on a pool of threads) until it holds about
//           run_bytes / runs of whole records.  T is the smallest last-loaded key over the runs not yet fully loaded, r* the first such run
//           whose last key is T; every loaded record with key < T, and those with key == T of runs up to r*, are settled.  They are
//           concatenated in run order and sorted with the same device call (stable, so ties keep run order and then the order within the
//           run, which is input order), passing the carry: the BGZF blocks are cut over the whole sorted stream.  r*'s last record is
//           always settled, so every window makes progress.
//   BAI     (SAMv1 §5.2) from each record's (refID, pos, end, bin, flag) and virtual offset: per bin its chunks, a chunk joined to the one
//           before when that one ends where it starts; the 16 kbp linear index, empty windows filled from the one before; pseudo-bin 37450
//           with the reference's offset span and its mapped / unmapped counts; n_no_coor.
//
// The device call is a parameter, so that tests/host_emul/bam_sort_emul.cpp runs all of this with the GPU swapped for a CPU restatement.
#pragma once
#include "bam_sort_device.cuh"
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <thread>
#include <unistd.h>
#include <vector>
#include <zlib.h>

// one buffer of records sorted and compressed (bm2_bam_sort_compress's arguments); device_s: its device time.  Returns 0 on success.
using SortCall = std::function<int(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry, int64_t carry_len,
                                   int last, bm2_sort_out *out, double *device_s)>;
// reports an error and does not return
using SortFail = std::function<void(const std::string &)>;

struct BaiBuilder {
    static constexpr uint64_t kUnset = ~(uint64_t) 0;
    struct Ref {
        std::map<uint32_t, std::vector<std::pair<uint64_t, uint64_t>>> bins;
        std::vector<uint64_t> lin;
        uint64_t beg = kUnset, end = 0, n_mapped = 0, n_unmapped = 0;
    };
    std::vector<Ref> refs;
    uint64_t n_no_coor = 0;
    bool have_prev = false;
    bm2_sort_rec prev{};
    uint64_t prev_voff = 0;

    explicit BaiBuilder(int n_ref = 0) : refs((size_t) n_ref) {}
    // records in file order with their virtual offsets; a record ends where the next begins
    void push(const bm2_sort_rec &r, uint64_t voff) { if (have_prev) add(prev, prev_voff, voff); prev = r; prev_voff = voff; have_prev = true; }
    void finish(uint64_t end_voff) { if (have_prev) add(prev, prev_voff, end_voff); have_prev = false; }
    void add(const bm2_sort_rec &r, uint64_t beg, uint64_t end) {
        if (r.rid < 0) { ++n_no_coor; return; }
        if ((size_t) r.rid >= refs.size()) refs.resize((size_t) r.rid + 1);
        Ref &R = refs[(size_t) r.rid];
        auto &ch = R.bins[r.bin];
        if (!ch.empty() && ch.back().second == beg) ch.back().second = end;
        else ch.push_back({beg, end});
        const int64_t p = r.pos > 0 ? r.pos : 0, e = r.end > p ? r.end : p + 1;
        const size_t w0 = (size_t) (p >> 14), w1 = (size_t) ((e - 1) >> 14);
        if (R.lin.size() < w1 + 1) R.lin.resize(w1 + 1, kUnset);
        for (size_t w = w0; w <= w1; ++w) if (R.lin[w] == kUnset) R.lin[w] = beg;
        if (R.beg == kUnset) R.beg = beg;
        R.end = end;
        ++((r.flag & 4) ? R.n_unmapped : R.n_mapped);
    }
    std::string bytes() const {
        std::string o("BAI\1", 4);
        auto i32 = [&](int32_t v) { o.append((const char *) &v, 4); };
        auto u64 = [&](uint64_t v) { o.append((const char *) &v, 8); };
        i32((int32_t) refs.size());
        for (const Ref &R : refs) {
            const bool any = R.beg != kUnset;
            i32((int32_t) R.bins.size() + (any ? 1 : 0));
            for (const auto &b : R.bins) {
                i32((int32_t) b.first); i32((int32_t) b.second.size());
                for (const auto &c : b.second) { u64(c.first); u64(c.second); }
            }
            if (any) { i32(37450); i32(2); u64(R.beg); u64(R.end); u64(R.n_mapped); u64(R.n_unmapped); }
            i32((int32_t) R.lin.size());
            uint64_t last = 0;
            for (uint64_t v : R.lin) { if (v != kUnset) last = v; u64(last); }
        }
        u64(n_no_coor);
        return o;
    }
};

// the sorted stream's writer: each call's members go to the file, each record's virtual offset to the index
struct SortedWriter {
    SortCall sort; SortFail fail; FILE *out = nullptr; BaiBuilder *bai = nullptr;
    uint64_t file_off = 0;                       // compressed bytes before the next member
    std::vector<uint8_t> carry;
    double device_s = 0;
    void write(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, bool last) {
        bm2_sort_out o;
        double ds = 0;
        if (sort(recs, n, starts, n_recs, carry.data(), (int64_t) carry.size(), last ? 1 : 0, &o, &ds)) fail("bm2_bam_sort_compress");
        device_s += ds;
        if (o.z_len && fwrite(o.z, 1, (size_t) o.z_len, out) != (size_t) o.z_len) fail("cannot write the sorted BAM");
        if (bai) {
            std::vector<uint64_t> addr((size_t) o.n_members + 1, file_off);
            for (int64_t k = 0; k < o.n_members; ++k) addr[(size_t) k + 1] = addr[(size_t) k] + (uint64_t) o.member_size[k];
            for (int64_t i = 0; i < o.n_recs; ++i) bai->push(o.recs[i], addr[(size_t) o.recs[i].block] << 16 | (uint64_t) o.recs[i].offset);
        }
        file_off += (uint64_t) o.z_len;
        carry.assign(o.carry, o.carry + o.carry_len);
        if (last && bai) bai->finish(file_off << 16);
    }
};

struct BamSortSink {
    struct Run { FILE *f = nullptr; std::vector<int32_t> members; };
    // settings
    SortCall sort; SortFail fail;
    int64_t run_bytes = (int64_t) 2 << 30;
    std::string tmp_prefix;                      // runs go to <tmp_prefix>NNNN
    int threads = 1;
    // state
    std::vector<uint8_t> cur; std::vector<int64_t> cur_starts;
    std::vector<uint8_t> pend; std::vector<int64_t> pend_starts;
    std::thread sorter;
    std::vector<Run> runs;
    // stats
    double sort_s = 0, merge_s = 0;
    int64_t spill_bytes = 0, merge_windows = 0;

    ~BamSortSink() { if (sorter.joinable()) sorter.join(); for (Run &r : runs) if (r.f) fclose(r.f); }

    // the records of one chunk, in output order
    void add(const uint8_t *p, int64_t len) {
        for (int64_t q = 0; q + 4 <= len;) {
            int32_t bs; memcpy(&bs, p + q, 4);
            const int64_t m = 4 + (int64_t) bs;
            if (bs < 32 || q + m > len) fail("a malformed BAM record");
            if (!cur_starts.empty() && (int64_t) cur.size() + m > run_bytes) hand_off();
            cur_starts.push_back((int64_t) cur.size());
            cur.insert(cur.end(), p + q, p + q + m);
            q += m;
        }
    }

    // the current run to the sorter thread, once the one before is on disk
    void hand_off() {
        if (sorter.joinable()) sorter.join();
        pend.swap(cur); pend_starts.swap(cur_starts);
        cur.clear(); cur_starts.clear();
        sorter = std::thread([this] { spill(); });
    }

    void spill() {
        char name[32];
        snprintf(name, sizeof name, "%04d", (int) runs.size());
        const std::string path = tmp_prefix + name;
        Run r;
        r.f = fopen(path.c_str(), "w+b");
        if (!r.f) fail("cannot create the temporary file " + path);
        unlink(path.c_str());
        SortedWriter w{sort, fail, r.f, nullptr};
        w.write(pend.data(), (int64_t) pend.size(), pend_starts.data(), (int64_t) pend_starts.size(), true);
        sort_s += w.device_s;
        // the members' sizes, from their BSIZE fields, read back as the merge will read them
        if (fflush(r.f) || fseek(r.f, 0, SEEK_SET)) fail("cannot write the temporary file " + path);
        spill_bytes += (int64_t) w.file_off;
        for (uint64_t at = 0; at < w.file_off;) {
            uint8_t h[18];
            if (fread(h, 1, 18, r.f) != 18) fail("cannot read the temporary file " + path);
            const int32_t sz = (int32_t) (h[16] | h[17] << 8) + 1;
            r.members.push_back(sz);
            at += (uint64_t) sz;
            if (fseek(r.f, (long) at, SEEK_SET)) fail("cannot read the temporary file " + path);
        }
        if (fseek(r.f, 0, SEEK_SET)) fail("cannot read the temporary file " + path);
        runs.push_back(std::move(r));
        std::vector<uint8_t>().swap(pend); std::vector<int64_t>().swap(pend_starts);
    }

    // everything has been added: the sorted records to out (its compressed offset now: out_off), the index to bai when not null
    void finish(FILE *out, uint64_t out_off, BaiBuilder *bai) {
        SortedWriter w{sort, fail, out, bai, out_off};
        if (!sorter.joinable() && runs.empty()) {
            w.write(cur.data(), (int64_t) cur.size(), cur_starts.data(), (int64_t) cur_starts.size(), true);
            sort_s += w.device_s;
            return;
        }
        if (!cur_starts.empty()) hand_off();
        sorter.join();
        merge(w);
    }

    struct Cursor {                              // a run being merged
        size_t next = 0;                          // next member to load
        std::vector<uint8_t> buf; size_t pos = 0; // loaded bytes, consumed up to pos
        std::vector<size_t> recs;                 // whole records at buf[pos..]: their starts
    };

    static uint64_t key_at(const uint8_t *r) { const BamFixed f = bam_fixed(r); return bam_coord_key(f.rid, f.pos, f.flag); }

    void merge(SortedWriter &w) {
        const double t0 = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
        const size_t nr = runs.size();
        const int64_t quota = std::max<int64_t>(run_bytes / (int64_t) nr, BGZF_BLOCK);
        std::vector<Cursor> c(nr);
        std::vector<uint8_t> win; std::vector<int64_t> win_starts;
        for (;;) {
            for (int round = 0;; ++round) {               // load until every unfinished run holds a quota and at least one whole record
                struct Job { size_t run; std::vector<uint8_t> z; size_t at; uint32_t isize; };
                std::vector<Job> jobs;
                for (size_t r = 0; r < nr; ++r) {
                    Cursor &x = c[r];
                    int64_t have = (int64_t) (x.buf.size() - x.pos);
                    const bool need_rec = x.recs.empty();
                    if (round > 0 && !need_rec) continue;
                    if (x.pos) { x.buf.erase(x.buf.begin(), x.buf.begin() + (long) x.pos); for (size_t &s : x.recs) s -= x.pos; x.pos = 0; }
                    const int64_t want = need_rec ? std::max<int64_t>(round == 0 ? quota : 0, have + 1) : quota;
                    while (x.next < runs[r].members.size() && have < want) {
                        Job j; j.run = r; j.z.resize((size_t) runs[r].members[x.next]);
                        if (fread(j.z.data(), 1, j.z.size(), runs[r].f) != j.z.size()) fail("cannot read a temporary file");
                        memcpy(&j.isize, j.z.data() + j.z.size() - 4, 4);
                        j.at = x.buf.size() + [&] { size_t s = 0; for (const Job &k : jobs) if (k.run == r) s += k.isize; return s; }();
                        have += j.isize; ++x.next;
                        jobs.push_back(std::move(j));
                    }
                }
                if (jobs.empty()) break;
                std::vector<size_t> grow(nr, 0);
                for (const Job &j : jobs) grow[j.run] += j.isize;
                for (size_t r = 0; r < nr; ++r) c[r].buf.resize(c[r].buf.size() + grow[r]);
                std::atomic<size_t> next{0}; std::atomic<bool> bad{false};
                auto inflate_some = [&] {
                    for (size_t k; (k = next++) < jobs.size();) {
                        const Job &j = jobs[k];
                        z_stream zs; memset(&zs, 0, sizeof zs);
                        if (inflateInit2(&zs, -15) != Z_OK) { bad = true; continue; }
                        zs.next_in = (Bytef *) j.z.data() + 18; zs.avail_in = (uInt) (j.z.size() - 26);
                        zs.next_out = c[j.run].buf.data() + j.at; zs.avail_out = j.isize;
                        if (inflate(&zs, Z_FINISH) != Z_STREAM_END || zs.avail_out) bad = true;
                        inflateEnd(&zs);
                    }
                };
                std::vector<std::thread> pool;
                for (int t = 1; t < std::min<int>(threads, (int) jobs.size()); ++t) pool.emplace_back(inflate_some);
                inflate_some();
                for (auto &t : pool) t.join();
                if (bad) fail("a temporary file does not inflate");
                for (size_t r = 0; r < nr; ++r) {                                    // the whole records now loaded
                    Cursor &x = c[r];
                    size_t q = x.recs.empty() ? x.pos : x.recs.back() + 4 + (size_t) bam_le32(x.buf.data() + x.recs.back());
                    while (q + 4 <= x.buf.size() && q + 4 + (size_t) bam_le32(x.buf.data() + q) <= x.buf.size()) {
                        x.recs.push_back(q); q += 4 + (size_t) bam_le32(x.buf.data() + q);
                    }
                }
            }
            // T and r* over the runs not fully loaded
            bool open = false; uint64_t T = 0; size_t rs = 0;
            for (size_t r = 0; r < nr; ++r) {
                if (c[r].next >= runs[r].members.size()) continue;
                const uint64_t k = key_at(c[r].buf.data() + c[r].recs.back());
                if (!open || k < T) { T = k; rs = r; open = true; }
            }
            win.clear(); win_starts.clear();
            for (size_t r = 0; r < nr; ++r) {
                Cursor &x = c[r];
                size_t k = 0;
                while (k < x.recs.size()) {
                    const uint64_t kk = key_at(x.buf.data() + x.recs[k]);
                    if (open && (kk > T || (kk == T && r > rs))) break;
                    ++k;
                }
                if (!k) continue;
                const size_t b = x.recs[0], e = x.recs[k - 1] + 4 + (size_t) bam_le32(x.buf.data() + x.recs[k - 1]);
                for (size_t i = 0; i < k; ++i) win_starts.push_back((int64_t) (win.size() + x.recs[i] - b));
                win.insert(win.end(), x.buf.begin() + (long) b, x.buf.begin() + (long) e);
                x.recs.erase(x.recs.begin(), x.recs.begin() + (long) k);
                x.pos = e;
            }
            w.write(win.data(), (int64_t) win.size(), win_starts.data(), (int64_t) win_starts.size(), !open);
            ++merge_windows;
            if (!open) break;
        }
        for (size_t r = 0; r < nr; ++r) if (c[r].pos != c[r].buf.size()) fail("a temporary file ends inside a record");
        merge_s += std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count() - t0;
    }
};

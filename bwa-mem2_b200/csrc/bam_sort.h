// bam_sort.h — the host side of bm2_mem --sort: coordinate-sorted BAM, and its BAI index, in bounded host memory.
//
//   runs    the records arrive in output order (add) and fill a run of at most run_bytes (a record larger than that is a run of its own).
//           A full run goes to a sorter thread, which sorts and compresses it with the device call and writes it to a temporary file
//           (opened, then unlinked at once, so that nothing is left behind whatever happens), while the next run fills: host memory is two
//           runs.  When the whole output fits in one run, that run, sorted, is the output and no file is written.
//   merge   window by window: every unfinished run loads its next members (inflated by zlib on a pool of threads: bgzf_inflate, which
//           bm2_applybqsr's window reader shares) until it holds about run_bytes / runs of whole records.  T is the smallest last-loaded key
//           over the runs not yet fully loaded, r* the first such run whose last key is T; every loaded record with key < T, and those with key == T of runs up to r*, are settled.  They are
//           concatenated in run order and sorted with the same device call (stable, so ties keep run order and then the order within the
//           run, which is input order), passing the carry: the BGZF blocks are cut over the whole sorted stream.  r*'s last record is
//           always settled, so every window makes progress.  With cmp set (bm2_sort -n), cmp orders the records in place of the key.
//   BAI     (SAMv1 §5.2) from each record's (refID, pos, end, bin, flag) and virtual offset: per bin its chunks, a chunk joined to the one
//           before when that one ends where it starts; the 16 kbp linear index, empty windows filled from the one before; pseudo-bin 37450
//           with the reference's offset span and its mapped / unmapped counts; n_no_coor.
//
//   markdup (--markdup, markdup_device.cuh's rule) each record comes with its template's id, and each chunk with its templates' entries.
//           The ids travel with the records: a spilled run writes its ids in sorted order to a second temporary file (8 bytes per record,
//           opened and unlinked the same way), and the merge reads them in step.  The entries are held up to sig_bytes (--sort-mem / 8, a
//           chosen figure, not a measured one), half of it filling while the sorter thread sorts the other half on the device and spills it
//           as a sorted run.  At finish, with the last record run spilled, the duplicates are resolved: in one call per space when nothing
//           spilled, else window by window over the sorted runs of each space, with the record merge's settle rule except that only keys
//           strictly below T are settled, so that every group is resolved whole (a group larger than a window grows the window: host memory
//           then grows by one entry per member of the largest group).  The duplicate templates become a bitset of 1 bit per input read,
//           uploaded to the sort context before the one-run sort or the first merge window, which set 0x400 on their records.
//
//   metrics (--markdup-metrics) the pair space holds located entries (bm2_dup_loc_entry, 48 bytes, counted as such against sig_bytes, and
//           spilled as such), resolved by the located call, which also returns the optical count of the call's pair groups.  A group never
//           straddles a window, so the sum over the windows is exact.
//
//   recal   (--recal-file) before_final arms the sort context's covariate counting (bm2_bqsr_sites) after the duplicates are resolved, so
//           that only the final pass (the one-run sort, or the merge windows) counts, with the records' final flags; the runs spilled
//           before are never counted.
//
// The device calls are parameters, so that tests/host_emul/bam_sort_emul.cpp, bamsort_emul.cpp and markdup_emul.cpp run all of this with the GPU swapped for a
// CPU restatement.
#pragma once
#include "bam_sort_device.cuh"
#include "markdup_device.cuh"
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <exception>
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
// the same with one template id per record (tids, may be null) carried through the sort (bm2_bam_sort_compress_ex): *tids_out gets them sorted
using SortCallEx = std::function<int(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tids, const uint8_t *carry,
                                     int64_t carry_len, int last, bm2_sort_out *out, const int64_t **tids_out, double *device_s)>;
// the entries of one duplicate space sorted (resolve 0) or resolved into the duplicates' template ids (bm2_dup_resolve's arguments)
using DupCall = std::function<int(const bm2_dup_entry *e, int64_t n, int resolve, const bm2_dup_entry **sorted, const int64_t **dups, int64_t *n_dups,
                                  double *device_s)>;
// the same over located entries with the optical count at the sink's optical_distance (bm2_dup_resolve_ex's arguments)
using DupCallEx = std::function<int(const bm2_dup_loc_entry *e, int64_t n, int resolve, const bm2_dup_loc_entry **sorted, const int64_t **dups,
                                    int64_t *n_dups, int64_t *n_optical, double *device_s)>;
// the duplicate bitset to the sort context (bm2_dup_set)
using DupSetCall = std::function<int(const uint64_t *bits, int64_t n_bits)>;
// the three-way order of two records (block_size first) that a SortCall sorts by: < 0, 0 or > 0
using RecCmp = std::function<int(const uint8_t *a, const uint8_t *b)>;
// reports an error and does not return
using SortFail = std::function<void(const std::string &)>;

// one BGZF member's raw DEFLATE data to inflate into out: isize bytes whose CRC32 must be crc
struct InflateJob { const uint8_t *deflate; size_t len; uint8_t *out; uint32_t isize, crc; };

// the jobs inflated by zlib on up to `threads` threads; false when one does not inflate to exactly isize bytes with its CRC32.
// busy_s (may be null) gets the threads' inflate time added, summed over the threads.
inline bool bgzf_inflate(const std::vector<InflateJob> &jobs, int threads, double *busy_s = nullptr) {
    std::atomic<size_t> next{0}; std::atomic<bool> bad{false};
    std::vector<double> busy((size_t) std::max(threads, 1), 0.0);
    auto inflate_some = [&](int t) {
        const auto t0 = std::chrono::steady_clock::now();
        for (size_t k; (k = next++) < jobs.size();) {
            const InflateJob &j = jobs[k];
            z_stream zs; memset(&zs, 0, sizeof zs);
            if (inflateInit2(&zs, -15) != Z_OK) { bad = true; continue; }
            zs.next_in = (Bytef *) j.deflate; zs.avail_in = (uInt) j.len;
            zs.next_out = j.out; zs.avail_out = j.isize;
            if (inflate(&zs, Z_FINISH) != Z_STREAM_END || zs.avail_out || zs.avail_in) bad = true;
            else if ((uint32_t) crc32(crc32(0L, Z_NULL, 0), j.out, j.isize) != j.crc) bad = true;
            inflateEnd(&zs);
        }
        busy[(size_t) t] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < std::min<int>(threads, (int) jobs.size()); ++t) pool.emplace_back(inflate_some, t);
    inflate_some(0);
    for (auto &t : pool) t.join();
    if (busy_s) for (double b : busy) *busy_s += b;
    return !bad;
}

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
    SortCallEx sort; SortFail fail; FILE *out = nullptr; BaiBuilder *bai = nullptr;
    uint64_t file_off = 0;                       // compressed bytes before the next member
    std::vector<uint8_t> carry;
    double device_s = 0;
    int64_t marked = 0;                          // records written with 0x400
    // tids: the records' template ids or null; tids_out: where their sorted ids go, or null
    void write(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tids, bool last,
               std::vector<int64_t> *tids_out = nullptr) {
        bm2_sort_out o;
        double ds = 0;
        const int64_t *ts = nullptr;
        if (sort(recs, n, starts, n_recs, tids, carry.data(), (int64_t) carry.size(), last ? 1 : 0, &o, tids ? &ts : nullptr, &ds))
            fail("bm2_bam_sort_compress");
        device_s += ds;
        if (tids_out) tids_out->assign(ts, ts + (ts ? n_recs : 0));
        for (int64_t i = 0; i < o.n_recs; ++i) marked += (o.recs[i].flag & 0x400) != 0;
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
    struct Run { FILE *f = nullptr, *tf = nullptr; std::vector<int32_t> members; };
    struct SigRun { FILE *f = nullptr; int64_t n = 0; };
    // settings
    SortCall sort; SortFail fail;
    SortCallEx sort_ex;                          // when set, used instead of sort
    DupCall dup; DupSetCall dup_set;             // --markdup when dup is set (sort_ex must be set then)
    DupCallEx dup_ex;                            // --markdup-metrics: the pair space through this one, with add_sigs_ex
    std::function<void()> before_final;          // --recal-file: called once the duplicates are known, before the one-run sort or the merge
    RecCmp cmp;                                  // the order sort sorts by (without input order), for the merge; unset: the coordinate key
    int64_t run_bytes = (int64_t) 2 << 30;
    int64_t sig_bytes = (int64_t) 256 << 20;     // entries held on the host (--sort-mem / 8)
    int64_t n_reads = 0;                         // the duplicate bitset's bits: set before finish
    std::string tmp_prefix;                      // runs go to <tmp_prefix>NNNN (their ids to <tmp_prefix>NNNN.id), signature runs to <tmp_prefix>dNNNN
    int threads = 1;
    // state
    std::vector<uint8_t> cur; std::vector<int64_t> cur_starts, cur_tids;
    std::vector<uint8_t> pend; std::vector<int64_t> pend_starts, pend_tids;
    std::thread sorter;
    std::exception_ptr sorter_error;             // a throwing fail() in the sorter thread, rethrown by join_sorter
    std::vector<Run> runs;
    std::vector<bm2_dup_entry> sig_cur[2], sig_pend[2];   // [0] pair space, [1] fragment space
    std::vector<SigRun> sig_runs[2];
    std::vector<bm2_dup_loc_entry> lsig_cur, lsig_pend;   // the pair space with dup_ex
    // stats
    double sort_s = 0, merge_s = 0, markdup_s = 0;
    int64_t spill_bytes = 0, merge_windows = 0;
    int64_t dup_templates = 0, dup_pair_templates = 0, dup_frag_templates = 0, dup_records = 0, dup_sig_runs = 0, dup_sig_bytes = 0;
    int64_t dup_pair_entries = 0, dup_frag_entries = 0, dup_optical_pairs = 0;   // with dup_ex: pair and fragment entries, optical duplicates

    ~BamSortSink() {
        if (sorter.joinable()) sorter.join();
        for (Run &r : runs) { if (r.f) fclose(r.f); if (r.tf) fclose(r.tf); }
        for (auto &v : sig_runs) for (SigRun &r : v) if (r.f) fclose(r.f);
    }

    // waits for the sorter thread; a fail() that threw there (the host emulation's) is thrown here, on the caller's thread
    void join_sorter() {
        if (sorter.joinable()) sorter.join();
        if (sorter_error) { const std::exception_ptr e = sorter_error; sorter_error = nullptr; std::rethrow_exception(e); }
    }
    template <class F> void start_sorter(F f) {
        sorter = std::thread([this, f] { try { f(); } catch (...) { sorter_error = std::current_exception(); } });
    }

    SortCallEx call() const {
        if (sort_ex) return sort_ex;
        SortCall s = sort;
        return [s](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, const int64_t *, const uint8_t *c, int64_t cl, int last, bm2_sort_out *o,
                   const int64_t **tids_out, double *ds) {
            if (tids_out) *tids_out = nullptr;
            return s(r, n, st, nr, c, cl, last, o, ds);
        };
    }

    // the records of one chunk, in output order; with --markdup, tids: each record's template id
    void add(const uint8_t *p, int64_t len, const int64_t *tids = nullptr) {
        int64_t k = 0;
        for (int64_t q = 0; q + 4 <= len; ++k) {
            int32_t bs; memcpy(&bs, p + q, 4);
            const int64_t m = 4 + (int64_t) bs;
            if (bs < 32 || q + m > len) fail("a malformed BAM record");
            if (!cur_starts.empty() && (int64_t) cur.size() + m > run_bytes) hand_off();
            cur_starts.push_back((int64_t) cur.size());
            cur.insert(cur.end(), p + q, p + q + m);
            if (dup) cur_tids.push_back(tids ? tids[k] : -1);
            q += m;
        }
    }

    // the entries of one chunk's templates (bm2_dup_signatures), in chunk order
    void add_sigs(const bm2_dup_entry *pairs, int64_t n_pairs, const bm2_dup_entry *frags, int64_t n_frags) {
        dup_templates += n_pairs;
        for (int64_t i = 0; i < n_frags; ++i) dup_templates += frags[i].kind == 1;
        sig_cur[0].insert(sig_cur[0].end(), pairs, pairs + n_pairs);
        sig_cur[1].insert(sig_cur[1].end(), frags, frags + n_frags);
        maybe_spill_sigs();
    }

    // the same with located pair entries (bm2_dup_signatures_ex), for dup_ex
    void add_sigs_ex(const bm2_dup_loc_entry *pairs, int64_t n_pairs, const bm2_dup_entry *frags, int64_t n_frags) {
        dup_templates += n_pairs; dup_pair_entries += n_pairs;
        for (int64_t i = 0; i < n_frags; ++i) { dup_templates += frags[i].kind == 1; dup_frag_entries += frags[i].kind == 1; }
        lsig_cur.insert(lsig_cur.end(), pairs, pairs + n_pairs);
        sig_cur[1].insert(sig_cur[1].end(), frags, frags + n_frags);
        maybe_spill_sigs();
    }

    void move_sigs_to_pending() {
        for (int s = 0; s < 2; ++s) { sig_pend[s].swap(sig_cur[s]); sig_cur[s].clear(); }
        lsig_pend.swap(lsig_cur); lsig_cur.clear();
    }

    void maybe_spill_sigs() {
        if ((int64_t) ((sig_cur[0].size() + sig_cur[1].size()) * sizeof(bm2_dup_entry) + lsig_cur.size() * sizeof(bm2_dup_loc_entry)) > sig_bytes / 2) {
            join_sorter();
            move_sigs_to_pending();
            start_sorter([this] { spill_sigs(); });
        }
    }

    int sort_entries(const bm2_dup_entry *e, int64_t n, const bm2_dup_entry **sorted, double *ds) { return dup(e, n, 0, sorted, nullptr, nullptr, ds); }
    int sort_entries(const bm2_dup_loc_entry *e, int64_t n, const bm2_dup_loc_entry **sorted, double *ds) {
        return dup_ex(e, n, 0, sorted, nullptr, nullptr, nullptr, ds);
    }

    // the pending entries, sorted on the device, as one more signature run of each space
    void spill_sigs() {
        for (int s = 0; s < 2; ++s) {
            if (s == 0 && dup_ex) spill_space(lsig_pend, 0);
            else spill_space(sig_pend[s], s);
        }
        ++dup_sig_runs;
    }

    template <class E> void spill_space(std::vector<E> &v, int s) {
        if (v.empty()) return;
        char name[32];
        snprintf(name, sizeof name, "d%04d", (int) (sig_runs[0].size() + sig_runs[1].size()));
        const std::string path = tmp_prefix + name;
        SigRun r;
        r.f = open_tmp(path, fail);
        const E *sorted = nullptr; double ds = 0;
        if (sort_entries(v.data(), (int64_t) v.size(), &sorted, &ds)) fail(sizeof(E) == sizeof(bm2_dup_entry) ? "bm2_dup_resolve" : "bm2_dup_resolve_ex");
        markdup_s += ds;
        if (fwrite(sorted, sizeof(E), v.size(), r.f) != v.size() || fflush(r.f) || fseek(r.f, 0, SEEK_SET))
            fail("cannot write the temporary file " + path);
        r.n = (int64_t) v.size();
        dup_sig_bytes += r.n * (int64_t) sizeof(E);
        sig_runs[s].push_back(r);
        std::vector<E>().swap(v);
    }

    // the current run to the sorter thread, once the one before is on disk
    void hand_off() {
        join_sorter();
        pend.swap(cur); pend_starts.swap(cur_starts); pend_tids.swap(cur_tids);
        cur.clear(); cur_starts.clear(); cur_tids.clear();
        start_sorter([this] { spill(); });
    }

    static FILE *open_tmp(const std::string &path, const SortFail &fail) {
        FILE *f = fopen(path.c_str(), "w+b");
        if (!f) fail("cannot create the temporary file " + path);
        unlink(path.c_str());
        return f;
    }

    void spill() {
        char name[32];
        snprintf(name, sizeof name, "%04d", (int) runs.size());
        const std::string path = tmp_prefix + name;
        Run r;
        r.f = open_tmp(path, fail);
        SortedWriter w{call(), fail, r.f, nullptr};
        std::vector<int64_t> ids;
        w.write(pend.data(), (int64_t) pend.size(), pend_starts.data(), (int64_t) pend_starts.size(), dup ? pend_tids.data() : nullptr, true,
                dup ? &ids : nullptr);
        sort_s += w.device_s;
        if (dup) {                                // the ids in sorted order, 8 bytes per record
            r.tf = open_tmp(path + ".id", fail);
            if (fwrite(ids.data(), 8, ids.size(), r.tf) != ids.size() || fflush(r.tf) || fseek(r.tf, 0, SEEK_SET))
                fail("cannot write the temporary file " + path + ".id");
            spill_bytes += (int64_t) ids.size() * 8;
            std::vector<int64_t>().swap(pend_tids);
        }
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
        SortedWriter w{call(), fail, out, bai, out_off};
        join_sorter();
        const bool one_run = runs.empty();
        if (!one_run && !cur_starts.empty()) { hand_off(); join_sorter(); }
        if (dup) resolve();
        if (before_final) before_final();
        if (one_run) {
            w.write(cur.data(), (int64_t) cur.size(), cur_starts.data(), (int64_t) cur_starts.size(), dup ? cur_tids.data() : nullptr, true);
            sort_s += w.device_s;
        } else merge(w);
        dup_records = w.marked;
    }

    static const bm2_dup_entry &base(const bm2_dup_entry &e) { return e; }
    static const bm2_dup_entry &base(const bm2_dup_loc_entry &e) { return e.e; }
    template <class E> static bool key_less(const E &x, const E &y) {
        const bm2_dup_entry &a = base(x), &b = base(y);
        return a.k1 != b.k1 ? a.k1 < b.k1 : a.k2 < b.k2;
    }

    // every duplicate template of both spaces, as the bitset given to dup_set
    void resolve() {
        std::vector<uint64_t> bits((size_t) ((n_reads + 63) / 64), 0);
        const bool spilled = dup_sig_runs > 0;
        if (spilled && (!sig_cur[0].empty() || !sig_cur[1].empty() || !lsig_cur.empty())) {
            move_sigs_to_pending();
            spill_sigs();
        }
        auto mark = [&](const int64_t *d, int64_t nd, int64_t &count) {
            for (int64_t i = 0; i < nd; ++i) {
                if (d[i] < 0 || d[i] >= n_reads) fail("a duplicate template id beyond the reads");
                bits[(size_t) (d[i] >> 6)] |= (uint64_t) 1 << (d[i] & 63);
            }
            count += nd;
        };
        for (int s = 0; s < 2; ++s) {
            int64_t &count = s ? dup_frag_templates : dup_pair_templates;
            if (s == 0 && dup_ex) {
                resolve_space(lsig_cur, sig_runs[0], spilled, [&](const std::vector<bm2_dup_loc_entry> &v) {
                    const int64_t *d = nullptr; int64_t nd = 0, nopt = 0; double ds = 0;
                    if (dup_ex(v.data(), (int64_t) v.size(), 1, nullptr, &d, &nd, &nopt, &ds)) fail("bm2_dup_resolve_ex");
                    markdup_s += ds;
                    dup_optical_pairs += nopt;
                    mark(d, nd, count);
                });
                continue;
            }
            resolve_space(sig_cur[s], sig_runs[s], spilled, [&](const std::vector<bm2_dup_entry> &v) {
                const int64_t *d = nullptr; int64_t nd = 0; double ds = 0;
                if (dup(v.data(), (int64_t) v.size(), 1, nullptr, &d, &nd, &ds)) fail("bm2_dup_resolve");
                markdup_s += ds;
                mark(d, nd, count);
            });
        }
        if (dup_set(bits.data(), n_reads)) fail("bm2_dup_set");
    }

    // one space: its entries in one call when nothing spilled, else its sorted runs window by window, keys strictly below T settling, so
    // that every group is resolved whole
    template <class E, class Take> void resolve_space(std::vector<E> &cur, std::vector<SigRun> &rs, bool spilled, Take take) {
        if (!spilled) { take(cur); std::vector<E>().swap(cur); return; }
        const size_t nr = rs.size();
        if (!nr) return;
        const int64_t quota = std::max<int64_t>(sig_bytes / (int64_t) sizeof(E) / (int64_t) nr, 1);
        std::vector<std::vector<E>> buf(nr);
        std::vector<int64_t> left(nr);
        for (size_t r = 0; r < nr; ++r) left[r] = rs[r].n;
        auto load = [&](size_t r, int64_t k) {
            k = std::min(k, left[r]);
            if (k <= 0) return;
            const size_t at = buf[r].size();
            buf[r].resize(at + (size_t) k);
            if (fread(buf[r].data() + at, sizeof(E), (size_t) k, rs[r].f) != (size_t) k) fail("cannot read a temporary file");
            left[r] -= k;
        };
        std::vector<E> win;
        for (bool grow = false;;) {
            for (size_t r = 0; r < nr; ++r) if (!grow) load(r, quota - (int64_t) buf[r].size());
            grow = false;
            bool open = false; E T{};
            for (size_t r = 0; r < nr; ++r)
                if (left[r] > 0 && (!open || key_less(buf[r].back(), T))) { T = buf[r].back(); open = true; }
            win.clear();
            for (size_t r = 0; r < nr; ++r) {
                size_t k = 0;
                while (k < buf[r].size() && (!open || key_less(buf[r][k], T))) ++k;
                win.insert(win.end(), buf[r].begin(), buf[r].begin() + (long) k);
                buf[r].erase(buf[r].begin(), buf[r].begin() + (long) k);
            }
            if (open && win.empty()) {               // one group fills the window: load more of the runs that end in it
                for (size_t r = 0; r < nr; ++r) if (left[r] > 0 && !key_less(T, buf[r].back())) load(r, quota);
                grow = true;
                continue;
            }
            if (!win.empty()) take(win);
            if (!open) break;
        }
    }

    struct Cursor {                              // a run being merged
        size_t next = 0;                          // next member to load
        std::vector<uint8_t> buf; size_t pos = 0; // loaded bytes, consumed up to pos
        std::vector<size_t> recs;                 // whole records at buf[pos..]: their starts
        std::vector<int64_t> tids;                // --markdup: their template ids
    };

    static uint64_t key_at(const uint8_t *r) { const BamFixed f = bam_fixed(r); return bam_coord_key(f.rid, f.pos, f.flag); }
    int rec_cmp(const uint8_t *a, const uint8_t *b) const {
        if (cmp) return cmp(a, b);
        const uint64_t x = key_at(a), y = key_at(b);
        return x < y ? -1 : x > y ? 1 : 0;
    }

    void merge(SortedWriter &w) {
        const double t0 = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
        const size_t nr = runs.size();
        const int64_t quota = std::max<int64_t>(run_bytes / (int64_t) nr, BGZF_BLOCK);
        std::vector<Cursor> c(nr);
        std::vector<uint8_t> win; std::vector<int64_t> win_starts, win_tids;
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
                std::vector<InflateJob> ij;
                for (const Job &j : jobs) {
                    uint32_t crc; memcpy(&crc, j.z.data() + j.z.size() - 8, 4);
                    ij.push_back({j.z.data() + 18, j.z.size() - 26, c[j.run].buf.data() + j.at, j.isize, crc});
                }
                if (!bgzf_inflate(ij, threads)) fail("a temporary file does not inflate");
                for (size_t r = 0; r < nr; ++r) {                                    // the whole records now loaded
                    Cursor &x = c[r];
                    size_t q = x.recs.empty() ? x.pos : x.recs.back() + 4 + (size_t) bam_le32(x.buf.data() + x.recs.back());
                    while (q + 4 <= x.buf.size() && q + 4 + (size_t) bam_le32(x.buf.data() + q) <= x.buf.size()) {
                        x.recs.push_back(q); q += 4 + (size_t) bam_le32(x.buf.data() + q);
                    }
                    if (dup && x.tids.size() < x.recs.size()) {                       // their ids, read in step
                        const size_t at = x.tids.size();
                        x.tids.resize(x.recs.size());
                        if (fread(x.tids.data() + at, 8, x.tids.size() - at, runs[r].tf) != x.tids.size() - at) fail("cannot read a temporary file");
                    }
                }
            }
            // T and r* over the runs not fully loaded
            bool open = false; const uint8_t *T = nullptr; size_t rs = 0;
            for (size_t r = 0; r < nr; ++r) {
                if (c[r].next >= runs[r].members.size()) continue;
                const uint8_t *k = c[r].buf.data() + c[r].recs.back();
                if (!open || rec_cmp(k, T) < 0) { T = k; rs = r; open = true; }
            }
            win.clear(); win_starts.clear(); win_tids.clear();
            for (size_t r = 0; r < nr; ++r) {
                Cursor &x = c[r];
                size_t k = 0;
                while (k < x.recs.size()) {
                    const int o = open ? rec_cmp(x.buf.data() + x.recs[k], T) : -1;
                    if (o > 0 || (o == 0 && r > rs)) break;
                    ++k;
                }
                if (!k) continue;
                const size_t b = x.recs[0], e = x.recs[k - 1] + 4 + (size_t) bam_le32(x.buf.data() + x.recs[k - 1]);
                for (size_t i = 0; i < k; ++i) win_starts.push_back((int64_t) (win.size() + x.recs[i] - b));
                win.insert(win.end(), x.buf.begin() + (long) b, x.buf.begin() + (long) e);
                x.recs.erase(x.recs.begin(), x.recs.begin() + (long) k);
                if (dup) { win_tids.insert(win_tids.end(), x.tids.begin(), x.tids.begin() + (long) k); x.tids.erase(x.tids.begin(), x.tids.begin() + (long) k); }
                x.pos = e;
            }
            w.write(win.data(), (int64_t) win.size(), win_starts.data(), (int64_t) win_starts.size(), dup ? win_tids.data() : nullptr, !open);
            ++merge_windows;
            if (!open) break;
        }
        for (size_t r = 0; r < nr; ++r) if (c[r].pos != c[r].buf.size()) fail("a temporary file ends inside a record");
        merge_s += std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count() - t0;
    }
};

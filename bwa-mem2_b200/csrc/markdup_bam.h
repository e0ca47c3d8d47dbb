// markdup_bam.h — the host half of bm2_markdup: Picard MarkDuplicates over one or more coordinate-sorted BAM files, written as one merged,
// marked BAM and a DuplicationMetrics file.  The device calls are parameters, so that tests/host_emul/markdup_bam_emul.cpp runs all of this
// with the GPU swapped for a CPU restatement.
//
//   inputs    each read by a BamWindowReader in windows of about `window` bytes; every input needs @HD SO:coordinate and the first input's @SQ
//             list (names, lengths, order).  A record whose coordinate key is below the one before it in its input is an error naming it.
//   merge     (MdbMerge) the inputs' records by bam_coord_key (refID -1 last), ties by input index and then by place in the input.  T is the
//             smallest last-loaded key over the inputs not yet fully loaded and r* the first such input whose last key is T; every loaded
//             record with key < T, and those with key == T of inputs up to r*, are settled and merged into the next window.  A record's
//             ordinal is its 0-based index in the merged stream.  The second pass re-reads the files and merges them the same way.
//   header    the first input's @HD and @SQ lines; the @RG lines of all inputs in input order (an ID seen before: written once when the line is
//             identical, an error otherwise); the @PG lines of all inputs, identical lines once, a later line whose ID is taken by another
//             line renamed ID.1, ID.2, ... with that input's PP references renamed to match; the @CO lines; then @PG ID:bm2_markdup (suffixed
//             the same way when taken) with PP the first input's last @PG.  Other header lines are not written.
//   libraries the LB values of the merged @RG lines and "Unknown Library", sorted by name in byte order.  A record's library is that of its
//             RG:Z value's @RG line; without the tag, with a value that is no @RG ID, or with an @RG line without LB: Unknown Library.
//   entries   (first pass) bm2_markdup_records gives each record's kind, end, score, read group, library and location.  A fragment gives
//             a fragment entry.  A half (0x1 without 0x8) is held, keyed by (QNAME, read group: its RG:Z value, records without the tag
//             sharing one), until the other half of that key arrives: after each window, the halves held from earlier windows (name bytes
//             included) and the window's own go to bm2_markdup_pair, which sorts them by (name hash, read group, ordinal) on the device and
//             joins them by name byte for byte within each run of equal hashes (dup_pair_run: each half to the first earlier unjoined half
//             of its name).  A joined pair gives, by dup_template_entries, the pair entry (located, its class and read group in loc:
//             DUP_LOC_RG_SHIFT) and the two pair-end entries, with tid the smaller ordinal.  An unmapped primary with 0x1 and without 0x8
//             is held the same way so that a half whose mate is unmapped is found.  A read group index must fit loc's bits above
//             DUP_LOC_RG_SHIFT; more distinct RG:Z values are an error.  After each window a held half
//             whose mate's (refID, pos) is before the window's last record is an error (its mate was missed, or a third primary has the
//             name), and a held unmapped record is dropped; a half still held at the end is an error.  The largest count held is
//             pending_max.  Each pair's two ordinals are kept for the mark pass: 16 bytes per pair of host memory.
//   resolve   one BamSortSink per library takes its entries (add_sigs_ex), spills them to sorted runs past sig_bytes / (the header's
//             libraries) - so that sig_bytes bounds them all together - (half filling while
//             the other half is sorted and written) and resolves them with its windowed resolve: bm2_mem --markdup's code.  The sinks'
//             sorter threads may call dup / dup_ex at the same time, so those calls must be safe to make from several threads.  Groups never
//             mix libraries, and each sink's optical count is its library's.  The duplicates' tids become a bitset of 1 bit per record; a
//             pair's second ordinal takes its first's bit; the bitset goes to the device (bm2_dup_set).
//   mark      (second pass) bm2_markdup_mark rewrites every record's 0x400 from the bitset and compresses the stream; the blocks are cut
//             by htslib's rule over all of it, so the bytes depend neither on the window nor on the threads.
//   output    written to <out>.tmp (or standard output) and renamed when complete; the index (BaiBuilder) to <out>.bai and the metrics
//             (markdup_metrics.h, one row per library with a record, by name) through <path>.tmp.  An error removes them.
#pragma once
#include "bam_window.h"
#include "bqsr_device.cuh"
#include "markdup_metrics.h"
#include <memory>
#include <set>

// one window's records (bm2_markdup_records): *out gets one bm2_markdup_rec per record
using MdbRecordsCall = std::function<int(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const bm2_markdup_rec **out)>;
// the halves of a window, carried ones first (bm2_markdup_pair): *partner gets each one's partner index or -1
using MdbPairCall = std::function<int(const bm2_markdup_half *h, int64_t n, const uint8_t *names, int64_t names_len, const int32_t **partner)>;
// the per-library counts since the start (bm2_markdup_counts: 2 per library)
using MdbCountsCall = std::function<int(int64_t *counts)>;
// one window of the second pass (bm2_markdup_mark)
using MdbMarkCall = std::function<int(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, int64_t first, const uint8_t *carry,
                                      int64_t carry_len, int last, bm2_sort_out *out)>;
// bytes compressed as BGZF blocks of their own (bm2_bgzf_compress without cuts)
using MdbCompressCall = std::function<int(const uint8_t *p, int64_t n, std::string *z)>;
// reports an error with the exit code and does not return
using MdbFail = std::function<void(int code, const std::string &)>;

// the value of a header line's tag ("ID:"), empty without it
inline std::string mdb_tag(const std::string &line, const char *tag) {
    const size_t at = line.find(std::string("\t") + tag);
    if (at == std::string::npos) return "";
    const size_t b = at + 4, e = line.find('\t', b);
    return line.substr(b, (e == std::string::npos ? line.size() : e) - b);
}

// the line with its first tag `tag` set to v
inline std::string mdb_set_tag(const std::string &line, const char *tag, const std::string &v) {
    const size_t at = line.find(std::string("\t") + tag);
    if (at == std::string::npos) return line;
    const size_t b = at + 4, e = line.find('\t', b);
    return line.substr(0, b) + v + (e == std::string::npos ? "" : line.substr(e));
}

inline std::vector<std::string> mdb_lines(const std::string &text) {
    std::vector<std::string> v;
    std::string t = text;
    while (!t.empty() && t.back() == '\0') t.pop_back();
    for (size_t b = 0; b < t.size();) {
        size_t e = t.find('\n', b); if (e == std::string::npos) e = t.size();
        if (e > b) v.push_back(t.substr(b, e - b));
        b = e + 1;
    }
    return v;
}

struct MdbHeader {
    std::string text;                                        // the output header's text
    std::vector<std::pair<std::string, int32_t>> refs;
    std::vector<std::string> rg_ids;                         // the merged @RG IDs
    std::vector<int32_t> rg_lib;                             // their libraries
    std::vector<std::string> libs;                           // the libraries by name
    int32_t unknown_lib = 0;
};

// the inputs' header texts and references -> the merged header (cl: this program's command line); returns an error or ""
inline std::string mdb_merge_headers(const std::vector<std::string> &names, const std::vector<std::string> &texts,
                                     const std::vector<std::vector<std::pair<std::string, int32_t>>> &refs, const std::string &cl, MdbHeader &h) {
    std::string hd, sq, rg, pg, co;
    std::map<std::string, std::string> rg_line;               // ID -> its line
    std::set<std::string> pg_lines, pg_ids;
    std::vector<std::string> rg_lb;
    std::string first_last_pg;
    for (size_t i = 0; i < texts.size(); ++i) {
        if (refs[i] != refs[0]) return names[i] + ": its @SQ lines differ from those of " + names[0];
        std::string so;
        std::map<std::string, std::string> ren;               // this input's @PG IDs -> their IDs in the output
        for (const std::string &l : mdb_lines(texts[i])) {
            if (l.compare(0, 4, "@HD\t") == 0) { if (so.empty()) so = mdb_tag(l, "SO:"); if (i == 0 && hd.empty()) hd = l + "\n"; }
            else if (l.compare(0, 4, "@SQ\t") == 0) { if (i == 0) sq += l + "\n"; }
            else if (l.compare(0, 4, "@RG\t") == 0) {
                const std::string id = mdb_tag(l, "ID:");
                auto it = rg_line.find(id);
                if (it != rg_line.end()) {
                    if (it->second != l) return names[i] + ": read group " + id + " differs from the @RG line of the same ID before it";
                    continue;
                }
                rg_line[id] = l;
                rg += l + "\n";
                h.rg_ids.push_back(id);
                rg_lb.push_back(mdb_tag(l, "LB:"));
            } else if (l.compare(0, 4, "@PG\t") == 0) {
                const std::string id = mdb_tag(l, "ID:"), pp = mdb_tag(l, "PP:");
                std::string m = l;
                if (!pp.empty() && ren.count(pp)) m = mdb_set_tag(m, "PP:", ren[pp]);
                if (pg_lines.count(m)) { ren[id] = id; if (i == 0) first_last_pg = id; continue; }
                std::string nid = id;
                for (int k = 1; pg_ids.count(nid); ++k) nid = id + "." + std::to_string(k);
                if (nid != id) m = mdb_set_tag(m, "ID:", nid);
                ren[id] = nid;
                if (i == 0) first_last_pg = nid;
                pg_lines.insert(m); pg_ids.insert(nid);
                pg += m + "\n";
            } else if (l.compare(0, 4, "@CO\t") == 0) co += l + "\n";
        }
        if (so != "coordinate") return names[i] + ": not coordinate-sorted (no @HD SO:coordinate)";
    }
    std::string id = "bm2_markdup";
    for (int k = 1; pg_ids.count(id); ++k) id = "bm2_markdup." + std::to_string(k);
    pg += "@PG\tID:" + id + "\tPN:bm2_markdup" + (first_last_pg.empty() ? "" : "\tPP:" + first_last_pg) + "\tVN:b200-r2\tCL:" + cl + "\n";
    h.text = hd + sq + rg + pg + co;
    h.refs = refs[0];
    std::set<std::string> ls(rg_lb.begin(), rg_lb.end());
    ls.erase("");
    ls.insert("Unknown Library");
    h.libs.assign(ls.begin(), ls.end());
    auto lib_of = [&](const std::string &lb) { return (int32_t) (std::lower_bound(h.libs.begin(), h.libs.end(), lb.empty() ? "Unknown Library" : lb) - h.libs.begin()); };
    for (const std::string &lb : rg_lb) h.rg_lib.push_back(lib_of(lb));
    h.unknown_lib = lib_of("");
    return "";
}

// the inputs' records merged into windows (see the file's comment)
struct MdbMerge {
    struct Src { BamWindowReader rd; std::vector<uint8_t> buf; std::vector<int64_t> st; size_t k = 0; bool done = false; uint64_t last = 0; int64_t seen = 0; };
    std::vector<std::unique_ptr<Src>> src;
    MdbFail fail;

    static uint64_t key_at(const uint8_t *r) { const BamFixed f = bam_fixed(r); return bam_coord_key(f.rid, f.pos, f.flag); }

    // opens every input and reads its header
    void open(const std::vector<std::string> &paths, int threads, int64_t window, std::vector<std::string> *texts,
              std::vector<std::vector<std::pair<std::string, int32_t>>> *refs) {
        for (const std::string &p : paths) {
            src.emplace_back(new Src);
            Src &s = *src.back();
            s.rd.name = p; s.rd.threads = threads; s.rd.window = window;
            s.rd.f = fopen(p.c_str(), "rb");
            if (!s.rd.f) fail(1, "cannot open " + p);
            std::string t; std::vector<std::pair<std::string, int32_t>> r;
            const std::string e = s.rd.header(t, r);
            if (!e.empty()) fail(1, e);
            if (texts) texts->push_back(t);
            if (refs) refs->push_back(r);
        }
    }
    ~MdbMerge() { for (auto &s : src) if (s->rd.f) fclose(s->rd.f); }

    int64_t in_bytes() const { int64_t b = 0; for (auto &s : src) b += s->rd.in_bytes; return b; }
    double inflate_s() const { double t = 0; for (auto &s : src) t += s->rd.inflate_s; return t; }
    std::string warnings() const { std::string w; for (auto &s : src) if (!s->rd.warning.empty()) w += s->rd.warning + "\n"; return w; }

    void load(Src &s) {
        const std::string e = s.rd.next(s.buf, s.st);
        if (!e.empty()) fail(1, e);
        s.k = 0;
        if (s.st.empty()) { s.done = true; return; }
        for (size_t i = 0; i < s.st.size(); ++i) {
            const uint64_t k = key_at(s.buf.data() + s.st[i]);
            if (s.seen + (int64_t) i > 0 && k < s.last)
                fail(1, s.rd.name + ": read " + std::string((const char *) s.buf.data() + s.st[i] + 36) + " is out of coordinate order");
            s.last = k;
        }
        s.seen += (int64_t) s.st.size();
    }

    // the next merged window (records contiguous, their starts, each one's input); false at the end
    bool next(std::vector<uint8_t> &win, std::vector<int64_t> &starts, std::vector<int32_t> &from) {
        win.clear(); starts.clear(); from.clear();
        for (auto &s : src) if (!s->done && s->k == s->st.size()) load(*s);
        bool open = false; uint64_t T = 0; size_t rs = 0;
        for (size_t r = 0; r < src.size(); ++r) {
            const Src &s = *src[r];
            if (s.done || (s.rd.ended && s.rd.rest.empty())) continue;   // fully loaded
            const uint64_t k = key_at(s.buf.data() + s.st.back());
            if (!open || k < T) { T = k; rs = r; open = true; }
        }
        std::vector<size_t> end(src.size());
        for (size_t r = 0; r < src.size(); ++r) {
            const Src &s = *src[r];
            size_t k = s.k;
            if (!s.done)
                while (k < s.st.size()) {
                    const uint64_t kk = key_at(s.buf.data() + s.st[k]);
                    if (open && (kk > T || (kk == T && r > rs))) break;
                    ++k;
                }
            end[r] = k;
        }
        for (;;) {                                                        // merged by (key, input)
            size_t best = src.size(); uint64_t bk = 0;
            for (size_t r = 0; r < src.size(); ++r) {
                const Src &s = *src[r];
                if (s.k >= end[r]) continue;
                const uint64_t k = key_at(s.buf.data() + s.st[s.k]);
                if (best == src.size() || k < bk) { best = r; bk = k; }
            }
            if (best == src.size()) break;
            Src &s = *src[best];
            const uint8_t *p = s.buf.data() + s.st[s.k];
            const size_t m = 4 + (size_t) bam_le32(p);
            starts.push_back((int64_t) win.size());
            from.push_back((int32_t) best);
            win.insert(win.end(), p, p + m);
            ++s.k;
        }
        return !starts.empty();
    }
};

struct MarkdupBam {
    // settings
    std::vector<std::string> paths;
    std::string out_path, metrics_path, bai_path, args, cl;  // out_path empty: standard output; bai_path empty: no index
    int threads = 1;
    int64_t window = (int64_t) 256 << 20, sig_bytes = (int64_t) 1 << 30, distance = 100;
    MdbRecordsCall records; MdbPairCall pair; MdbCountsCall counts; MdbMarkCall mark; MdbCompressCall compress;
    DupCall dup; DupCallEx dup_ex; DupSetCall dup_upload;
    std::function<int(const MdbHeader &)> set_header;          // the read groups to the device (bm2_markdup_set)
    MdbFail fail;
    // state
    MdbHeader hdr;
    std::vector<std::string> tmps;                             // files being written, removed on an error
    // stats
    int64_t n_records = 0, n_pairs = 0, n_frags = 0, pending_max = 0, n_windows = 0, dup_pair_templates = 0, dup_frag_templates = 0, dup_records = 0;
    int64_t dup_optical_pairs = 0, dup_sig_runs = 0, dup_sig_bytes = 0, in_bytes = 0, out_bytes = 0, n_libraries = 0;
    double inflate_s = 0, resolve_s = 0;
    std::string warning;

    [[noreturn]] void die(int code, const std::string &m) {
        for (const std::string &p : tmps) unlink(p.c_str());
        tmps.clear();
        fail(code, m);
        abort();
    }
    MdbFail failer() { return [this](int c, const std::string &m) { die(c, m); }; }

    struct Held { int64_t ord; uint64_t end, hash; int32_t score, flag, kind, lib, rgk, mrid, mpos, input, tile, x, y, loc; std::string name; };

    static std::string qname(const uint8_t *r) { return std::string((const char *) r + 36, r[12] ? r[12] - 1 : 0); }

    // the first pass: every library's entries resolved into the bitset, uploaded; the metrics rows
    std::vector<DupMetrics> first_pass() {
        MdbMerge mg; mg.fail = failer();
        std::vector<std::string> texts;
        std::vector<std::vector<std::pair<std::string, int32_t>>> refs;
        mg.open(paths, threads, window, &texts, &refs);
        const std::string e = mdb_merge_headers(paths, texts, refs, cl, hdr);
        if (!e.empty()) die(1, e);
        if (set_header(hdr)) die(3, "bm2_markdup_set");
        const size_t nl = hdr.libs.size();
        std::vector<std::unique_ptr<BamSortSink>> sinks;
        std::vector<uint64_t> bits;
        for (size_t l = 0; l < nl; ++l) {
            sinks.emplace_back(new BamSortSink);
            BamSortSink &s = *sinks.back();
            s.dup = dup; s.dup_ex = dup_ex;
            s.dup_set = [&bits](const uint64_t *b, int64_t n_bits) {
                for (size_t w = 0; w < (size_t) ((n_bits + 63) / 64); ++w) bits[w] |= b[w];
                return 0;
            };
            s.fail = [this](const std::string &m) { die(2, m); };
            s.sig_bytes = std::max<int64_t>(sig_bytes / (int64_t) nl, 1); s.threads = threads;
            s.tmp_prefix = metrics_path + ".tmp." + std::to_string(l) + ".";
        }
        std::vector<uint8_t> win; std::vector<int64_t> st; std::vector<int32_t> from;
        std::vector<Held> held;                                  // halves whose mates are still to come, in ordinal order
        std::vector<std::pair<int64_t, int64_t>> pairs;        // each pair's two ordinals
        std::map<std::string, int32_t> other_rg;                // RG:Z values that are no @RG ID
        std::vector<char> seen(nl, 0);
        std::vector<std::vector<bm2_dup_loc_entry>> lp(nl);
        std::vector<std::vector<bm2_dup_entry>> fe(nl);
        const int32_t n_ids = (int32_t) hdr.rg_ids.size();
        while (mg.next(win, st, from)) {
            const bm2_markdup_rec *R = nullptr;
            if (records(win.data(), (int64_t) win.size(), st.data(), (int64_t) st.size(), &R)) die(3, "bm2_markdup_records");
            for (size_t i = 0; i < st.size(); ++i) {
                const uint8_t *r = win.data() + st[i];
                const bm2_markdup_rec &x = R[i];
                const int64_t ord = n_records + (int64_t) i;
                seen[(size_t) x.lib] = 1;
                if (x.kind == BM2_MDB_FRAG) { fe[(size_t) x.lib].push_back(bm2_dup_entry{x.end, 0, ord, x.score, DUP_KIND_FRAG}); continue; }
                if (x.kind != BM2_MDB_HALF && x.kind != BM2_MDB_UNMAPPED_HALF) continue;
                int32_t rgk = x.rg;
                if (rgk < 0) {                                   // the value is no @RG ID: a read group of its own past the header's
                    int32_t len = 0;
                    const int32_t at = bqsr_aux_rg(r, &len);
                    const std::string v((const char *) r + at, (size_t) len);
                    auto it = other_rg.find(v);
                    if (it == other_rg.end() && (int64_t) n_ids + 1 + (int64_t) other_rg.size() >= ((int64_t) 1 << (32 - DUP_LOC_RG_SHIFT)))
                        die(1, paths[(size_t) from[i]] + ": read " + qname(r) + ": more distinct RG:Z values than loc's read-group bits hold");
                    rgk = it != other_rg.end() ? it->second : (other_rg[v] = n_ids + 1 + (int32_t) other_rg.size());
                }
                const BamFixed f = bam_fixed(r);
                held.push_back(Held{ord, x.end, x.hash, x.score, f.flag, x.kind, x.lib, rgk, bam_le32(r + 24), bam_le32(r + 28), from[i], x.tile, x.x,
                                    x.y, x.loc, qname(r)});
            }
            // the carried halves and this window's, paired on the device by (hash, read group) and then by name
            std::vector<bm2_markdup_half> hs(held.size());
            std::string names;
            for (size_t k = 0; k < held.size(); ++k) {
                hs[k] = bm2_markdup_half{held[k].hash, held[k].rgk, (int32_t) held[k].name.size(), (int64_t) names.size()};
                names += held[k].name;
            }
            const int32_t *partner = nullptr;
            if (pair(hs.data(), (int64_t) hs.size(), (const uint8_t *) names.data(), (int64_t) names.size(), &partner)) die(3, "bm2_markdup_pair");
            std::vector<Held> open;
            for (size_t k = 0; k < held.size(); ++k) {
                const int32_t p = partner[k];
                if (p < 0) { open.push_back(std::move(held[k])); continue; }
                if ((size_t) p < k) continue;
                const Held &h = held[k], &x = held[(size_t) p];              // h has the smaller ordinal
                if (h.kind == BM2_MDB_UNMAPPED_HALF && x.kind == BM2_MDB_UNMAPPED_HALF) continue;
                if (h.kind != x.kind)
                    die(1, paths[(size_t) (x.kind == BM2_MDB_HALF ? x.input : h.input)] + ": read " + h.name + " lacks flag 0x8, but its mate is unmapped");
                const int mapped[2] = { 1, 1 };
                const uint64_t end[2] = { h.end, x.end };
                const int32_t score[2] = { h.score, x.score };
                bm2_dup_entry pe, pf[2];
                int has_pair = 0, n_frag = 0;
                dup_template_entries(2, mapped, end, score, h.ord, &pe, &has_pair, pf, &n_frag);
                const int32_t loc = h.loc | dup_pair_class(h.flag, x.flag) | (int32_t) ((uint32_t) h.rgk << DUP_LOC_RG_SHIFT);
                lp[(size_t) x.lib].push_back(bm2_dup_loc_entry{pe, h.tile, h.x, h.y, loc});
                fe[(size_t) x.lib].insert(fe[(size_t) x.lib].end(), pf, pf + n_frag);
                pairs.push_back({h.ord, x.ord});
            }
            held.swap(open);
            n_records += (int64_t) st.size();
            ++n_windows;
            pending_max = std::max<int64_t>(pending_max, (int64_t) held.size());
            // a held record whose mate lies before the window's last record: a half is an error, an unmapped record is dropped
            const BamFixed lf = bam_fixed(win.data() + st.back());
            auto before_last = [&](int32_t rid, int32_t pos) {
                return (uint32_t) rid != (uint32_t) lf.rid ? (uint32_t) rid < (uint32_t) lf.rid : pos < lf.pos;
            };
            std::vector<Held> kept;
            const Held *bad = nullptr;
            for (Held &h : held) {
                if (!before_last(h.mrid, h.mpos)) kept.push_back(std::move(h));
                else if (h.kind == BM2_MDB_HALF) { if (!bad) bad = &h; }      // in ordinal order: the first is the smallest
            }
            if (bad)
                die(1, paths[(size_t) bad->input] + ": read " + bad->name + ": no mate at its mate position " + std::to_string(bad->mrid) + ":" +
                           std::to_string((int64_t) bad->mpos + 1) + " (a missing mate, or a third primary record of that name)");
            held.swap(kept);
            for (size_t l = 0; l < nl; ++l) {
                if (lp[l].empty() && fe[l].empty()) continue;
                n_pairs += (int64_t) lp[l].size();
                for (const bm2_dup_entry &x : fe[l]) n_frags += x.kind == DUP_KIND_FRAG;
                sinks[l]->add_sigs_ex(lp[l].data(), (int64_t) lp[l].size(), fe[l].data(), (int64_t) fe[l].size());
                lp[l].clear(); fe[l].clear();
            }
        }
        {
            for (const Held &h : held)
                if (h.kind == BM2_MDB_HALF) die(1, paths[(size_t) h.input] + ": read " + h.name + ": its mate never appears");
        }
        in_bytes = mg.in_bytes(); inflate_s = mg.inflate_s(); warning = mg.warnings();
        std::vector<int64_t> c(2 * nl, 0);
        if (counts(c.data())) die(3, "bm2_markdup_counts");
        bits.assign((size_t) ((n_records + 63) / 64), 0);
        std::vector<DupMetrics> rows;
        for (size_t l = 0; l < nl; ++l) {
            BamSortSink &s = *sinks[l];
            s.n_reads = n_records;
            s.join_sorter();
            s.resolve();
            resolve_s += s.markdup_s;
            dup_pair_templates += s.dup_pair_templates; dup_frag_templates += s.dup_frag_templates; dup_optical_pairs += s.dup_optical_pairs;
            dup_sig_runs += s.dup_sig_runs; dup_sig_bytes += s.dup_sig_bytes;
            if (!seen[l]) continue;
            DupMetrics m;
            m.library = hdr.libs[l];
            m.unpaired_reads = s.dup_frag_entries; m.read_pairs = s.dup_pair_entries;
            m.secondary_or_supplementary = c[2 * l]; m.unmapped = c[2 * l + 1];
            m.unpaired_dups = s.dup_frag_templates; m.pair_dups = s.dup_pair_templates; m.optical_pairs = s.dup_optical_pairs;
            rows.push_back(m);
        }
        n_libraries = (int64_t) rows.size();
        for (const auto &p : pairs)
            if ((bits[(size_t) (p.first >> 6)] >> (p.first & 63)) & 1) bits[(size_t) (p.second >> 6)] |= (uint64_t) 1 << (p.second & 63);
        if (dup_upload(bits.data(), n_records)) die(3, "bm2_dup_set");
        return rows;
    }

    static void write_file(MarkdupBam &m, const std::string &path, const std::string &bytes) {
        const std::string tmp = path + ".tmp";
        m.tmps.push_back(tmp);
        FILE *f = fopen(tmp.c_str(), "wb");
        if (!f || fwrite(bytes.data(), 1, bytes.size(), f) != bytes.size() || fclose(f)) m.die(2, "cannot write " + path);
    }

    // both passes and every file
    void run() {
        const std::vector<DupMetrics> rows = first_pass();
        FILE *out = stdout;
        if (!out_path.empty()) {
            tmps.push_back(out_path + ".tmp");
            out = fopen(tmps.back().c_str(), "wb");
            if (!out) die(2, "cannot open " + out_path + ".tmp");
        }
        std::string h("BAM\1", 4);
        auto i32 = [&](int32_t v) { h.append((const char *) &v, 4); };
        i32((int32_t) hdr.text.size()); h += hdr.text;
        i32((int32_t) hdr.refs.size());
        for (const auto &r : hdr.refs) { i32((int32_t) r.first.size() + 1); h.append(r.first.c_str(), r.first.size() + 1); i32(r.second); }
        std::string z;
        if (compress((const uint8_t *) h.data(), (int64_t) h.size(), &z)) die(3, "bm2_bgzf_compress");
        if (fwrite(z.data(), 1, z.size(), out) != z.size()) die(2, "cannot write the output");
        BaiBuilder bai((int) hdr.refs.size());
        int64_t first = 0;
        SortedWriter w{[this, &first](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, const int64_t *, const uint8_t *c, int64_t cl, int last,
                                      bm2_sort_out *o, const int64_t **, double *) { return mark(r, n, st, nr, first, c, cl, last, o); },
                       [this](const std::string &m) { die(m == "bm2_bam_sort_compress" ? 3 : 2, m == "bm2_bam_sort_compress" ? "bm2_markdup_mark" : m); },
                       out, bai_path.empty() ? nullptr : &bai, (uint64_t) z.size()};
        MdbMerge mg; mg.fail = failer();
        mg.open(paths, threads, window, nullptr, nullptr);
        std::vector<uint8_t> win; std::vector<int64_t> st; std::vector<int32_t> from;
        while (mg.next(win, st, from)) {
            w.write(win.data(), (int64_t) win.size(), st.data(), (int64_t) st.size(), nullptr, false);
            first += (int64_t) st.size();
        }
        if (first != n_records) die(1, "the inputs changed between the two passes");
        in_bytes += mg.in_bytes(); inflate_s += mg.inflate_s();                          // both passes
        w.write(nullptr, 0, nullptr, 0, nullptr, true);
        dup_records = w.marked;
        static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        if (fwrite(eof, 1, sizeof eof, out) != sizeof eof || fflush(out)) die(2, "cannot write the output");
        out_bytes = (int64_t) (w.file_off + sizeof eof);
        if (out != stdout && fclose(out)) die(2, "cannot write " + out_path + ".tmp");
        write_file(*this, metrics_path, dup_metrics_file(rows, "bm2_markdup", args));
        if (!bai_path.empty()) write_file(*this, bai_path, bai.bytes());
        for (const std::string &p : { metrics_path, bai_path, out_path })
            if (!p.empty() && rename((p + ".tmp").c_str(), p.c_str())) die(2, "cannot write " + p);
        tmps.clear();
    }
};

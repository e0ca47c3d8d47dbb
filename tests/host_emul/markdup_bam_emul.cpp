// markdup_bam_emul.cpp — TEST ONLY: bm2_markdup on the CPU.  markdup_bam.h drives it unchanged; the record kernel is restated one record at a
// time over markdup_device.cuh's helpers (the warp's sums as a loop over the 32 lanes), bm2_dup_resolve as markdup_emul.cpp's restatement,
// bm2_dup_resolve_ex's optical count as markdup_metrics_emul.cpp's per group, summed over the group's read groups, and bm2_markdup_mark as the
// flags set from the bitset followed by bam_sort_emul.cpp's compression (the merged stream is already in coordinate order, so its stable
// sort keeps it).  The GPU must give these bytes exactly.
#include "markdup_bam.h"
#include <mutex>
#include <stdexcept>

extern "C" int bam_sort_emul_once(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry, int64_t carry_len,
                                  int last, uint8_t *z, int64_t cap, uint8_t *carry_out, bm2_sort_rec *recs_out, int64_t *sizes);
extern "C" int64_t bgzf_emul(const uint8_t *in, int64_t n, const int64_t *cut, int64_t n_cut, uint8_t *out, int64_t cap);
extern "C" void markdup_emul_resolve(const bm2_dup_entry *e, int64_t n, int res, bm2_dup_entry *sorted_out, int64_t *dups_out, int64_t *n_dups);
extern "C" int64_t mm_optical_group(const bm2_dup_loc_entry *g, int64_t sz, int64_t d);

namespace {

struct RgMap { std::vector<std::string> ids; std::vector<int32_t> libs; int32_t n_lib = 1, unknown_lib = 0; };

// mdb_record_kernel, one record
bm2_markdup_rec record(const uint8_t *rec, const RgMap &m, int64_t *cnt) {
    const int32_t flag = (int32_t) bam_le16(rec + 18);
    int32_t len = 0;
    const int32_t at = bqsr_aux_rg(rec, &len);
    int rg = (int) m.ids.size(), lib = m.unknown_lib;
    if (at >= 0) {
        rg = -1;
        for (size_t j = 0; j < m.ids.size(); ++j)
            if (m.ids[j] == std::string((const char *) rec + at, (size_t) len)) { rg = (int) j; lib = m.libs[j]; break; }
    }
    bm2_markdup_rec o{};
    o.rg = rg; o.lib = lib; o.kind = BM2_MDB_NONE;
    if (!dup_is_primary(flag)) ++cnt[2 * lib];
    else if (flag & 4) {
        ++cnt[2 * lib + 1];
        if ((flag & 1) && !(flag & 8)) o.kind = BM2_MDB_UNMAPPED_HALF;
    } else {
        o.kind = (flag & 1) && !(flag & 8) ? BM2_MDB_HALF : BM2_MDB_FRAG;
        uint32_t q = 0;
        for (int lane = 0; lane < 32; ++lane) q += dup_qual_part(rec, lane, 32);
        o.score = dup_read_score(q);
        const DupCigar c = dup_cigar(rec);
        int64_t rl = 0;
        for (int lane = 0; lane < 32; ++lane) rl += dup_ref_len_part(c, lane, 32);
        o.end = dup_read_end(rec, c, rl);
        if (o.kind == BM2_MDB_HALF) o.loc = dup_name_location(rec + 36, std::max<int>((int) rec[12] - 1, 0), &o.tile, &o.x, &o.y);
    }
    if (o.kind == BM2_MDB_HALF || o.kind == BM2_MDB_UNMAPPED_HALF) o.hash = dup_name_hash(rec + 36, std::max<int>((int) rec[12] - 1, 0));
    return o;
}

// bm2_dup_resolve_ex restated with the read groups kept apart in the optical count
void resolve_ex(const bm2_dup_loc_entry *e, int64_t n, int res, int64_t d, std::vector<bm2_dup_loc_entry> &s, std::vector<int64_t> &dups, int64_t *opt) {
    s.assign(e, e + n);
    std::stable_sort(s.begin(), s.end(), [](const bm2_dup_loc_entry &a, const bm2_dup_loc_entry &b) { return dup_less(a.e, b.e); });
    dups.clear();
    if (!res) return;
    std::vector<bm2_dup_entry> base((size_t) n);
    for (int64_t i = 0; i < n; ++i) base[(size_t) i] = e[i].e;
    dups.resize((size_t) n + 1);
    int64_t nd = 0;
    markdup_emul_resolve(base.data(), n, 1, nullptr, dups.data(), &nd);
    dups.resize((size_t) nd);
    *opt = 0;
    for (int64_t g0 = 0; g0 < n;) {
        int64_t g1 = g0 + 1;
        while (g1 < n && dup_same_key(s[(size_t) g1].e, s[(size_t) g0].e)) ++g1;
        if (s[(size_t) g0].e.kind == DUP_KIND_PAIR && g1 - g0 >= 2 && g1 - g0 <= DUP_OPTICAL_MAX_SET) {
            std::map<uint32_t, std::vector<bm2_dup_loc_entry>> by_rg;
            for (int64_t i = g0; i < g1; ++i) by_rg[dup_loc_rg(s[(size_t) i].loc)].push_back(s[(size_t) i]);
            for (auto &kv : by_rg) *opt += mm_optical_group(kv.second.data(), (int64_t) kv.second.size(), d);
        }
        g0 = g1;
    }
}

// bm2_markdup_pair restated: a stable sort of the indices by (hash, read group), then each run as the kernel's thread takes it
void pair(const bm2_markdup_half *h, int64_t n, const uint8_t *names, std::vector<int32_t> &partner) {
    std::vector<uint32_t> ord((size_t) n);
    for (int64_t i = 0; i < n; ++i) ord[(size_t) i] = (uint32_t) i;
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return h[a].hash != h[b].hash ? h[a].hash < h[b].hash : (uint32_t) h[a].rg < (uint32_t) h[b].rg; });
    partner.assign((size_t) n, -1);
    for (int64_t a = 0; a < n;) {
        int64_t b = a + 1;
        while (b < n && h[ord[(size_t) b]].hash == h[ord[(size_t) a]].hash && h[ord[(size_t) b]].rg == h[ord[(size_t) a]].rg) ++b;
        dup_pair_run(h, ord.data(), a, b, names, partner.data());
        a = b;
    }
}

}  // namespace

// bm2_markdup_pair restated, for the tests: partner gets n values
extern "C" void mdb_emul_pair(const bm2_markdup_half *h, int64_t n, const uint8_t *names, int32_t *partner) {
    std::vector<int32_t> p;
    pair(h, n, names, p);
    std::copy(p.begin(), p.end(), partner);
}

// bm2_dup_resolve_ex restated with the read groups kept apart: dups_out (room for n), *n_dups, *n_optical
extern "C" void mdb_emul_resolve_ex(const bm2_dup_loc_entry *e, int64_t n, int64_t d, int64_t *dups_out, int64_t *n_dups, int64_t *n_optical) {
    std::vector<bm2_dup_loc_entry> s; std::vector<int64_t> dd;
    resolve_ex(e, n, 1, d, s, dd, n_optical);
    std::copy(dd.begin(), dd.end(), dups_out);
    *n_dups = (int64_t) dd.size();
}

// the record kernel over one window: ids '\n'-joined (n_ids of them) with their libraries; out gets n_recs records, cnt 2 n_lib counts
extern "C" void mdb_emul_records(const uint8_t *recs, const int64_t *starts, int64_t n_recs, const char *ids, const int32_t *libs, int32_t n_ids,
                                 int32_t n_lib, int32_t unknown_lib, bm2_markdup_rec *out, int64_t *cnt) {
    RgMap m;
    std::string cur;
    if (n_ids)
        for (const char *p = ids;; ++p) {
            if (*p == '\n' || !*p) { m.ids.push_back(cur); cur.clear(); if (!*p) break; } else cur += *p;
        }
    m.libs.assign(libs, libs + n_ids); m.n_lib = n_lib; m.unknown_lib = unknown_lib;
    for (int64_t i = 0; i < n_recs; ++i) out[i] = record(recs + starts[i], m, cnt);
}

// bm2_markdup over the files (paths '\n'-joined): returns the exit code, with the message in err; stats: records, pairs, fragments,
// pending_max, pair duplicates, fragment duplicates, records marked, optical, signature runs, signature bytes, windows, libraries
extern "C" int mdb_emul_run(const char *paths, const char *out_path, const char *metrics_path, const char *bai_path, const char *args, const char *cl,
                            int threads, int64_t window, int64_t sig_bytes, int64_t distance, int64_t *stats, char *err, int err_cap) {
    struct Fail { int code; std::string m; };
    MarkdupBam md;
    std::string p = paths;
    for (size_t b = 0; b <= p.size();) { size_t e = p.find('\n', b); if (e == std::string::npos) e = p.size(); md.paths.push_back(p.substr(b, e - b)); b = e + 1; }
    md.out_path = out_path; md.metrics_path = metrics_path; md.bai_path = bai_path; md.args = args; md.cl = cl;
    md.threads = threads; md.window = window; md.sig_bytes = sig_bytes; md.distance = distance;
    md.fail = [](int code, const std::string &m) { throw Fail{code, m}; };
    RgMap map;
    std::vector<int64_t> cnt;
    std::vector<bm2_markdup_rec> rr;
    std::vector<uint64_t> bits;
    md.set_header = [&](const MdbHeader &h) {
        map.ids = h.rg_ids; map.libs = h.rg_lib; map.n_lib = (int32_t) h.libs.size(); map.unknown_lib = h.unknown_lib;
        cnt.assign(2 * h.libs.size(), 0);
        return 0;
    };
    md.records = [&](const uint8_t *r, int64_t, const int64_t *st, int64_t nr, const bm2_markdup_rec **out) {
        rr.resize((size_t) nr);
        for (int64_t i = 0; i < nr; ++i) rr[(size_t) i] = record(r + st[i], map, cnt.data());
        *out = rr.data();
        return 0;
    };
    std::vector<int32_t> part;
    md.pair = [&](const bm2_markdup_half *h, int64_t n, const uint8_t *names, int64_t, const int32_t **partner) {
        pair(h, n, names, part);
        *partner = part.data();
        return 0;
    };
    md.counts = [&](int64_t *c) { std::copy(cnt.begin(), cnt.end(), c); return 0; };
    std::mutex mu;
    md.dup = [&](const bm2_dup_entry *e, int64_t n, int res, const bm2_dup_entry **sorted, const int64_t **dups, int64_t *n_dups, double *ds) {
        thread_local std::vector<bm2_dup_entry> s; thread_local std::vector<int64_t> d;
        std::lock_guard<std::mutex> g(mu);
        s.resize((size_t) n + 1); d.resize((size_t) n + 1);
        int64_t nd = 0;
        markdup_emul_resolve(e, n, res, s.data(), d.data(), &nd);
        if (res) { *dups = d.data(); *n_dups = nd; } else *sorted = s.data();
        *ds = 0;
        return 0;
    };
    md.dup_ex = [&](const bm2_dup_loc_entry *e, int64_t n, int res, const bm2_dup_loc_entry **sorted, const int64_t **dups, int64_t *n_dups,
                    int64_t *n_opt, double *ds) {
        thread_local std::vector<bm2_dup_loc_entry> s; thread_local std::vector<int64_t> d;
        std::lock_guard<std::mutex> g(mu);
        int64_t opt = 0;
        resolve_ex(e, n, res, distance, s, d, &opt);
        if (res) { *dups = d.data(); *n_dups = (int64_t) d.size(); if (n_opt) *n_opt = opt; } else *sorted = s.data();
        *ds = 0;
        return 0;
    };
    md.dup_upload = [&](const uint64_t *b, int64_t nb) { bits.assign(b, b + (nb + 63) / 64); return 0; };
    std::vector<uint8_t> work, z, carry(65536);
    std::vector<bm2_sort_rec> srecs;
    std::vector<int32_t> sizes;
    md.mark = [&](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, int64_t first, const uint8_t *c, int64_t cl, int last, bm2_sort_out *o) {
        work.assign(r, r + n);
        for (int64_t i = 0; i < nr; ++i) {
            uint8_t *x = work.data() + st[i];
            const int64_t ord = first + i;
            const bool dup = ord < (int64_t) bits.size() * 64 && ((bits[(size_t) (ord >> 6)] >> (ord & 63)) & 1);
            const uint32_t f = (bam_le16(x + 18) & ~0x400u) | (dup ? 0x400u : 0u);
            x[18] = (uint8_t) f; x[19] = (uint8_t) (f >> 8);
        }
        const int64_t cap = n + cl + 64 * (n / 65280 + nr + 4);
        std::vector<uint8_t> cin(c, c + cl);                          // c may be this call's own carry buffer
        z.resize((size_t) cap); srecs.resize((size_t) nr + 1);
        int64_t sz[3];
        if (bam_sort_emul_once(work.data(), n, st, nr, cin.data(), cl, last, z.data(), cap, carry.data(), srecs.data(), sz)) return 1;
        sizes.clear();
        for (int64_t at = 0; at < sz[0];) { const int32_t s = (int32_t) (z[(size_t) at + 16] | z[(size_t) at + 17] << 8) + 1; sizes.push_back(s); at += s; }
        o->z = z.data(); o->z_len = sz[0]; o->member_size = sizes.data(); o->n_members = sz[2];
        o->carry = carry.data(); o->carry_len = sz[1]; o->recs = srecs.data(); o->n_recs = nr;
        return 0;
    };
    md.compress = [](const uint8_t *q, int64_t n, std::string *out) {
        std::vector<uint8_t> b((size_t) (n + 64 * (n / 65280 + 2)));
        const int64_t k = bgzf_emul(q, n, nullptr, 0, b.data(), (int64_t) b.size());
        if (k < 0) return 1;
        out->assign((const char *) b.data(), (size_t) k);
        return 0;
    };
    try {
        md.run();
    } catch (const Fail &f) {
        snprintf(err, (size_t) err_cap, "%s", f.m.c_str());
        return f.code;
    }
    const int64_t v[] = { md.n_records, md.n_pairs, md.n_frags, md.pending_max, md.dup_pair_templates, md.dup_frag_templates, md.dup_records,
                          md.dup_optical_pairs, md.dup_sig_runs, md.dup_sig_bytes, md.n_windows, md.n_libraries };
    std::copy(v, v + 12, stats);
    err[0] = 0;
    return 0;
}

// markdup_emul.cpp — TEST ONLY: bm2_mem --markdup on the CPU.  The per-template and per-group logic is markdup_device.cuh's, compiled here;
// the warp's sums are restated as a loop over the 32 lanes, cub's radix sorts as std::stable_sort by the same order, and
// bm2_bam_sort_compress_ex as bam_sort_emul.cpp's bm2_bam_sort_compress restatement run on the records with the bitset's flags already set
// (the coordinate key does not read 0x400) and the ids carried by the same stable sort.  bam_sort.h drives it all unchanged.  The GPU must
// give these bytes exactly.
#include "bam_sort.h"
#include <numeric>
#include <stdexcept>

extern "C" int bam_sort_emul_once(const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const uint8_t *carry, int64_t carry_len,
                                  int last, uint8_t *z, int64_t cap, uint8_t *carry_out, bm2_sort_rec *recs_out, int64_t *sizes);

namespace {

// one template as the warp of dup_sig_kernel computes it
void template_entries(const uint8_t *recs, const int64_t *starts, int64_t r0, int64_t r1, int64_t tid, std::vector<bm2_dup_entry> &pairs,
                      std::vector<bm2_dup_entry> &frags) {
    int n_prim = 0;
    int64_t prim[2] = { 0, 0 };
    for (int64_t i = r0; i < r1 && n_prim <= 2; ++i)
        if (dup_is_primary((int32_t) bam_le16(recs + starts[i] + 18))) { if (n_prim < 2) prim[n_prim] = i; ++n_prim; }
    int mapped[2] = { 0, 0 };
    uint64_t end[2] = { 0, 0 };
    int32_t score[2] = { 0, 0 };
    for (int k = 0; k < n_prim && k < 2; ++k) {
        const uint8_t *r = recs + starts[prim[k]];
        mapped[k] = !(bam_le16(r + 18) & 4);
        uint32_t q = 0;
        for (int lane = 0; lane < 32; ++lane) q += dup_qual_part(r, lane, 32);
        score[k] = dup_read_score(q);
        if (mapped[k]) {
            const DupCigar c = dup_cigar(r);
            int64_t rl = 0;
            for (int lane = 0; lane < 32; ++lane) rl += dup_ref_len_part(c, lane, 32);
            end[k] = dup_read_end(r, c, rl);
        }
    }
    bm2_dup_entry pe, fe[2];
    int has_pair = 0, n_frag = 0;
    dup_template_entries(n_prim, mapped, end, score, tid, &pe, &has_pair, fe, &n_frag);
    if (has_pair) pairs.push_back(pe);
    for (int k = 0; k < n_frag; ++k) frags.push_back(fe[k]);
}

// bm2_dup_resolve restated: a stable sort, then each group as dup_group_kernel / dup_mark_kernel decide it
void resolve(const bm2_dup_entry *e, int64_t n, int res, std::vector<bm2_dup_entry> &sorted, std::vector<int64_t> &dups) {
    sorted.assign(e, e + n);
    std::stable_sort(sorted.begin(), sorted.end(), [](const bm2_dup_entry &a, const bm2_dup_entry &b) { return dup_less(a, b); });
    dups.clear();
    if (!res) return;
    for (int64_t g0 = 0; g0 < n;) {
        int64_t g1 = g0 + 1;
        while (g1 < n && dup_same_key(sorted[(size_t) g1], sorted[(size_t) g0])) ++g1;
        int has_pe = 0; int64_t first = -1;
        for (int64_t i = g0; i < g1; ++i) {
            if (sorted[(size_t) i].kind == DUP_KIND_PAIR_END) has_pe = 1;
            else if (first < 0) first = i;
        }
        for (int64_t i = g0; i < g1; ++i) if (dup_is_duplicate(sorted[(size_t) i].kind, has_pe, first, i)) dups.push_back(sorted[(size_t) i].tid);
        g0 = g1;
    }
}

struct EmulState {
    std::vector<uint64_t> bits; int64_t n_bits = 0;
    std::vector<uint8_t> z, carry, work; std::vector<bm2_sort_rec> recs; std::vector<int64_t> tids; std::vector<int32_t> sizes;
    std::vector<bm2_dup_entry> sorted; std::vector<int64_t> dups;
};

int emul_sort_ex(EmulState &S, const uint8_t *recs, int64_t n, const int64_t *starts, int64_t n_recs, const int64_t *tids, const uint8_t *carry,
                 int64_t carry_len, int last, bm2_sort_out *out, const int64_t **tids_out) {
    S.work.assign(recs, recs + n);
    std::vector<uint64_t> key((size_t) n_recs);
    for (int64_t i = 0; i < n_recs; ++i) {
        uint8_t *r = S.work.data() + starts[i];
        if (tids && S.n_bits) {
            const uint16_t f = dup_marked_flag((uint16_t) bam_le16(r + 18), tids[i], S.bits.data(), S.n_bits);
            r[18] = (uint8_t) f; r[19] = (uint8_t) (f >> 8);
        }
        const BamFixed f = bam_fixed(r);
        key[(size_t) i] = bam_coord_key(f.rid, f.pos, f.flag);
    }
    std::vector<int64_t> ord((size_t) n_recs);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int64_t a, int64_t b) { return key[(size_t) a] < key[(size_t) b]; });
    S.tids.clear();
    if (tids) for (int64_t k : ord) S.tids.push_back(tids[k]);
    const int64_t cap = n + carry_len + 64 * (n / 65280 + n_recs + 4);
    S.z.resize((size_t) cap); S.carry.resize(65536); S.recs.resize((size_t) n_recs + 1);
    int64_t sizes[3];
    if (bam_sort_emul_once(S.work.data(), n, starts, n_recs, carry, carry_len, last, S.z.data(), cap, S.carry.data(), S.recs.data(), sizes)) return 1;
    // member sizes from the BSIZE fields
    S.sizes.clear();
    for (int64_t at = 0; at < sizes[0];) { const int32_t sz = (int32_t) (S.z[(size_t) at + 16] | S.z[(size_t) at + 17] << 8) + 1; S.sizes.push_back(sz); at += sz; }
    out->z = S.z.data(); out->z_len = sizes[0];
    out->member_size = S.sizes.data(); out->n_members = sizes[2];
    out->carry = S.carry.data(); out->carry_len = sizes[1];
    out->recs = S.recs.data(); out->n_recs = n_recs;
    if (tids_out) *tids_out = tids ? S.tids.data() : nullptr;
    return 0;
}

}  // namespace

// bm2_dup_signatures restated: pairs_out / frags_out have room for n_tmpl / 2 n_tmpl entries
extern "C" void markdup_emul_signatures(const uint8_t *recs, const int64_t *starts, const int64_t *tmpl_first, const int64_t *tmpl_id, int64_t n_tmpl,
                                        bm2_dup_entry *pairs_out, int64_t *n_pairs, bm2_dup_entry *frags_out, int64_t *n_frags) {
    std::vector<bm2_dup_entry> p, f;
    for (int64_t t = 0; t < n_tmpl; ++t) template_entries(recs, starts, tmpl_first[t], tmpl_first[t + 1], tmpl_id[t], p, f);
    std::copy(p.begin(), p.end(), pairs_out); *n_pairs = (int64_t) p.size();
    std::copy(f.begin(), f.end(), frags_out); *n_frags = (int64_t) f.size();
}

// bm2_dup_resolve restated: sorted_out (n entries) when !res, else dups_out (room for n ids) and *n_dups
extern "C" void markdup_emul_resolve(const bm2_dup_entry *e, int64_t n, int res, bm2_dup_entry *sorted_out, int64_t *dups_out, int64_t *n_dups) {
    std::vector<bm2_dup_entry> s; std::vector<int64_t> d;
    resolve(e, n, res, s, d);
    if (!res) std::copy(s.begin(), s.end(), sorted_out);
    else { std::copy(d.begin(), d.end(), dups_out); *n_dups = (int64_t) d.size(); }
}

// bm2_mem --markdup's sorted part: templates [tmpl_first[t], tmpl_first[t+1]) of the records (uncompressed BAM in output order) with their
// ids, added chunk_tmpl templates at a time (records, their ids, then the chunk's entries), sorted in runs of run_bytes with sig_bytes of
// entries, marked, merged and written to out_path.  stats: runs, merge windows, signature runs, signature bytes, templates with an entry,
// pair duplicates, fragment duplicates, records marked, spill bytes.  Returns 0, or 1 with the message in err.
extern "C" int markdup_emul_file(const uint8_t *recs, int64_t n, const int64_t *tmpl_first, const int64_t *tmpl_id, int64_t n_tmpl, int64_t chunk_tmpl,
                                 int64_t run_bytes, int64_t sig_bytes, int64_t n_reads, const char *tmp_prefix, int threads, const char *out_path,
                                 int64_t *stats, char *err, int err_cap) {
    try {
        EmulState S;
        BamSortSink sink;
        sink.sort_ex = [&S](const uint8_t *r, int64_t nb, const int64_t *st, int64_t nr, const int64_t *tids, const uint8_t *c, int64_t cl, int last,
                            bm2_sort_out *o, const int64_t **to, double *ds) {
            *ds = 0;
            return emul_sort_ex(S, r, nb, st, nr, tids, c, cl, last, o, to);
        };
        sink.dup = [&S](const bm2_dup_entry *e, int64_t ne, int res, const bm2_dup_entry **sorted, const int64_t **dups, int64_t *nd, double *ds) {
            *ds = 0;
            resolve(e, ne, res, S.sorted, S.dups);
            if (sorted) *sorted = S.sorted.data();
            if (res) { *dups = S.dups.data(); *nd = (int64_t) S.dups.size(); }
            return 0;
        };
        sink.dup_set = [&S](const uint64_t *b, int64_t nb) { S.bits.assign(b, b + (nb + 63) / 64); S.n_bits = nb; return 0; };
        sink.fail = [](const std::string &m) { throw std::runtime_error(m); };
        sink.run_bytes = run_bytes; sink.sig_bytes = sig_bytes; sink.n_reads = n_reads; sink.tmp_prefix = tmp_prefix; sink.threads = threads;
        std::vector<int64_t> st;
        for (int64_t q = 0; q + 4 <= n; q += 4 + (int64_t) bam_le32(recs + q)) st.push_back(q);
        for (int64_t t0 = 0; t0 < n_tmpl; t0 += chunk_tmpl) {
            const int64_t t1 = std::min(n_tmpl, t0 + chunk_tmpl), i0 = tmpl_first[t0], i1 = tmpl_first[t1];
            std::vector<int64_t> ids, first;
            for (int64_t t = t0; t < t1; ++t) { first.push_back(tmpl_first[t] - i0); for (int64_t i = tmpl_first[t]; i < tmpl_first[t + 1]; ++i) ids.push_back(tmpl_id[t]); }
            first.push_back(i1 - i0);
            const int64_t b0 = i0 < (int64_t) st.size() ? st[(size_t) i0] : n, b1 = i1 < (int64_t) st.size() ? st[(size_t) i1] : n;
            sink.add(recs + b0, b1 - b0, ids.data());
            std::vector<bm2_dup_entry> p, f;
            for (int64_t t = t0; t < t1; ++t) template_entries(recs, st.data(), tmpl_first[t], tmpl_first[t + 1], tmpl_id[t], p, f);
            sink.add_sigs(p.data(), (int64_t) p.size(), f.data(), (int64_t) f.size());
        }
        FILE *out = fopen(out_path, "wb");
        if (!out) throw std::runtime_error("cannot open the output");
        sink.finish(out, 0, nullptr);
        fclose(out);
        const int64_t v[] = { (int64_t) sink.runs.size(), sink.merge_windows, sink.dup_sig_runs, sink.dup_sig_bytes, sink.dup_templates,
                              sink.dup_pair_templates, sink.dup_frag_templates, sink.dup_records, sink.spill_bytes };
        std::copy(v, v + 9, stats);
        return 0;
    } catch (const std::exception &e) {
        snprintf(err, (size_t) err_cap, "%s", e.what());
        return 1;
    }
}

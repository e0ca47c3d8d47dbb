// bamsort_emul.cpp — TEST ONLY: bm2_sort on the CPU, in both orders.  bam_sort.h (runs, temporary files, merge windows, BAI) runs unchanged,
// with the device call restated: bm2_bam_sort_compress as std::stable_sort by the coordinate key, bm2_bam_qname_sort_compress
// (bwa-mem2_b200/csrc/bam_sort.cu) as std::stable_sort with bam_qname_cmp, and for -n the sink merging with bam_qname_rec_cmp, as the tool
// does.  The blocks are laid out by bam_sort_layout and compressed by bgzf_emul.cpp's restatement of the BGZF kernel.  The GPU must give
// these bytes exactly.
#include "bam_sort.h"
#include <stdexcept>

extern "C" int bgzf_emul_block(const uint8_t *d, int n, uint8_t *o);

namespace {

struct EmulState { std::vector<uint8_t> z, carry; std::vector<int32_t> sizes; std::vector<bm2_sort_rec> recs; };

int emul_sort(EmulState &S, bool by_name, const uint8_t *recs, const int64_t *starts, int64_t n_recs, const uint8_t *carry, int64_t carry_len,
              int last, bm2_sort_out *out) {
    std::vector<int64_t> len((size_t) n_recs), ord((size_t) n_recs);
    for (int64_t i = 0; i < n_recs; ++i) { len[(size_t) i] = 4 + (int64_t) bam_le32(recs + starts[i]); ord[(size_t) i] = i; }
    std::stable_sort(ord.begin(), ord.end(), [&](int64_t a, int64_t b) {
        const uint8_t *x = recs + starts[a], *y = recs + starts[b];
        if (by_name) return bam_qname_cmp(x + 36, bam_le16(x + 18), a, y + 36, bam_le16(y + 18), b) < 0;
        const BamFixed f = bam_fixed(x), g = bam_fixed(y);
        return bam_coord_key(f.rid, f.pos, f.flag) < bam_coord_key(g.rid, g.pos, g.flag);
    });
    std::vector<int64_t> offs((size_t) n_recs + 1, 0);
    std::vector<uint8_t> stream(carry, carry + carry_len);
    S.recs.resize((size_t) n_recs);
    for (int64_t i = 0; i < n_recs; ++i) {
        const int64_t k = ord[(size_t) i];
        offs[(size_t) i + 1] = offs[(size_t) i] + len[(size_t) k];
        stream.insert(stream.end(), recs + starts[k], recs + starts[k] + len[(size_t) k]);
        S.recs[(size_t) i] = bam_sort_rec(recs + starts[k]);
    }
    std::vector<int64_t> cut;
    SortLayout L;
    bam_sort_layout(carry_len, offs.data(), n_recs, offs[(size_t) n_recs], last != 0, cut, L, S.recs.data());
    S.z.clear(); S.sizes.clear();
    std::vector<uint8_t> m(BGZF_MAX_MEMBER);
    for (int64_t b = 0; b < L.n_full; ++b) {
        const int k = bgzf_emul_block(stream.data() + L.starts[(size_t) b], (int) (L.starts[(size_t) b + 1] - L.starts[(size_t) b]), m.data());
        if (k <= 0) return 2;
        S.z.insert(S.z.end(), m.begin(), m.begin() + k); S.sizes.push_back(k);
    }
    S.carry.assign(stream.begin() + L.starts[(size_t) L.n_full], stream.end());
    out->z = S.z.data(); out->z_len = (int64_t) S.z.size();
    out->member_size = S.sizes.data(); out->n_members = L.n_full;
    out->carry = S.carry.data(); out->carry_len = (int64_t) S.carry.size();
    out->recs = S.recs.data(); out->n_recs = n_recs;
    return 0;
}

}  // namespace

// bam_qname_cmp of n pairs of names (flag bits and ordinals equal): names holds NUL-terminated names at offs[k]; pairs[2i], pairs[2i+1] index
// them; out[i] gets -1, 0 or 1
extern "C" void bamsort_emul_cmp(const uint8_t *names, const int64_t *offs, const int64_t *pairs, int64_t n, int32_t *out) {
    for (int64_t i = 0; i < n; ++i) out[i] = bam_qname_cmp(names + offs[pairs[2 * i]], 0, 0, names + offs[pairs[2 * i + 1]], 0, 0);
}

// one device call (by_name: bm2_bam_qname_sort_compress, else bm2_bam_sort_compress): z (cap bytes), carry (room for 65280), recs (n_recs);
// sizes[0] = z bytes, sizes[1] = carry bytes, sizes[2] = members.  Returns 0, or -1 when z does not fit.
extern "C" int bamsort_emul_once(int by_name, const uint8_t *recs, const int64_t *starts, int64_t n_recs, const uint8_t *carry, int64_t carry_len,
                                 int last, uint8_t *z, int64_t cap, uint8_t *carry_out, bm2_sort_rec *recs_out, int64_t *sizes) {
    EmulState S; bm2_sort_out o;
    if (emul_sort(S, by_name != 0, recs, starts, n_recs, carry, carry_len, last, &o)) return -2;
    if (o.z_len > cap) return -1;
    memcpy(z, o.z, (size_t) o.z_len); memcpy(carry_out, o.carry, (size_t) o.carry_len);
    memcpy(recs_out, o.recs, (size_t) n_recs * sizeof(bm2_sort_rec));
    sizes[0] = o.z_len; sizes[1] = o.carry_len; sizes[2] = o.n_members;
    return 0;
}

// bm2_sort's record part: the records (uncompressed BAM) added chunk by chunk (chunk: bytes per add, at record boundaries; 0 = all at once),
// sorted in runs of run_bytes, merged, and written to out_path as the members that follow out_off compressed bytes of header; the index to
// bai_path unless null.  stats: runs, spill bytes, merge windows.  Returns 0, or 1 with the message in err.
extern "C" int bamsort_emul_file(int by_name, const uint8_t *recs, int64_t n, int64_t chunk, int64_t run_bytes, const char *tmp_prefix, int threads,
                                 uint64_t out_off, int n_ref, const char *out_path, const char *bai_path, int64_t *stats, char *err, int err_cap) {
    try {
        EmulState S;
        BamSortSink sink;
        sink.sort = [&S, by_name](const uint8_t *r, int64_t, const int64_t *st, int64_t nr, const uint8_t *c, int64_t cl, int last, bm2_sort_out *o,
                                  double *device_s) {
            *device_s = 0;
            return emul_sort(S, by_name != 0, r, st, nr, c, cl, last, o);
        };
        if (by_name) sink.cmp = bam_qname_rec_cmp;
        sink.fail = [](const std::string &m) { throw std::runtime_error(m); };
        sink.run_bytes = run_bytes; sink.tmp_prefix = tmp_prefix; sink.threads = threads;
        std::vector<int64_t> st;
        for (int64_t q = 0; q + 4 <= n; q += 4 + (int64_t) bam_le32(recs + q)) st.push_back(q);
        int64_t from = 0;
        for (size_t i = 0; i <= st.size(); ++i) {
            const int64_t at = i < st.size() ? st[i] : n;
            if (at > from && (i == st.size() || (chunk > 0 && at - from >= chunk))) { sink.add(recs + from, at - from); from = at; }
        }
        FILE *out = fopen(out_path, "wb");
        if (!out) throw std::runtime_error("cannot open the output");
        BaiBuilder bai(n_ref);
        sink.finish(out, out_off, bai_path ? &bai : nullptr);
        fclose(out);
        if (bai_path) {
            FILE *f = fopen(bai_path, "wb");
            const std::string b = bai.bytes();
            if (!f || fwrite(b.data(), 1, b.size(), f) != b.size()) throw std::runtime_error("cannot write the index");
            fclose(f);
        }
        stats[0] = (int64_t) sink.runs.size(); stats[1] = sink.spill_bytes; stats[2] = sink.merge_windows;
        return 0;
    } catch (const std::exception &e) {
        snprintf(err, (size_t) err_cap, "%s", e.what());
        return 1;
    }
}

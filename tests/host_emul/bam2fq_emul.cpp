// bam2fq_emul.cpp — TEST ONLY: bm2_bam2fq on the CPU.  bam2fq.h drives it unchanged; the record kernel and the format kernel are restated
// one record at a time over bam2fq_device.cuh's helpers (a warp's vote as a loop over the 32 lanes, its writes as one lane of one),
// bm2_markdup_pair as markdup_bam_emul.cpp's restatement, and the compression as bgzf_emul.cpp's.  The GPU must give these bytes exactly.
#include "bam2fq.h"
#include "bam2fq_device.cuh"
#include "markdup_device.cuh"
#include <stdexcept>

extern "C" int64_t bgzf_emul(const uint8_t *in, int64_t n, const int64_t *cut, int64_t n_cut, uint8_t *out, int64_t cap);
extern "C" void mdb_emul_pair(const bm2_markdup_half *h, int64_t n, const uint8_t *names, int32_t *partner);

namespace {

// b2f_record_kernel, one record; *err gets the record's error (0: none)
bm2_bam2fq_rec record(const uint8_t *r, int suffixes, int *err) {
    const B2fView v = b2f_view(r, suffixes);
    bm2_bam2fq_rec o{};
    o.kind = b2f_kind(v.flag);
    *err = B2F_ERR_NONE;
    if (o.kind != B2F_SKIP) {
        if (v.l_seq == 0) *err = B2F_ERR_EMPTY;
        else for (int lane = 0; lane < 32; ++lane) if (b2f_check_part(v, lane, 32) != B2F_ERR_NONE) *err = B2F_ERR_QUAL;
        o.text_len = b2f_text_len(v);
        if (o.kind != B2F_OTHER) o.hash = dup_name_hash(v.name, v.name_len);
    }
    return o;
}

const uint8_t *pick(int64_t ref, const uint8_t *win, const int64_t *wst, const uint8_t *x, const int64_t *xs) {
    return ref >= 0 ? win + wst[ref] : x + xs[~ref];
}

// b2f_len_kernel, the scan and b2f_format_kernel: the text of the listed records appended to out
void text(const int64_t *list, int64_t n, const uint8_t *win, const int64_t *wst, const uint8_t *x, const int64_t *xs, int suffixes, std::string &out) {
    for (int64_t i = 0; i < n; ++i) {
        const B2fView v = b2f_view(pick(list[i], win, wst, x, xs), suffixes);
        const size_t at = out.size();
        out.resize(at + (size_t) b2f_text_len(v));
        b2f_write_part(v, (uint8_t *) &out[at], 0, 1);
    }
}

std::string compress(const std::string &in) {
    std::vector<uint8_t> b(in.size() + 64 * (in.size() / 65280 + 2));
    const int64_t k = bgzf_emul((const uint8_t *) in.data(), (int64_t) in.size(), nullptr, 0, b.data(), (int64_t) b.size());
    if (k < 0) throw std::runtime_error("bgzf_emul");
    return std::string((const char *) b.data(), (size_t) k);
}

}  // namespace

// the record kernel over one window: out gets n_recs records; returns the first error as index << 4 | kind, or -1
extern "C" int64_t b2f_emul_records(const uint8_t *recs, const int64_t *starts, int64_t n_recs, int suffixes, bm2_bam2fq_rec *out) {
    int64_t first = -1;
    for (int64_t i = 0; i < n_recs; ++i) {
        int e = 0;
        out[i] = record(recs + starts[i], suffixes, &e);
        if (e && first < 0) first = i << 4 | e;
    }
    return first;
}

// the text of the listed records (window records >= 0, extra records ~k): returns its length, written to out when it fits cap
extern "C" int64_t b2f_emul_text(const int64_t *list, int64_t n, const uint8_t *win, const int64_t *wst, const uint8_t *x, const int64_t *xs,
                                 int suffixes, uint8_t *out, int64_t cap) {
    std::string t;
    text(list, n, win, wst, x, xs, suffixes, t);
    if ((int64_t) t.size() <= cap) memcpy(out, t.data(), t.size());
    return (int64_t) t.size();
}

// bm2_bam2fq over in_path: paths '\n'-joined in the order -o / -1, -2, -0, -s (empty: not given); returns the exit code, with the message
// in err; stats: records, kept, pairs, others, singletons, others dropped, singletons dropped, pending_max, pending_bytes_max, windows
extern "C" int b2f_emul_run(const char *in_path, const char *paths, int split, int suffixes, int threads, int64_t window, int64_t *stats, char *err,
                            int err_cap) {
    struct Fail { int code; std::string m; };
    Bam2fq b;
    b.in_path = in_path; b.split = split != 0; b.suffixes = suffixes; b.threads = threads; b.window = window;
    std::string p = paths;
    for (size_t at = 0, k = 0; at <= p.size() && k < 4; ++k) {
        size_t e = p.find('\n', at); if (e == std::string::npos) e = p.size();
        b.path[k] = p.substr(at, e - at); at = e + 1;
    }
    b.fail = [](int code, const std::string &m) { throw Fail{code, m}; };
    std::vector<bm2_bam2fq_rec> rr;
    const uint8_t *win = nullptr;
    const int64_t *wst = nullptr;
    int64_t wn = 0;
    b.records = [&](const uint8_t *r, int64_t, const int64_t *st, int64_t nr) -> const bm2_bam2fq_rec * {
        rr.resize((size_t) nr + 1);
        const int64_t e = b2f_emul_records(r, st, nr, suffixes, rr.data());
        if (e >= 0) {
            const uint8_t *x = r + st[e >> 4];
            b.die(1, "bm2_bam2fq_records: read " + std::string((const char *) x + 36, x[12] ? x[12] - 1 : 0) + " (record " + std::to_string(e >> 4) +
                         " of the window) " + ((e & 15) == B2F_ERR_EMPTY ? "has no bases (l_seq 0)" : "has a quality above 93"));
        }
        win = r; wst = st; wn = nr;
        return rr.data();
    };
    std::vector<int32_t> part;
    b.pair = [&](const bm2_markdup_half *h, int64_t n, const uint8_t *names, int64_t) -> const int32_t * {
        part.resize((size_t) n + 1);
        mdb_emul_pair(h, n, names, part.data());
        return part.data();
    };
    std::string data, tail;
    b.format = [&](const int64_t *list, int64_t n, const uint8_t *x, int64_t, const int64_t *xs, int64_t, const uint8_t *c, int64_t cl, int gz,
                   int last, bm2_bam2fq_out *o) {
        for (int64_t i = 0; i < n; ++i) if (list[i] >= wn) b.die(3, "a listed record outside the window");
        std::string t((const char *) c, (size_t) cl);
        text(list, n, win, wst, x, xs, suffixes, t);
        o->text_len = (int64_t) t.size() - cl;
        if (!gz) data = t, tail.clear();
        else {
            const size_t cut = last ? t.size() : t.size() / 65280 * 65280;
            data = compress(t.substr(0, cut));
            tail = t.substr(cut);
        }
        o->data = (const uint8_t *) data.data(); o->len = (int64_t) data.size();
        o->tail = (const uint8_t *) tail.data(); o->tail_len = (int64_t) tail.size();
    };
    try {
        b.run();
    } catch (const Fail &f) {
        snprintf(err, (size_t) err_cap, "%s", f.m.c_str());
        return f.code;
    }
    const int64_t v[] = {b.n_records, b.kept, b.pairs, b.others, b.singletons, b.others_dropped, b.singletons_dropped, b.pending_max,
                         b.pending_bytes_max, b.n_windows};
    std::copy(v, v + 10, stats);
    snprintf(err, (size_t) err_cap, "%s", b.warning.c_str());
    return 0;
}

// bm2_markdup — Picard MarkDuplicates on the GPU over one or more coordinate-sorted BAM files (several lanes, read groups and libraries),
// written as one merged, coordinate-sorted BAM with the duplicate flags set, plus Picard's DuplicationMetrics file (C++, over the C ABI of
// include/bm2_b200.h only).
//
//   bm2_markdup [-t INT] [--window SIZE] [--sig-mem SIZE] [--optical-distance N] [--write-index] -M metrics.txt [-o out.bam] in1.bam [in2.bam ...]
//
//   The rule, the merge, the pairing and the files are markdup_bam.h's; the per-record kernel and the flag kernel are markdup_bam.cu's; the
//   entries are resolved by bm2_dup_resolve / bm2_dup_resolve_ex on a context of their own, so that the sinks' sorter threads never share
//   a context with the record windows.  The inputs are read twice, so they must be files.
// Exit codes: 0 success, 1 a usage, header or input error, 2 an output file that cannot be written, 3 a device error.
#include "bm2_b200.h"
#include "../csrc/markdup_bam.h"
#include <chrono>
#include <cstdlib>
#include <mutex>

namespace {

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

[[noreturn]] void fail(int code, const std::string &m) {
    fprintf(stderr, "[E::bm2_markdup] %s\n", m.c_str());
    fflush(stderr);
    _Exit(code);
}

void usage() {
    fprintf(stderr,
            "Usage: bm2_markdup [options] -M metrics.txt in1.bam [in2.bam ...]\n"
            "Marks duplicates in one or more coordinate-sorted BAM files on the GPU (Picard MarkDuplicates on coordinate-sorted input at its\n"
            "defaults: several read groups and libraries, the library in the duplicate key, optical duplicates within a read group) and writes\n"
            "one merged, coordinate-sorted BAM with only the 0x400 flags rewritten, and Picard's duplication metrics per library.\n"
            "  -M FILE                 the duplication metrics file (required)\n"
            "  -o FILE                 output file [standard output]\n"
            "  --write-index           also write FILE.bai (needs -o)\n"
            "  -t INT                  inflate threads [1]\n"
            "  --window SIZE           uncompressed bytes per input and window, suffix K, M or G [256M]\n"
            "  --sig-mem SIZE          host bytes of duplicate entries, shared by the libraries, before they spill to sorted runs [1G]\n"
            "  --optical-distance N    the largest pixel distance of two optical duplicates, 0 to 2147483647 [100]\n");
}

bool parse_size(const char *s, long long *v) {
    char *e;
    if (*s < '0' || *s > '9') return false;
    const unsigned long long x = strtoull(s, &e, 10);
    int shift = 0;
    if (*e == 'k' || *e == 'K') shift = 10, ++e;
    else if (*e == 'm' || *e == 'M') shift = 20, ++e;
    else if (*e == 'g' || *e == 'G') shift = 30, ++e;
    if (*e || x == 0 || x > (unsigned long long) (INT64_MAX >> shift)) return false;
    *v = (long long) (x << shift);
    return true;
}

}  // namespace

int main(int argc, char **argv) {
    const double t_start = now_s();
    MarkdupBam md;
    md.fail = fail;
    bool write_index = false;
    long long threads = 1, window = 256LL << 20, sig_mem = 1LL << 30, distance = 100;   // 256M and 1G: chosen figures, not measured ones
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) md.out_path = value("-o");
        else if (!strcmp(s, "-M")) md.metrics_path = value("-M");
        else if (!strcmp(s, "--write-index")) write_index = true;
        else if (!strcmp(s, "-t")) {
            char *e; threads = strtoll(value("-t"), &e, 10);
            if (*e || threads < 1 || threads > 1024) fail(1, "-t takes a number of threads from 1 to 1024");
        } else if (!strcmp(s, "--window")) {
            if (!parse_size(value("--window"), &window)) fail(1, "--window takes a size such as 64K, 256M or 1G");
        } else if (!strcmp(s, "--sig-mem")) {
            if (!parse_size(value("--sig-mem"), &sig_mem)) fail(1, "--sig-mem takes a size such as 64K, 256M or 1G");
        } else if (!strcmp(s, "--optical-distance")) {
            const char *v = value("--optical-distance");
            char *e; distance = strtoll(v, &e, 10);
            if (*v < '0' || *v > '9' || *e || distance < 0 || distance > INT32_MAX) fail(1, "--optical-distance takes a decimal integer from 0 to 2147483647");
        } else if (!strcmp(s, "-")) fail(1, "standard input cannot be an input: the inputs are read twice");
        else if (s[0] == '-' && s[1]) { usage(); fail(1, std::string("unknown option ") + s); }
        else md.paths.push_back(s);
    }
    if (md.paths.empty()) { usage(); fail(1, "no input BAM"); }
    if (md.metrics_path.empty()) { usage(); fail(1, "-M is required"); }
    if (write_index && md.out_path.empty()) fail(1, "--write-index needs -o");
    if (write_index) md.bai_path = md.out_path + ".bai";
    md.threads = (int) threads; md.window = window; md.sig_bytes = sig_mem; md.distance = distance;
    for (int i = 1; i < argc; ++i) md.args += std::string(i > 1 ? " " : "") + argv[i];
    md.cl = std::string(argv[0]) + (md.args.empty() ? "" : " " + md.args);

    // the devices: ctx takes the record windows, the bitset and the second pass; dctx the resolve, from any sink's thread
    bm2_mem_opt_t opt;
    bm2_opt_init(&opt);
    bm2_ctx *ctx = nullptr, *dctx = nullptr;
    if (bm2_create(&ctx, 0, nullptr, &opt) || bm2_create(&dctx, 0, nullptr, &opt)) { fprintf(stderr, "bm2_markdup: %s\n", bm2_last_error(nullptr)); return 3; }
    int64_t device_bytes = 0;
    {
        const int64_t merged = window * (int64_t) md.paths.size();   // a merged window holds at most one window of each input
        int64_t avail = 0;
        if (bm2_markdup_memory(ctx, merged, &device_bytes, &avail)) fail(3, std::string("bm2_markdup_memory: ") + bm2_last_error(ctx));
        if (device_bytes > avail)
            fail(1, "--window " + std::to_string(window) + " over " + std::to_string(md.paths.size()) + " inputs: one window needs " +
                        std::to_string(device_bytes) + " bytes of device memory, " + std::to_string(avail) + " bytes free");
    }
    std::vector<std::string> ids;
    std::vector<const char *> cids;
    md.set_header = [&](const MdbHeader &h) {
        ids = h.rg_ids;
        cids.clear();
        for (const std::string &s : ids) cids.push_back(s.c_str());
        if (bm2_markdup_set(ctx, (int32_t) ids.size(), cids.data(), h.rg_lib.data(), (int32_t) h.libs.size(), h.unknown_lib)) md.die(1, bm2_last_error(ctx));
        return 0;
    };
    md.records = [ctx, &md](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, const bm2_markdup_rec **out) {
        if (bm2_markdup_records(ctx, r, n, st, nr, out)) md.die(3, std::string("bm2_markdup_records: ") + bm2_last_error(ctx));
        return 0;
    };
    md.pair = [ctx, &md](const bm2_markdup_half *h, int64_t n, const uint8_t *names, int64_t nl, const int32_t **partner) {
        if (bm2_markdup_pair(ctx, h, n, names, nl, partner)) md.die(3, std::string("bm2_markdup_pair: ") + bm2_last_error(ctx));
        return 0;
    };
    md.counts = [ctx, &md](int64_t *c) {
        if (bm2_markdup_counts(ctx, c)) md.die(3, std::string("bm2_markdup_counts: ") + bm2_last_error(ctx));
        return 0;
    };
    // md.die removes the files being written.  The resolve: one call at a time on dctx, its results copied out for the calling thread
    // before the next call may start
    std::mutex dmu;
    md.dup = [&](const bm2_dup_entry *e, int64_t n, int resolve, const bm2_dup_entry **sorted, const int64_t **dups, int64_t *n_dups, double *ds) {
        thread_local std::vector<bm2_dup_entry> s; thread_local std::vector<int64_t> d;
        std::lock_guard<std::mutex> g(dmu);
        const bm2_dup_entry *so = nullptr; const int64_t *du = nullptr; int64_t nd = 0;
        if (bm2_dup_resolve(dctx, e, n, resolve, &so, &du, &nd)) md.die(3, std::string("bm2_dup_resolve: ") + bm2_last_error(dctx));
        if (resolve) { d.assign(du, du + nd); *dups = d.data(); *n_dups = nd; }
        else { s.assign(so, so + n); *sorted = s.data(); }
        double ms = 0; bm2_last_dup_stats(dctx, nullptr, &ms); *ds = ms / 1e3;
        return 0;
    };
    md.dup_ex = [&](const bm2_dup_loc_entry *e, int64_t n, int resolve, const bm2_dup_loc_entry **sorted, const int64_t **dups, int64_t *n_dups,
                    int64_t *n_opt, double *ds) {
        thread_local std::vector<bm2_dup_loc_entry> s; thread_local std::vector<int64_t> d;
        std::lock_guard<std::mutex> g(dmu);
        const bm2_dup_loc_entry *so = nullptr; const int64_t *du = nullptr; int64_t nd = 0;
        if (bm2_dup_resolve_ex(dctx, e, n, resolve, distance, &so, &du, &nd, n_opt)) md.die(3, std::string("bm2_dup_resolve_ex: ") + bm2_last_error(dctx));
        if (resolve) { d.assign(du, du + nd); *dups = d.data(); *n_dups = nd; }
        else { s.assign(so, so + n); *sorted = s.data(); }
        double ms = 0; bm2_last_dup_stats(dctx, nullptr, &ms); *ds = ms / 1e3;
        return 0;
    };
    md.dup_upload = [ctx, &md](const uint64_t *bits, int64_t n_bits) {
        if (bm2_dup_set(ctx, bits, n_bits)) md.die(3, std::string("bm2_dup_set: ") + bm2_last_error(ctx));
        return 0;
    };
    md.mark = [ctx, &md](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, int64_t first, const uint8_t *c, int64_t cl, int last, bm2_sort_out *o) {
        if (bm2_markdup_mark(ctx, r, n, st, nr, first, c, cl, last, o)) md.die(3, std::string("bm2_markdup_mark: ") + bm2_last_error(ctx));
        return 0;
    };
    md.compress = [ctx, &md](const uint8_t *p, int64_t n, std::string *z) {
        const uint8_t *o = nullptr; int64_t ol = 0;
        if (bm2_bgzf_compress(ctx, p, n, nullptr, 0, &o, &ol)) md.die(3, std::string("bm2_bgzf_compress: ") + bm2_last_error(ctx));
        z->assign((const char *) o, (size_t) ol);
        return 0;
    };
    md.run();
    if (!md.warning.empty()) fprintf(stderr, "[W::bm2_markdup] %s", md.warning.c_str());
    bm2_markdup_stats_t s;
    if (bm2_last_markdup_stats(ctx, &s)) fail(3, "bm2_last_markdup_stats");
    fprintf(stderr, "{\"records\": %lld, \"inputs\": %lld, \"libraries\": %lld, \"read_groups\": %lld, \"pairs\": %lld, \"fragments\": %lld, "
                    "\"pending_max\": %lld, \"dup_pair_templates\": %lld, \"dup_fragment_templates\": %lld, \"dup_records\": %lld, "
                    "\"dup_optical_pairs\": %lld, \"dup_sig_runs\": %lld, \"dup_sig_bytes\": %lld, \"windows\": %lld, \"in_bytes\": %lld, "
                    "\"out_bytes\": %lld, \"inflate_s\": %.6f, \"sig_s\": %.6f, \"pair_s\": %.6f, \"resolve_s\": %.6f, \"mark_s\": %.6f, \"bgzf_s\": %.6f, "
                    "\"device_bytes\": %lld, \"wall_s\": %.6f}\n",
            (long long) md.n_records, (long long) md.paths.size(), (long long) md.n_libraries, (long long) md.hdr.rg_ids.size(), (long long) md.n_pairs,
            (long long) md.n_frags, (long long) md.pending_max, (long long) md.dup_pair_templates, (long long) md.dup_frag_templates,
            (long long) md.dup_records, (long long) md.dup_optical_pairs, (long long) md.dup_sig_runs, (long long) md.dup_sig_bytes,
            (long long) md.n_windows, (long long) md.in_bytes, (long long) md.out_bytes, md.inflate_s, s.records_ms / 1e3, s.pair_ms / 1e3, md.resolve_s, s.mark_ms / 1e3,
            s.bgzf_ms / 1e3, (long long) device_bytes, now_s() - t_start);
    bm2_destroy(dctx);
    bm2_destroy(ctx);
    return 0;
}

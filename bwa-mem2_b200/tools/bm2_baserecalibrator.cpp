// bm2_baserecalibrator — GATK BaseRecalibrator on the GPU: the recalibration table of one or more BAM files with several read groups, with
// the covariates counted on the GPU (C++, over the C ABI of include/bm2_b200.h only).
//
//   bm2_baserecalibrator [-t INT] [--window SIZE] --known-sites VCF [--known-sites VCF ...] -o table.txt <idxbase> <in.bam | -> [in.bam ...]
//
//   reference    <idxbase>.ann, .amb and .pac (mm_read_reference); the FM index is not loaded.  Each input's reference list must equal the
//                .ann contigs.
//   known sites  the VCFs (known_sites.h), read on a thread of their own while the headers are read, the device starts and the first window
//                inflates
//   read groups  the union of the inputs' @RG lines, each ID mapped to its covariate (bqsr_recal.h)
//   inputs       in any sort order, read one after the other (the counts are integer sums, so no merge is needed), each in windows of about
//                --window uncompressed bytes (bam_window.h): the members are inflated by zlib on -t threads, and the next window inflates on a
//                thread of its own while the GPU counts the current one
//   counting     bm2_recal_add (recal.cu, bqsr_device.cuh's rule) per window: bm2_mem --recal-file's rule with 0x400 read from the input,
//                each record into the tables of its read group's covariate
//   output       the report of every covariate (bqsr_report.h), in the byte order of the covariates, to <table>.tmp, renamed once complete
// Exit codes: 0 success, 1 a usage, reference, VCF, input or read error, 2 an output that cannot be written, 3 a device error.
#include "bm2_b200.h"
#include "../csrc/bam_window.h"
#include "../csrc/bqsr_recal.h"
#include "../csrc/known_sites.h"
#include "../csrc/mm_metrics.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <unistd.h>
#include <vector>

namespace {

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

std::string g_tmp;                                  // the table being written, removed on an error

// _Exit: the VCF and inflate threads may still be running
[[noreturn]] void fail(int code, const std::string &m) {
    fprintf(stderr, "[E::bm2_baserecalibrator] %s\n", m.c_str());
    fflush(stderr);
    if (!g_tmp.empty()) unlink(g_tmp.c_str());
    _Exit(code);
}

void usage() {
    fprintf(stderr,
            "Usage: bm2_baserecalibrator [options] --known-sites VCF -o table.txt <idxbase> <in.bam | -> [in.bam ...]\n"
            "Writes GATK BaseRecalibrator's recalibration table (GATK 4 at its defaults, substitution covariates only) of one or more BAM files\n"
            "in any order, with one row set per read group covariate (PU, else ID), counted on the GPU.  Reads only <idxbase>.ann, .amb and .pac.\n"
            "  -o FILE               the recalibration table (required)\n"
            "  --known-sites FILE    a VCF of known variants, plain, gzip or BGZF (required, may be repeated)\n"
            "  -t INT                inflate threads [1]\n"
            "  --window SIZE         uncompressed input bytes per window, suffix K, M or G [256M]\n");
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
    const char *out_path = nullptr, *prefix = nullptr;
    std::vector<std::string> in_paths, vcfs;
    long long threads = 1, window = 256LL << 20;        // 256M: a chosen figure, not a measured one
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) out_path = value("-o");
        else if (!strcmp(s, "--known-sites")) vcfs.push_back(value("--known-sites"));
        else if (!strcmp(s, "-t")) {
            char *e; threads = strtoll(value("-t"), &e, 10);
            if (*e || threads < 1 || threads > 1024) fail(1, "-t takes a number of threads from 1 to 1024");
        } else if (!strcmp(s, "--window")) {
            if (!parse_size(value("--window"), &window)) fail(1, "--window takes a size such as 64K, 256M or 1G");
        } else if (s[0] == '-' && s[1]) { usage(); fail(1, std::string("unknown option ") + s); }
        else if (!prefix) prefix = s;
        else in_paths.push_back(s);
    }
    if (!prefix) { usage(); fail(1, "no index prefix"); }
    if (in_paths.empty()) { usage(); fail(1, "no input BAM"); }
    if (!out_path || !*out_path) { usage(); fail(1, "no output table (-o)"); }
    if (vcfs.empty()) { usage(); fail(1, "at least one --known-sites is required"); }
    int n_stdin = 0;
    for (const std::string &p : in_paths) n_stdin += p == "-";
    if (n_stdin > 1) fail(1, "standard input (-) can be only one of the inputs");

    // the reference, then the VCFs on a thread of their own
    MmReference ref;
    std::string e = mm_read_reference(prefix, ref);
    if (!e.empty()) fail(1, e);
    KnownSites known;
    std::string e_known;
    double known_s = 0;
    std::thread known_thread([&] {
        const double t0 = now_s();
        e_known = read_known_sites(vcfs, ref.names, ref.off, std::vector<int64_t>(ref.len.begin(), ref.len.end()), ref.l_pac, known);
        known_s = now_s() - t0;
    });

    // the headers: read with a window of 0, so that no more than the header is inflated before the device is ready
    std::vector<std::unique_ptr<BamWindowReader>> rds;
    std::vector<std::string> texts, names;
    for (const std::string &p : in_paths) {
        rds.emplace_back(new BamWindowReader);
        BamWindowReader &rd = *rds.back();
        rd.name = p == "-" ? "standard input" : p;
        rd.f = p == "-" ? stdin : fopen(p.c_str(), "rb");
        if (!rd.f) fail(1, "cannot open " + p);
        rd.threads = (int) threads; rd.window = 0;
        std::string text;
        std::vector<std::pair<std::string, int32_t>> refs;
        e = rd.header(text, refs);
        if (!e.empty()) fail(1, e);
        e = wgs_check_refs(refs, ref);
        if (!e.empty()) fail(1, rd.where() + e);
        rd.window = window;
        texts.push_back(text); names.push_back(rd.name);
    }
    BqsrReadGroups groups;
    e = bqsr_read_groups(texts, names, groups);
    if (!e.empty()) fail(1, e);
    std::vector<uint8_t> blob;
    e = bqsr_rg_map(groups.ids, groups.id_cov, blob);
    if (!e.empty()) fail(1, e);

    // the windows of the inputs in turn; the first one inflates while the device starts and the VCFs are read
    size_t cur_in = 0;
    auto next_window = [&](std::vector<uint8_t> &buf, std::vector<int64_t> &st) -> std::string {
        for (; cur_in < rds.size(); ++cur_in) {
            const std::string err = rds[cur_in]->next(buf, st);
            if (!err.empty() || !st.empty()) return err;
        }
        return "";
    };
    std::vector<uint8_t> buf[2];
    std::vector<int64_t> starts[2];
    std::string e_first;
    std::thread first([&] { e_first = next_window(buf[0], starts[0]); });

    // the device
    bm2_mem_opt_t opt;
    bm2_opt_init(&opt);
    bm2_ctx *ctx = nullptr;
    if (bm2_create(&ctx, 0, nullptr, &opt)) fail(3, bm2_last_error(nullptr));
    auto die = [&](const char *what) { fail(3, std::string(what) + ": " + bm2_last_error(ctx)); };
    int64_t need = 0, avail = 0;
    if (bm2_recal_memory(ctx, ref.l_pac, window, (int32_t) groups.covs.size(), &need, &avail)) die("bm2_recal_memory");
    known_thread.join();
    first.join();
    if (!e_known.empty()) fail(1, e_known);
    if (need > avail)
        fail(1, "a reference of " + std::to_string(ref.l_pac) + " bases with --window " + std::to_string(window) + " and " +
                    std::to_string(groups.covs.size()) + " read groups needs " + std::to_string(need) + " bytes of device memory, " +
                    std::to_string(avail) + " bytes free");
    std::vector<const char *> cids;
    for (const std::string &s : groups.ids) cids.push_back(s.c_str());
    bm2_recal_set_t rs;
    rs.n_contigs = (int32_t) ref.names.size(); rs.contig_off = ref.off.data(); rs.contig_len = ref.len.data();
    rs.l_pac = ref.l_pac; rs.pac = ref.pac.data(); rs.holes = ref.holes.data(); rs.n_holes = (int64_t) ref.hole_char.size();   // every .amb hole reads as N
    rs.covered = known.covered.data(); rs.junction = known.junction.data();
    rs.n_ids = (int32_t) cids.size(); rs.ids = cids.data(); rs.id_cov = groups.id_cov.data(); rs.n_cov = (int32_t) groups.covs.size();
    if (bm2_recal_set(ctx, &rs)) die("bm2_recal_set");
    g_tmp = std::string(out_path) + ".tmp";                  // opened before the inputs are counted, so that an unwritable output fails early
    FILE *out = fopen(g_tmp.c_str(), "wb");
    if (!out) { g_tmp.clear(); fail(2, "cannot open " + std::string(out_path) + ".tmp"); }
    if (!e_first.empty()) fail(1, e_first);

    // the windows: the next one inflates while the device counts the current one
    int64_t n_windows = 0, n_records = 0;
    for (int c = 0; !starts[c].empty(); c ^= 1) {
        std::string e_next;
        std::thread next([&] { e_next = next_window(buf[c ^ 1], starts[c ^ 1]); });
        const int rc = bm2_recal_add(ctx, buf[c].data(), (int64_t) buf[c].size(), starts[c].data(), (int64_t) starts[c].size());
        if (rc) { next.join(); fail(rc == 2 ? 1 : 3, bm2_last_error(ctx)); }
        n_records += (int64_t) starts[c].size(); ++n_windows;
        next.join();
        if (!e_next.empty()) fail(1, e_next);
    }
    int64_t in_bytes = 0;
    double inflate_s = 0;
    for (auto &rd : rds) {
        if (!rd->warning.empty()) fprintf(stderr, "[W::bm2_baserecalibrator] %s\n", rd->warning.c_str());
        if (rd->f != stdin) fclose(rd->f);
        in_bytes += rd->in_bytes; inflate_s += rd->inflate_s;
    }

    // the report
    std::vector<std::vector<int64_t>> keep(groups.covs.size());
    std::vector<BqsrCovTables> covs;
    int64_t reads = 0, bases = 0;
    double recal_ms = 0;
    for (size_t c = 0; c < groups.covs.size(); ++c) {
        bm2_bqsr_tables_t t;
        if (bm2_recal_tables(ctx, (int32_t) c, &t)) die("bm2_recal_tables");
        std::vector<int64_t> &k = keep[c];
        for (const auto &a : {std::make_pair(t.qual_obs, BQSR_NQ), std::make_pair(t.qual_err, BQSR_NQ), std::make_pair(t.ctx_obs, BQSR_NQ * BQSR_NCTX),
                              std::make_pair(t.ctx_err, BQSR_NQ * BQSR_NCTX), std::make_pair(t.cyc_obs, BQSR_NQ * BQSR_NCYC),
                              std::make_pair(t.cyc_err, BQSR_NQ * BQSR_NCYC)})
            k.insert(k.end(), a.first, a.first + a.second);
        reads += t.reads; bases += t.bases; recal_ms = t.ms;
    }
    for (size_t c = 0; c < groups.covs.size(); ++c) {
        const int64_t *p = keep[c].data();
        covs.push_back({groups.covs[c], p, p + BQSR_NQ, p + 2 * BQSR_NQ, p + 2 * BQSR_NQ + BQSR_NQ * BQSR_NCTX, p + 2 * BQSR_NQ + 2 * BQSR_NQ * BQSR_NCTX,
                        p + 2 * BQSR_NQ + 2 * BQSR_NQ * BQSR_NCTX + BQSR_NQ * BQSR_NCYC});
    }
    const std::string text = bqsr_report_text(covs);
    if (fwrite(text.data(), 1, text.size(), out) != text.size() || fclose(out)) fail(2, "cannot write " + g_tmp);
    if (rename(g_tmp.c_str(), out_path)) fail(2, std::string("cannot write ") + out_path);
    g_tmp.clear();
    fprintf(stderr, "{\"records\": %lld, \"counted_reads\": %lld, \"counted_bases\": %lld, \"read_groups\": %lld, \"known_sites\": %lld, "
                    "\"known_sites_s\": %.6f, \"windows\": %lld, \"in_bytes\": %lld, \"inflate_s\": %.6f, \"recal_s\": %.6f, \"wall_s\": %.6f}\n",
            (long long) n_records, (long long) reads, (long long) bases, (long long) groups.covs.size(), (long long) known.records, known_s,
            (long long) n_windows, (long long) in_bytes, inflate_s, recal_ms / 1e3, now_s() - t_start);
    bm2_destroy(ctx);
    return 0;
}

// bm2_wgsmetrics — Picard CollectWgsMetrics on the GPU: the coverage metrics of a coordinate-sorted BAM file, with per-base coverage counted
// on the GPU (C++, over the C ABI of include/bm2_b200.h only).
//
//   bm2_wgsmetrics [-t INT] [--window SIZE] [-o FILE] [--min-mapq INT] [--min-baseq INT] [--coverage-cap INT] [--count-unpaired] <idxbase> <in.bam | ->
//
//   reference  <idxbase>.ann (contigs) and <idxbase>.amb (the N / n / . holes are no-call) only (wgs_metrics.h); the index is not loaded.
//              The BAM's @HD must say SO:coordinate and its reference list must equal the .ann contigs.
//   input      read in windows of about --window uncompressed bytes (bam_window.h): the members are inflated by zlib on -t threads, and the
//              next window inflates on a thread of its own while the GPU counts the current one.  A record out of coordinate order is an error.
//   counting   bm2_wgs_add (wgs.cu, wgs_device.cuh's rule) per window, bm2_wgs_finish once: the depth histogram and the exclusions
//   output     Picard's WgsMetrics file (wgs_metrics.h) to -o (written to <out>.tmp and renamed once complete) or standard output
// Exit codes: 0 success, 1 a usage, reference, input or read error, 2 an output file that cannot be written, 3 a device error.
#include "bm2_b200.h"
#include "../csrc/bam_window.h"
#include "../csrc/wgs_metrics.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <unistd.h>
#include <vector>

namespace {

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

std::string g_tmp;                                  // the output being written, removed on an error

[[noreturn]] void fail(int code, const std::string &m) {
    fprintf(stderr, "[E::bm2_wgsmetrics] %s\n", m.c_str());
    fflush(stderr);
    if (!g_tmp.empty()) unlink(g_tmp.c_str());
    _Exit(code);
}

void usage() {
    fprintf(stderr,
            "Usage: bm2_wgsmetrics [options] <idxbase> <in.bam | ->\n"
            "Writes Picard CollectWgsMetrics's metrics (picard.analysis.WgsMetrics and the coverage histogram) of a coordinate-sorted BAM file,\n"
            "with per-base coverage counted on the GPU.  Reads only <idxbase>.ann and <idxbase>.amb of the bwa-mem2 index.\n"
            "  -o FILE               output file [standard output]\n"
            "  --min-mapq INT        MINIMUM_MAPPING_QUALITY, 0..255 [20]\n"
            "  --min-baseq INT       MINIMUM_BASE_QUALITY, 0..93 [20]\n"
            "  --coverage-cap INT    COVERAGE_CAP, 1..10000 [250]\n"
            "  --count-unpaired      COUNT_UNPAIRED=true: count reads without a mapped mate\n"
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

int int_in(const char *opt, const char *s, long long lo, long long hi) {
    char *e;
    const long long v = strtoll(s, &e, 10);
    if (!*s || *e || v < lo || v > hi) fail(1, std::string(opt) + " takes a whole number from " + std::to_string(lo) + " to " + std::to_string(hi));
    return (int) v;
}

}  // namespace

int main(int argc, char **argv) {
    const double t_start = now_s();
    const char *out_path = nullptr, *prefix = nullptr, *in_path = nullptr;
    long long threads = 1, window = 256LL << 20;        // 256M: a chosen figure, not a measured one
    bm2_wgs_params_t prm{20, 20, 250, 0};
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) out_path = value("-o");
        else if (!strcmp(s, "--min-mapq")) prm.min_mapq = int_in("--min-mapq", value("--min-mapq"), 0, 255);
        else if (!strcmp(s, "--min-baseq")) prm.min_baseq = int_in("--min-baseq", value("--min-baseq"), 0, 93);
        else if (!strcmp(s, "--coverage-cap")) prm.coverage_cap = int_in("--coverage-cap", value("--coverage-cap"), 1, BM2_WGS_MAX_CAP);
        else if (!strcmp(s, "--count-unpaired")) prm.count_unpaired = 1;
        else if (!strcmp(s, "-t")) threads = int_in("-t", value("-t"), 1, 1024);
        else if (!strcmp(s, "--window")) {
            if (!parse_size(value("--window"), &window)) fail(1, "--window takes a size such as 64K, 256M or 1G");
        } else if (s[0] == '-' && s[1]) { usage(); fail(1, std::string("unknown option ") + s); }
        else if (!prefix) prefix = s;
        else if (!in_path) in_path = s;
        else { usage(); fail(1, "more than one input"); }
    }
    if (!prefix) { usage(); fail(1, "no index prefix"); }
    if (!in_path) { usage(); fail(1, "no input BAM"); }

    // the reference and the header
    WgsReference ref;
    std::string e = wgs_read_reference(prefix, ref);
    if (!e.empty()) fail(1, e);
    BamWindowReader rd;
    rd.name = strcmp(in_path, "-") ? in_path : "standard input";
    rd.f = strcmp(in_path, "-") ? fopen(in_path, "rb") : stdin;
    if (!rd.f) fail(1, std::string("cannot open ") + in_path);
    rd.threads = (int) threads; rd.window = window;
    std::string text;
    std::vector<std::pair<std::string, int32_t>> refs;
    e = rd.header(text, refs);
    if (!e.empty()) fail(1, e);
    e = wgs_check_header(text, refs, ref);
    if (!e.empty()) fail(1, rd.where() + e);

    // the device
    bm2_mem_opt_t opt;
    bm2_opt_init(&opt);
    bm2_ctx *ctx = nullptr;
    if (bm2_create(&ctx, 0, nullptr, &opt)) { fprintf(stderr, "[E::bm2_wgsmetrics] %s\n", bm2_last_error(nullptr)); return 3; }
    auto die = [&](const char *what) { fail(3, std::string(what) + ": " + bm2_last_error(ctx)); };
    int64_t need = 0, avail = 0;
    if (bm2_wgs_memory(ctx, ref.l_pac, window, &need, &avail)) die("bm2_wgs_memory");
    if (need > avail)
        fail(1, "a reference of " + std::to_string(ref.l_pac) + " bases with --window " + std::to_string(window) + " needs " + std::to_string(need) +
                    " bytes of device memory, " + std::to_string(avail) + " bytes free");
    if (bm2_wgs_set(ctx, ref.off.data(), ref.len.data(), (int32_t) ref.names.size(), ref.l_pac, ref.nocall.data(), (int64_t) ref.nocall.size() / 2, &prm))
        die("bm2_wgs_set");
    if (out_path) {                                     // opened before the input is read, so that an unwritable output fails early
        g_tmp = std::string(out_path) + ".tmp";
        FILE *t = fopen(g_tmp.c_str(), "wb");
        if (!t) { g_tmp.clear(); fail(2, std::string("cannot open ") + out_path + ".tmp"); }
        fclose(t);
    }

    // the windows: the next one inflates while the device takes the current one
    std::vector<uint8_t> buf[2];
    std::vector<int64_t> starts[2];
    e = rd.next(buf[0], starts[0]);
    if (!e.empty()) fail(1, e);
    int64_t n_windows = 0, n_records = 0;
    WgsOrder order;
    for (int cur = 0; !starts[cur].empty(); cur ^= 1) {
        std::string e_next;
        std::thread next([&] { e_next = rd.next(buf[cur ^ 1], starts[cur ^ 1]); });
        const std::vector<uint8_t> &B = buf[cur];
        const std::vector<int64_t> &S = starts[cur];
        for (size_t i = 0; i < S.size(); ++i) {
            const std::string oe = order.check(B.data() + S[i]);
            if (!oe.empty()) { next.join(); fail(1, rd.where() + oe); }
        }
        const int rc = bm2_wgs_add(ctx, B.data(), (int64_t) B.size(), S.data(), (int64_t) S.size());
        if (rc) { next.join(); fail(rc == 2 ? 1 : 3, bm2_last_error(ctx)); }
        n_records += (int64_t) S.size(); ++n_windows;
        next.join();
        if (!e_next.empty()) fail(1, e_next);
    }
    if (!rd.warning.empty()) fprintf(stderr, "[W::bm2_wgsmetrics] %s\n", rd.warning.c_str());
    if (rd.f != stdin) fclose(rd.f);
    bm2_wgs_result_t res;
    if (bm2_wgs_finish(ctx, &res)) die("bm2_wgs_finish");
    WgsCounts x;
    x.hist.assign(res.hist, res.hist + res.cap + 1);
    for (int k = 0; k < WGS_NEXC; ++k) x.exc[k] = res.exc[k];
    std::string args;
    for (int i = 1; i < argc; ++i) args += (i > 1 ? " " : "") + std::string(argv[i]);
    const std::string o = wgs_metrics_text(x, args);
    if (out_path) {
        FILE *f = fopen(g_tmp.c_str(), "wb");
        if (!f || fwrite(o.data(), 1, o.size(), f) != o.size() || fclose(f)) fail(2, "cannot write " + g_tmp);
        if (rename(g_tmp.c_str(), out_path)) fail(2, std::string("cannot write ") + out_path);
        g_tmp.clear();
    } else if (fwrite(o.data(), 1, o.size(), stdout) != o.size() || fflush(stdout)) fail(2, "cannot write the output");
    fprintf(stderr, "{\"records\": %lld, \"counted_records\": %lld, \"windows\": %lld, \"in_bytes\": %lld, \"inflate_s\": %.6f, \"add_s\": %.6f, "
                    "\"finish_s\": %.6f, \"carried_max\": %lld, \"device_bytes\": %lld, \"wall_s\": %.6f}\n",
            (long long) n_records, (long long) res.counted_records, (long long) n_windows, (long long) rd.in_bytes, rd.inflate_s, res.add_ms / 1e3,
            res.finish_ms / 1e3, (long long) res.carried_max, (long long) need, now_s() - t_start);
    bm2_destroy(ctx);
    return 0;
}

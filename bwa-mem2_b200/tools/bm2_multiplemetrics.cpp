// bm2_multiplemetrics — Picard CollectMultipleMetrics's alignment summary and insert size programs on the GPU: the two metrics files of a
// BAM file in any order, with the per-base mismatch count on the GPU (C++, over the C ABI of include/bm2_b200.h only).
//
//   bm2_multiplemetrics [-t INT] [--window SIZE] -o PREFIX <idxbase> <in.bam | ->
//
//   reference  <idxbase>.ann (contigs), .amb (holes and their letters) and .pac (packed bases) (mm_metrics.h); the FM index is not loaded.
//              The BAM's reference list must equal the .ann contigs; its sort order is not checked.
//   input      read in windows of about --window uncompressed bytes (bam_window.h): the members are inflated by zlib on -t threads, and the
//              next window inflates on a thread of its own while the GPU counts the current one.
//   counting   bm2_mm_add (mm.cu, mm_device.cuh's rule) per window, bm2_mm_finish once
//   output     PREFIX.alignment_summary_metrics and PREFIX.insert_size_metrics (mm_metrics.h), each written to <name>.tmp and renamed once
//              complete
// Exit codes: 0 success, 1 a usage, reference, input or read error, 2 an output file that cannot be written, 3 a device error.
#include "bm2_b200.h"
#include "../csrc/bam_window.h"
#include "../csrc/mm_metrics.h"
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

std::vector<std::string> g_tmp;                     // the outputs being written, removed on an error

[[noreturn]] void fail(int code, const std::string &m) {
    fprintf(stderr, "[E::bm2_multiplemetrics] %s\n", m.c_str());
    fflush(stderr);
    for (const std::string &t : g_tmp) unlink(t.c_str());
    _Exit(code);
}

void usage() {
    fprintf(stderr,
            "Usage: bm2_multiplemetrics [options] -o PREFIX <idxbase> <in.bam | ->\n"
            "Writes Picard CollectMultipleMetrics's PREFIX.alignment_summary_metrics and PREFIX.insert_size_metrics of a BAM file in any order,\n"
            "with the per-base mismatch count on the GPU.  Reads only <idxbase>.ann, .amb and .pac of the bwa-mem2 index.\n"
            "  -o PREFIX             output prefix (required)\n"
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

void write_tmp(const std::string &tmp, const std::string &o) {
    FILE *f = fopen(tmp.c_str(), "wb");
    if (!f || fwrite(o.data(), 1, o.size(), f) != o.size() || fclose(f)) fail(2, "cannot write " + tmp);
}

}  // namespace

int main(int argc, char **argv) {
    const double t_start = now_s();
    const char *out_prefix = nullptr, *prefix = nullptr, *in_path = nullptr;
    long long threads = 1, window = 256LL << 20;        // 256M: a chosen figure, not a measured one
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) out_prefix = value("-o");
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
    if (!out_prefix || !*out_prefix) { usage(); fail(1, "no output prefix (-o)"); }
    const std::string out_as = std::string(out_prefix) + ".alignment_summary_metrics", out_is = std::string(out_prefix) + ".insert_size_metrics";

    // the reference and the header
    MmReference ref;
    std::string e = mm_read_reference(prefix, ref);
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
    e = wgs_check_refs(refs, ref);
    if (!e.empty()) fail(1, rd.where() + e);

    // the device
    bm2_mem_opt_t opt;
    bm2_opt_init(&opt);
    bm2_ctx *ctx = nullptr;
    if (bm2_create(&ctx, 0, nullptr, &opt)) { fprintf(stderr, "[E::bm2_multiplemetrics] %s\n", bm2_last_error(nullptr)); return 3; }
    auto die = [&](const char *what) { fail(3, std::string(what) + ": " + bm2_last_error(ctx)); };
    int64_t need = 0, avail = 0;
    if (bm2_mm_memory(ctx, ref.l_pac, window, &need, &avail)) die("bm2_mm_memory");
    if (need > avail)
        fail(1, "a reference of " + std::to_string(ref.l_pac) + " bases with --window " + std::to_string(window) + " needs " + std::to_string(need) +
                    " bytes of device memory, " + std::to_string(avail) + " bytes free");
    if (bm2_mm_set(ctx, ref.off.data(), ref.len.data(), (int32_t) ref.names.size(), ref.l_pac, ref.pac.data(), ref.holes.data(), ref.hole_char.data(),
                   (int64_t) ref.hole_char.size()))
        die("bm2_mm_set");
    for (const std::string &p : {out_as, out_is}) {     // opened before the input is read, so that an unwritable output fails early
        const std::string t = p + ".tmp";
        FILE *f = fopen(t.c_str(), "wb");
        if (!f) fail(2, "cannot open " + t);
        fclose(f);
        g_tmp.push_back(t);
    }

    // the windows: the next one inflates while the device takes the current one
    std::vector<uint8_t> buf[2];
    std::vector<int64_t> starts[2];
    e = rd.next(buf[0], starts[0]);
    if (!e.empty()) fail(1, e);
    int64_t n_windows = 0, n_records = 0;
    for (int cur = 0; !starts[cur].empty(); cur ^= 1) {
        std::string e_next;
        std::thread next([&] { e_next = rd.next(buf[cur ^ 1], starts[cur ^ 1]); });
        const std::vector<uint8_t> &B = buf[cur];
        const std::vector<int64_t> &S = starts[cur];
        const int rc = bm2_mm_add(ctx, B.data(), (int64_t) B.size(), S.data(), (int64_t) S.size());
        if (rc) { next.join(); fail(rc == 2 ? 1 : 3, bm2_last_error(ctx)); }
        n_records += (int64_t) S.size(); ++n_windows;
        next.join();
        if (!e_next.empty()) fail(1, e_next);
    }
    if (!rd.warning.empty()) fprintf(stderr, "[W::bm2_multiplemetrics] %s\n", rd.warning.c_str());
    if (rd.f != stdin) fclose(rd.f);
    bm2_mm_result_t res;
    if (bm2_mm_finish(ctx, &res)) die("bm2_mm_finish");
    const MmCounts x = mm_counts(res.counts, res.max_len, res.len_hist, res.mism_hist, res.nocall, res.max_insert, res.insert_hist, res.insert_big,
                                 res.n_big);
    std::string args;
    for (int i = 1; i < argc; ++i) args += (i > 1 ? " " : "") + std::string(argv[i]);
    int64_t pairs = 0;
    const std::string as = mm_summary_text(x, args), is = mm_insert_text(x, args, &pairs);
    if (!pairs) fprintf(stderr, "[W::bm2_multiplemetrics] no read pair entered the insert sizes: %s has no rows and no histogram\n", out_is.c_str());
    write_tmp(g_tmp[0], as);
    write_tmp(g_tmp[1], is);
    if (rename(g_tmp[0].c_str(), out_as.c_str())) fail(2, "cannot write " + out_as);
    if (rename(g_tmp[1].c_str(), out_is.c_str())) { unlink(out_as.c_str()); fail(2, "cannot write " + out_is); }
    g_tmp.clear();
    int64_t counted = 0;
    for (int c = 0; c < MM_NCAT; ++c) counted += x.c[c][MM_TOTAL];
    fprintf(stderr, "{\"records\": %lld, \"counted_records\": %lld, \"aligned_bases\": %lld, \"pairs\": %lld, \"windows\": %lld, \"in_bytes\": %lld, "
                    "\"inflate_s\": %.6f, \"add_s\": %.6f, \"finish_s\": %.6f, \"device_bytes\": %lld, \"wall_s\": %.6f}\n",
            (long long) n_records, (long long) counted,
            (long long) (x.c[MM_FIRST][MM_ALIGNED_BASES] + x.c[MM_SECOND][MM_ALIGNED_BASES] + x.c[MM_UNPAIRED][MM_ALIGNED_BASES]), (long long) pairs,
            (long long) n_windows, (long long) rd.in_bytes, rd.inflate_s, res.add_ms / 1e3, res.finish_ms / 1e3, (long long) need, now_s() - t_start);
    bm2_destroy(ctx);
    return 0;
}

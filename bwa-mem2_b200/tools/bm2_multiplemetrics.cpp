// bm2_multiplemetrics — Picard CollectMultipleMetrics's alignment summary, insert size and GC bias programs on the GPU: their metrics files
// of a BAM file in any order, with the per-base mismatch count and the reference's GC windows on the GPU (C++, over the C ABI of
// include/bm2_b200.h only).
//
//   bm2_multiplemetrics [-t INT] [--window SIZE] [--program NAME ...] -o PREFIX <idxbase> <in.bam | ->
//
//   programs   Picard's PROGRAM: CollectAlignmentSummaryMetrics, CollectInsertSizeMetrics, CollectGcBiasMetrics, each --program adding one;
//              without --program the first two, as before (their files and the JSON line unchanged)
//
//   reference  <idxbase>.ann (contigs), .amb (holes and their letters) and .pac (packed bases) (mm_metrics.h); the FM index is not loaded.
//              The BAM's reference list must equal the .ann contigs; its sort order is not checked.
//   input      read in windows of about --window uncompressed bytes (bam_window.h): the members are inflated by zlib on -t threads, and the
//              next window inflates on a thread of its own while the GPU counts the current one.
//   counting   bm2_mm_add (mm.cu, mm_device.cuh's rule) per window, bm2_mm_finish once; with GC bias bm2_mm_gc_set (the reference scan)
//              before the first window and bm2_mm_gc_finish once
//   output     PREFIX.alignment_summary_metrics and PREFIX.insert_size_metrics (mm_metrics.h), PREFIX.gc_bias.detail_metrics and
//              PREFIX.gc_bias.summary_metrics (mm_gcbias.h), those of the programs run, each written to <name>.tmp and renamed once all are
//              complete
// Exit codes: 0 success, 1 a usage, reference, input or read error, 2 an output file that cannot be written, 3 a device error.  A --program
// name that is not one of the three (Picard's other programs included) is a usage error, found before anything is read.
#include "bm2_b200.h"
#include "../csrc/bam_window.h"
#include "../csrc/mm_gcbias.h"
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
            "Writes Picard CollectMultipleMetrics's metrics files of a BAM file in any order, with the per-base mismatch count and the\n"
            "reference's GC windows on the GPU.  Reads only <idxbase>.ann, .amb and .pac of the bwa-mem2 index.\n"
            "  -o PREFIX             output prefix (required)\n"
            "  -t INT                inflate threads [1]\n"
            "  --window SIZE         uncompressed input bytes per window, suffix K, M or G [256M]\n"
            "  --program NAME        a program to run, may be repeated; replaces the default list:\n"
            "                          CollectAlignmentSummaryMetrics  PREFIX.alignment_summary_metrics (default)\n"
            "                          CollectInsertSizeMetrics        PREFIX.insert_size_metrics (default)\n"
            "                          CollectGcBiasMetrics            PREFIX.gc_bias.detail_metrics and PREFIX.gc_bias.summary_metrics\n");
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
    static const char *const kPrograms[3] = {"CollectAlignmentSummaryMetrics", "CollectInsertSizeMetrics", "CollectGcBiasMetrics"};
    bool run[3] = {false, false, false}, named = false;
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) out_prefix = value("-o");
        else if (!strcmp(s, "-t")) threads = int_in("-t", value("-t"), 1, 1024);
        else if (!strcmp(s, "--window")) {
            if (!parse_size(value("--window"), &window)) fail(1, "--window takes a size such as 64K, 256M or 1G");
        } else if (!strcmp(s, "--program")) {
            const char *v = value("--program");
            int k = 0;
            while (k < 3 && strcmp(v, kPrograms[k])) ++k;
            if (k == 3)
                fail(1, std::string("--program ") + v + " is not a program of this tool; the programs are CollectAlignmentSummaryMetrics, "
                                                        "CollectInsertSizeMetrics and CollectGcBiasMetrics");
            run[k] = named = true;
        } else if (s[0] == '-' && s[1]) { usage(); fail(1, std::string("unknown option ") + s); }
        else if (!prefix) prefix = s;
        else if (!in_path) in_path = s;
        else { usage(); fail(1, "more than one input"); }
    }
    if (!prefix) { usage(); fail(1, "no index prefix"); }
    if (!in_path) { usage(); fail(1, "no input BAM"); }
    if (!out_prefix || !*out_prefix) { usage(); fail(1, "no output prefix (-o)"); }
    if (!named) run[0] = run[1] = true;
    const bool gc = run[2];
    // the outputs of the programs run, in this order: alignment summary, insert size, GC bias detail, GC bias summary
    const std::string pre(out_prefix);
    std::vector<std::string> outs;
    if (run[0]) outs.push_back(pre + ".alignment_summary_metrics");
    if (run[1]) outs.push_back(pre + ".insert_size_metrics");
    if (gc) { outs.push_back(pre + ".gc_bias.detail_metrics"); outs.push_back(pre + ".gc_bias.summary_metrics"); }

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
    int64_t need = 0, avail = 0, gc_need = 0;
    if (bm2_mm_memory(ctx, ref.l_pac, window, &need, &avail)) die("bm2_mm_memory");
    if (gc && bm2_mm_gc_memory(ctx, window, &gc_need)) die("bm2_mm_gc_memory");
    need += gc_need;
    if (need > avail)
        fail(1, "a reference of " + std::to_string(ref.l_pac) + " bases with --window " + std::to_string(window) + " needs " + std::to_string(need) +
                    " bytes of device memory, " + std::to_string(avail) + " bytes free");
    if (bm2_mm_set(ctx, ref.off.data(), ref.len.data(), (int32_t) ref.names.size(), ref.l_pac, ref.pac.data(), ref.holes.data(), ref.hole_char.data(),
                   (int64_t) ref.hole_char.size()))
        die("bm2_mm_set");
    if (gc && bm2_mm_gc_set(ctx)) die("bm2_mm_gc_set");
    for (const std::string &p : outs) {                 // opened before the input is read, so that an unwritable output fails early
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
    std::vector<std::string> texts;
    if (run[0]) texts.push_back(mm_summary_text(x, args));
    if (run[1]) {
        texts.push_back(mm_insert_text(x, args, &pairs));
        if (!pairs)
            fprintf(stderr, "[W::bm2_multiplemetrics] no read pair entered the insert sizes: %s has no rows and no histogram\n", (pre + ".insert_size_metrics").c_str());
    } else {
        mm_insert_text(x, args, &pairs);                 // the JSON line's pairs
    }
    bm2_mm_gc_result_t gr;
    MmGcCounts gx;
    if (gc) {
        if (bm2_mm_gc_finish(ctx, &gr)) die("bm2_mm_gc_finish");
        for (int k = 0; k < MM_GC_BINS; ++k) { gx.windows[k] = gr.windows[k]; gx.reads[k] = gr.reads[k]; gx.bases[k] = gr.bases[k]; gx.errors[k] = gr.errors[k]; }
        gx.clusters = gr.total_clusters; gx.aligned = gr.aligned_reads;
        texts.push_back(mm_gc_detail_text(gx, args));
        texts.push_back(mm_gc_summary_text(gx, args));
    }
    for (size_t k = 0; k < outs.size(); ++k) write_tmp(g_tmp[k], texts[k]);
    for (size_t k = 0; k < outs.size(); ++k)
        if (rename(g_tmp[k].c_str(), outs[k].c_str())) {
            for (size_t j = 0; j < k; ++j) unlink(outs[j].c_str());
            fail(2, "cannot write " + outs[k]);
        }
    g_tmp.clear();
    int64_t counted = 0;
    for (int c = 0; c < MM_NCAT; ++c) counted += x.c[c][MM_TOTAL];
    std::string gc_json;
    if (gc) {
        int64_t w = 0, r = 0;
        for (int k = 0; k < MM_GC_BINS; ++k) { w += gx.windows[k]; r += gx.reads[k]; }
        char b[256];
        snprintf(b, sizeof b, ", \"gc_windows\": %lld, \"gc_read_starts\": %lld, \"gc_scan_s\": %.6f, \"gc_add_s\": %.6f", (long long) w, (long long) r,
                 gr.scan_ms / 1e3, gr.add_ms / 1e3);
        gc_json = b;
    }
    fprintf(stderr, "{\"records\": %lld, \"counted_records\": %lld, \"aligned_bases\": %lld, \"pairs\": %lld, \"windows\": %lld, \"in_bytes\": %lld, "
                    "\"inflate_s\": %.6f, \"add_s\": %.6f, \"finish_s\": %.6f, \"device_bytes\": %lld%s, \"wall_s\": %.6f}\n",
            (long long) n_records, (long long) counted,
            (long long) (x.c[MM_FIRST][MM_ALIGNED_BASES] + x.c[MM_SECOND][MM_ALIGNED_BASES] + x.c[MM_UNPAIRED][MM_ALIGNED_BASES]), (long long) pairs,
            (long long) n_windows, (long long) rd.in_bytes, rd.inflate_s, res.add_ms / 1e3, res.finish_ms / 1e3, (long long) need, gc_json.c_str(),
            now_s() - t_start);
    bm2_destroy(ctx);
    return 0;
}

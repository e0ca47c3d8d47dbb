// bm2_bam2fq — the reads of a BAM file in any order back to FASTQ, mates paired, the FASTQ text written and compressed on the GPU (C++,
// over the C ABI of include/bm2_b200.h only).
//
//   bm2_bam2fq [-t INT] [--window SIZE] [-n | -N] (-1 R1 -2 R2 [-0 OTHER] [-s SINGLE] | [-o OUT]) <in.bam | ->
//
//   The rule is bam2fq_device.cuh's, the pairing order and the streams bam2fq.h's.  The input is read in windows of about --window
//   uncompressed bytes (bam_window.h), inflated on -t threads; the next window inflates while the GPU takes the current one.
// Exit codes: 0 success, 1 a usage, input or read error, 2 an output file that cannot be written, 3 a device error.
#include "bm2_b200.h"
#include "../csrc/bam2fq.h"
#include <chrono>
#include <cstdlib>
#include <cstring>

namespace {

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

[[noreturn]] void fail(int code, const std::string &m) {
    fprintf(stderr, "[E::bm2_bam2fq] %s\n", m.c_str());
    fflush(stderr);
    _Exit(code);
}

void usage() {
    fprintf(stderr,
            "Usage: bm2_bam2fq [options] (-1 R1 -2 R2 [-0 OTHER] [-s SINGLE] | [-o OUT]) <in.bam | ->\n"
            "Writes the reads of a BAM file in any order as FASTQ (FASTA for a read without qualities), mates paired wherever they lie, in the\n"
            "order of each pair's later record; reads without their mate come last.  A file name ending in .gz is written as BGZF, compressed on\n"
            "the GPU; any other name, and standard output, gets plain text.  Records with 0x100 or 0x800 are skipped.\n"
            "  -o FILE          the interleaved output [standard output]\n"
            "  -1 FILE, -2 FILE split output: READ1 (0x40) and READ2 (0x80) of each pair\n"
            "  -0 FILE          split output: records with both or neither of 0x40 and 0x80\n"
            "  -s FILE          split output: READ1 and READ2 records whose mate never comes\n"
            "  -N               add /1 and /2 to the names of READ1 and READ2 records [on when interleaved]\n"
            "  -n               do not add /1 and /2 [off when split]\n"
            "  -t INT           inflate threads [1]\n"
            "  --window SIZE    uncompressed input bytes per window, suffix K, M or G [256M]\n");
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
    Bam2fq b;
    b.fail = fail;
    const char *o = nullptr, *p1 = nullptr, *p2 = nullptr, *p0 = nullptr, *ps = nullptr, *in = nullptr;
    bool n_opt = false, N_opt = false;
    long long threads = 1, window = 256LL << 20;        // 256M: a chosen figure, not a measured one
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) o = value("-o");
        else if (!strcmp(s, "-1")) p1 = value("-1");
        else if (!strcmp(s, "-2")) p2 = value("-2");
        else if (!strcmp(s, "-0")) p0 = value("-0");
        else if (!strcmp(s, "-s")) ps = value("-s");
        else if (!strcmp(s, "-n")) n_opt = true;
        else if (!strcmp(s, "-N")) N_opt = true;
        else if (!strcmp(s, "-t")) {
            char *e; threads = strtoll(value("-t"), &e, 10);
            if (*e || threads < 1 || threads > 1024) fail(1, "-t takes a number of threads from 1 to 1024");
        } else if (!strcmp(s, "--window")) {
            if (!parse_size(value("--window"), &window)) fail(1, "--window takes a size such as 64K, 256M or 1G");
        } else if (s[0] == '-' && s[1]) { usage(); fail(1, std::string("unknown option ") + s); }
        else if (in) { usage(); fail(1, "more than one input"); }
        else in = s;
    }
    if (!in) { usage(); fail(1, "no input BAM"); }
    if (n_opt && N_opt) fail(1, "-n and -N cannot both be given");
    if (!p1 != !p2) fail(1, "-1 and -2 must be given together");
    b.split = p1 != nullptr;
    if (b.split && o) fail(1, "-o cannot be given with -1 and -2");
    if (!b.split && (p0 || ps)) fail(1, std::string(p0 ? "-0" : "-s") + " needs split output (-1 and -2)");
    if (b.split) { b.path[Bam2fq::S_MAIN] = p1; b.path[Bam2fq::S_R2] = p2; b.path[Bam2fq::S_OTHER] = p0 ? p0 : ""; b.path[Bam2fq::S_SINGLE] = ps ? ps : ""; }
    else b.path[Bam2fq::S_MAIN] = o ? o : "";
    b.suffixes = N_opt ? 1 : n_opt ? 0 : !b.split;
    b.in_path = in; b.threads = (int) threads; b.window = window;

    bm2_mem_opt_t opt;
    bm2_opt_init(&opt);
    bm2_ctx *ctx = nullptr;
    if (bm2_create(&ctx, 0, nullptr, &opt)) { fprintf(stderr, "bm2_bam2fq: %s\n", bm2_last_error(nullptr)); return 3; }
    int64_t device_bytes = 0;
    {
        int64_t avail = 0;
        if (bm2_bam2fq_memory(ctx, window, &device_bytes, &avail)) fail(3, std::string("bm2_bam2fq_memory: ") + bm2_last_error(ctx));
        if (device_bytes > avail)
            fail(1, "--window " + std::to_string(window) + ": one window needs " + std::to_string(device_bytes) + " bytes of device memory, " +
                        std::to_string(avail) + " bytes free");
    }
    b.records = [ctx, &b](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr) {
        const bm2_bam2fq_rec *out = nullptr;
        if (const int rc = bm2_bam2fq_records(ctx, r, n, st, nr, b.suffixes, &out)) b.die(rc == 2 ? 1 : 3, bm2_last_error(ctx));
        return out;
    };
    b.pair = [ctx, &b](const bm2_markdup_half *h, int64_t n, const uint8_t *names, int64_t nl) {
        const int32_t *partner = nullptr;
        if (bm2_markdup_pair(ctx, h, n, names, nl, &partner)) b.die(3, std::string("bm2_markdup_pair: ") + bm2_last_error(ctx));
        return partner;
    };
    b.format = [ctx, &b](const int64_t *list, int64_t n, const uint8_t *x, int64_t xl, const int64_t *xs, int64_t nx, const uint8_t *c, int64_t cl,
                         int compress, int last, bm2_bam2fq_out *out) {
        if (bm2_bam2fq_format(ctx, list, n, x, xl, xs, nx, b.suffixes, c, cl, compress, last, out)) b.die(3, bm2_last_error(ctx));
    };
    b.run();
    for (size_t at = 0; at < b.warning.size();) {
        const size_t e = b.warning.find('\n', at);
        fprintf(stderr, "[W::bm2_bam2fq] %s\n", b.warning.substr(at, e - at).c_str());
        at = e + 1;
    }
    bm2_bam2fq_stats_t s;
    bm2_markdup_stats_t ms;
    if (bm2_last_bam2fq_stats(ctx, &s) || bm2_last_markdup_stats(ctx, &ms)) fail(3, "bm2_last_bam2fq_stats");
    fprintf(stderr, "{\"records\": %lld, \"kept\": %lld, \"pairs\": %lld, \"others\": %lld, \"singletons\": %lld, \"others_dropped\": %lld, "
                    "\"singletons_dropped\": %lld, \"pending_max\": %lld, \"pending_bytes_max\": %lld, \"windows\": %lld, \"in_bytes\": %lld, "
                    "\"out_bytes\": %lld, \"inflate_s\": %.6f, \"record_s\": %.6f, \"pair_s\": %.6f, \"format_s\": %.6f, \"bgzf_s\": %.6f, "
                    "\"device_bytes\": %lld, \"wall_s\": %.6f}\n",
            (long long) b.n_records, (long long) b.kept, (long long) b.pairs, (long long) b.others, (long long) b.singletons, (long long) b.others_dropped,
            (long long) b.singletons_dropped, (long long) b.pending_max, (long long) b.pending_bytes_max, (long long) b.n_windows, (long long) b.in_bytes,
            (long long) b.out_bytes, b.inflate_s, s.record_ms / 1e3, ms.pair_ms / 1e3, s.format_ms / 1e3, s.bgzf_ms / 1e3, (long long) device_bytes,
            now_s() - t_start);
    bm2_destroy(ctx);
    return 0;
}

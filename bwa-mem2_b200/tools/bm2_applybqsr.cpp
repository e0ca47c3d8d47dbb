// bm2_applybqsr — GATK ApplyBQSR on the GPU: a BAM file's base qualities recalibrated from a BaseRecalibrator table (such as the one
// bm2_mem --recal-file writes), BGZF-compressed on the GPU (C++, over the C ABI of include/bm2_b200.h only).
//
//   bm2_applybqsr [-t INT] [-o out.bam] [--write-index] [--window SIZE] --bqsr-recal-file table.txt <in.bam | ->
//
//   table      parsed by bqsr_report.h into each read group's dense tables; a malformed table is an error naming the file and the line
//   input      read in windows of about --window uncompressed bytes (bam_window.h): the members are inflated by zlib on -t threads, and the
//              next window inflates on a thread of its own while the GPU recalibrates and compresses the current one, so host memory is
//              about two windows and device memory about one window, the BGZF slots and the tables
//   records    bm2_bqsr_apply (bqsr_apply.cu, bqsr_device.cuh's rule) rewrites the QUAL bytes on the device and compresses the stream with
//              the blocks cut by htslib's rule over all of it, so the bytes depend neither on -t nor on --window
//   output     the input's header plus an @PG line, in blocks of its own, the records in input order, the EOF block; with -o written to
//              <out>.tmp and renamed once complete.  --write-index (needs -o and a header with SO:coordinate) writes <out>.bai with the
//              BaiBuilder of bm2_mem --write-index; a record whose coordinate key is below the one before it is an error
// Exit codes: 0 success, 1 a usage, table, input or read error, 2 an output file that cannot be written, 3 a device error.
#include "bm2_b200.h"
#include "../csrc/bqsr_report.h"
#include "../csrc/bam_window.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <string>
#include <thread>
#include <unistd.h>
#include <vector>

namespace {

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

std::string g_tmp;                                  // the output being written, removed on an error

[[noreturn]] void fail(int code, const std::string &m) {
    fprintf(stderr, "[E::bm2_applybqsr] %s\n", m.c_str());
    fflush(stderr);
    if (!g_tmp.empty()) unlink(g_tmp.c_str());
    _Exit(code);
}

void usage() {
    fprintf(stderr,
            "Usage: bm2_applybqsr [options] --bqsr-recal-file table.txt <in.bam | ->\n"
            "Recalibrates the base qualities of a BAM file on the GPU from a GATK BaseRecalibrator table (GATK 4 ApplyBQSR at its defaults:\n"
            "no quantization, qualities below 6 kept, no OQ tag) and writes the same BAM with only the QUAL bytes changed.\n"
            "  --bqsr-recal-file FILE  the recalibration table (GATKReport v1.1), e.g. from bm2_mem --recal-file\n"
            "  -o FILE                 output file [standard output]\n"
            "  --write-index           also write FILE.bai (needs -o and a coordinate-sorted input)\n"
            "  -t INT                  inflate threads [1]\n"
            "  --window SIZE           uncompressed input bytes per window, suffix K, M or G [256M]\n");
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

// the value of a header line's tag ("ID:"), empty without it
std::string tag_of(const std::string &line, const char *tag) {
    const size_t at = line.find(std::string("\t") + tag);
    if (at == std::string::npos) return "";
    const size_t b = at + 4, e = line.find('\t', b);
    return line.substr(b, (e == std::string::npos ? line.size() : e) - b);
}

}  // namespace

int main(int argc, char **argv) {
    const double t_start = now_s();
    const char *out_path = nullptr, *table_path = nullptr, *in_path = nullptr;
    bool write_index = false;
    long long threads = 1, window = 256LL << 20;        // 256M: a chosen figure, not a measured one
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) out_path = value("-o");
        else if (!strcmp(s, "--bqsr-recal-file")) table_path = value("--bqsr-recal-file");
        else if (!strcmp(s, "--write-index")) write_index = true;
        else if (!strcmp(s, "-t")) {
            char *e; threads = strtoll(value("-t"), &e, 10);
            if (*e || threads < 1 || threads > 1024) fail(1, "-t takes a number of threads from 1 to 1024");
        } else if (!strcmp(s, "--window")) {
            if (!parse_size(value("--window"), &window)) fail(1, "--window takes a size such as 64K, 256M or 1G");
        } else if (s[0] == '-' && s[1]) { usage(); fail(1, std::string("unknown option ") + s); }
        else if (in_path) { usage(); fail(1, "more than one input"); }
        else in_path = s;
    }
    if (!in_path) { usage(); fail(1, "no input BAM"); }
    if (!table_path) { usage(); fail(1, "--bqsr-recal-file is required"); }
    if (write_index && !out_path) fail(1, "--write-index needs -o");

    // the table
    BqsrApplyTables tabs;
    {
        FILE *f = fopen(table_path, "rb");
        if (!f) fail(1, std::string("cannot open ") + table_path);
        std::string text;
        char buf[1 << 16];
        for (size_t k; (k = fread(buf, 1, sizeof buf, f)) > 0;) text.append(buf, k);
        fclose(f);
        const std::string e = bqsr_parse_report(text, table_path, tabs);
        if (!e.empty()) fail(1, e);
    }

    // the header
    BamWindowReader rd;
    rd.name = strcmp(in_path, "-") ? in_path : "standard input";
    rd.f = strcmp(in_path, "-") ? fopen(in_path, "rb") : stdin;
    if (!rd.f) fail(1, std::string("cannot open ") + in_path);
    rd.threads = (int) threads; rd.window = window;
    std::string text;
    std::vector<std::pair<std::string, int32_t>> refs;
    std::string e = rd.header(text, refs);
    if (!e.empty()) fail(1, e);
    std::vector<std::string> ids;
    std::vector<int32_t> id_table;
    std::set<std::string> pg_ids;
    std::string last_pg, hd;
    for (size_t b = 0; b < text.size();) {
        size_t en = text.find('\n', b); if (en == std::string::npos) en = text.size();
        const std::string line = text.substr(b, en - b);
        if (line.compare(0, 4, "@RG\t") == 0) {
            ids.push_back(tag_of(line, "ID:"));
            const std::string rg = bqsr_read_group(line);
            int32_t k = -1;
            for (size_t j = 0; j < tabs.rgs.size(); ++j) if (tabs.rgs[j] == rg) { k = (int32_t) j; break; }
            id_table.push_back(k);
        } else if (line.compare(0, 4, "@PG\t") == 0) {
            last_pg = tag_of(line, "ID:");
            pg_ids.insert(last_pg);
        } else if (line.compare(0, 4, "@HD\t") == 0 && hd.empty()) hd = line;
        b = en + 1;
    }
    if (write_index && tag_of(hd, "SO:") != "coordinate") fail(1, "--write-index needs a coordinate-sorted input (@HD SO:coordinate)");

    // the device
    bm2_mem_opt_t opt;
    bm2_opt_init(&opt);
    bm2_ctx *ctx = nullptr;
    if (bm2_create(&ctx, 0, nullptr, &opt)) { fprintf(stderr, "bm2_applybqsr: %s\n", bm2_last_error(nullptr)); return 3; }
    auto die = [&](const char *what) { fail(3, std::string(what) + ": " + bm2_last_error(ctx)); };
    {
        int64_t need = 0, avail = 0;
        if (bm2_bqsr_apply_memory(ctx, window, (int32_t) tabs.rgs.size(), &need, &avail)) die("bm2_bqsr_apply_memory");
        if (need > avail)
            fail(1, "--window " + std::to_string(window) + ": one window needs " + std::to_string(need) + " bytes of device memory, " +
                        std::to_string(avail) + " bytes free");
    }
    std::vector<const char *> cids;
    for (const std::string &s : ids) cids.push_back(s.c_str());
    bm2_bqsr_apply_tables_t at;
    at.n_rg = (int32_t) tabs.rgs.size(); at.P = tabs.P.data(); at.ctx = tabs.ctx.data(); at.cyc = tabs.cyc.data();
    at.n_ids = (int32_t) ids.size(); at.ids = cids.data(); at.id_table = id_table.data();
    if (bm2_bqsr_apply_set(ctx, &at)) fail(1, bm2_last_error(ctx));

    // the output header: the input's, plus this program's @PG line, in blocks of its own
    std::string pg_id = "bm2_applybqsr";
    for (int k = 1; pg_ids.count(pg_id); ++k) pg_id = "bm2_applybqsr." + std::to_string(k);
    std::string out_text = text;
    while (!out_text.empty() && out_text.back() == '\0') out_text.pop_back();
    if (!out_text.empty() && out_text.back() != '\n') out_text += '\n';
    out_text += "@PG\tID:" + pg_id + "\tPN:bm2_applybqsr" + (last_pg.empty() ? "" : "\tPP:" + last_pg) + "\tVN:b200-r2\tCL:" + argv[0];
    for (int i = 1; i < argc; ++i) out_text += std::string(" ") + argv[i];
    out_text += "\n";
    std::string h("BAM\1", 4);
    auto i32 = [&](int32_t v) { h.append((const char *) &v, 4); };
    i32((int32_t) out_text.size()); h += out_text;
    i32((int32_t) refs.size());
    for (const auto &r : refs) { i32((int32_t) r.first.size() + 1); h.append(r.first.c_str(), r.first.size() + 1); i32(r.second); }
    FILE *out = stdout;
    if (out_path) {
        g_tmp = std::string(out_path) + ".tmp";
        out = fopen(g_tmp.c_str(), "wb");
        if (!out) { g_tmp.clear(); fail(2, std::string("cannot open ") + out_path + ".tmp"); }
    }
    const uint8_t *z = nullptr; int64_t zl = 0;
    if (bm2_bgzf_compress(ctx, (const uint8_t *) h.data(), (int64_t) h.size(), nullptr, 0, &z, &zl)) die("bm2_bgzf_compress");
    if (fwrite(z, 1, (size_t) zl, out) != (size_t) zl) fail(2, "cannot write the output");

    // the windows: the next one inflates while the device takes the current one
    BaiBuilder bai((int) refs.size());
    SortedWriter w{[ctx](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, const int64_t *, const uint8_t *c, int64_t cl, int last,
                         bm2_sort_out *o, const int64_t **, double *) {
                       if (bm2_bqsr_apply(ctx, r, n, st, nr, c, cl, last, o)) {
                           bm2_bqsr_apply_stats_t s;
                           fail(!bm2_last_bqsr_apply_stats(ctx, &s) && s.err_kind ? 1 : 3, bm2_last_error(ctx));
                       }
                       return 0;
                   },
                   [](const std::string &m) { fail(2, m == "bm2_bam_sort_compress" ? "bm2_bqsr_apply" : m); }, out, write_index ? &bai : nullptr,
                   (uint64_t) zl};
    std::vector<uint8_t> buf[2];
    std::vector<int64_t> starts[2];
    e = rd.next(buf[0], starts[0]);
    if (!e.empty()) fail(1, e);
    int64_t n_windows = 0, n_records = 0;
    uint64_t prev_key = 0;
    for (int cur = 0; !starts[cur].empty(); cur ^= 1) {
        std::string e_next;
        std::thread next([&] { e_next = rd.next(buf[cur ^ 1], starts[cur ^ 1]); });
        const std::vector<uint8_t> &B = buf[cur];
        const std::vector<int64_t> &S = starts[cur];
        if (write_index)
            for (size_t i = 0; i < S.size(); ++i) {
                const BamFixed f = bam_fixed(B.data() + S[i]);
                const uint64_t k = bam_coord_key(f.rid, f.pos, f.flag);
                if (n_records + (int64_t) i > 0 && k < prev_key) {
                    next.join();
                    fail(1, "--write-index: read " + std::string((const char *) B.data() + S[i] + 36) + " is out of coordinate order");
                }
                prev_key = k;
            }
        w.write(B.data(), (int64_t) B.size(), S.data(), (int64_t) S.size(), nullptr, false);
        n_records += (int64_t) S.size(); ++n_windows;
        next.join();
        if (!e_next.empty()) fail(1, e_next);
    }
    w.write(nullptr, 0, nullptr, 0, nullptr, true);
    static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (fwrite(eof, 1, sizeof eof, out) != sizeof eof || fflush(out)) fail(2, "cannot write the output");
    if (!rd.warning.empty()) fprintf(stderr, "[W::bm2_applybqsr] %s\n", rd.warning.c_str());
    if (rd.f != stdin) fclose(rd.f);
    if (out_path) {
        if (fclose(out)) fail(2, std::string("cannot write ") + g_tmp);
        if (write_index) {
            const std::string b = bai.bytes(), path = std::string(out_path) + ".bai", tmp = path + ".tmp";
            FILE *f = fopen(tmp.c_str(), "wb");
            if (!f || fwrite(b.data(), 1, b.size(), f) != b.size() || fclose(f) || rename(tmp.c_str(), path.c_str())) {
                unlink(tmp.c_str());
                fail(2, "cannot write " + path);
            }
        }
        if (rename(g_tmp.c_str(), out_path)) fail(2, std::string("cannot write ") + out_path);
        g_tmp.clear();
    }
    bm2_bqsr_apply_stats_t s;
    if (bm2_last_bqsr_apply_stats(ctx, &s)) die("bm2_last_bqsr_apply_stats");
    fprintf(stderr, "{\"records\": %lld, \"recal_records\": %lld, \"unrecalibrated_records\": %lld, \"recal_bases\": %lld, \"windows\": %lld, "
                    "\"in_bytes\": %lld, \"out_bytes\": %lld, \"inflate_s\": %.6f, \"apply_s\": %.6f, \"bgzf_s\": %.6f, \"wall_s\": %.6f}\n",
            (long long) n_records, (long long) s.recal_records, (long long) s.kept_records, (long long) s.bases_changed, (long long) n_windows,
            (long long) rd.in_bytes, (long long) (w.file_off + sizeof eof), rd.inflate_s, s.apply_ms / 1e3, s.bgzf_ms / 1e3, now_s() - t_start);
    bm2_destroy(ctx);
    return 0;
}

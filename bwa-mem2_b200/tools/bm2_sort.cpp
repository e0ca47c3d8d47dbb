// bm2_sort — samtools sort of one BAM file in any order, by coordinate or by read name (-n), the runs sorted and compressed on the GPU in
// bounded memory (C++, over the C ABI of include/bm2_b200.h only).
//
//   bm2_sort [-n] [-t INT] [--window SIZE] [--sort-mem SIZE] [--write-index] [-o out.bam] <in.bam | ->
//
//   input    read in windows of about --window uncompressed bytes (bam_window.h), inflated on -t threads; the next window inflates on a
//            thread of its own while the records of the current one are checked and added to the sink
//   runs     bam_sort.h's BamSortSink, as for bm2_mem --sort: runs of --sort-mem uncompressed bytes sorted on the GPU and spilled to unlinked
//            temporary files (<out>.tmp.NNNN, or ${TMPDIR:-/tmp}/bm2_sort.<pid>.NNNN on standard output), merged window by window.
//            Coordinate order is bm2_bam_sort_compress's key; -n is bm2_bam_qname_sort_compress, with bam_qname_cmp as the sink's merge order
//   output   the input's header with its @HD line first and SO set, plus an @PG line, in blocks of its own; the records byte for byte in the
//            new order, cut into blocks by htslib's rule over the whole stream; the EOF block.  With -o written to <out>.tmp and renamed once
//            complete; --write-index (coordinate order and -o only) writes <out>.bai with bm2_mem --write-index's BaiBuilder
// Exit codes: 0 success, 1 a usage, input or read error, 2 an output file that cannot be written, 3 a device error.
#include "bm2_b200.h"
#include "../csrc/bam_window.h"
#include "../csrc/sort_header.h"
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
    fprintf(stderr, "[E::bm2_sort] %s\n", m.c_str());
    fflush(stderr);
    if (!g_tmp.empty()) unlink(g_tmp.c_str());
    _Exit(code);
}

void usage() {
    fprintf(stderr,
            "Usage: bm2_sort [options] <in.bam | ->\n"
            "Sorts the records of a BAM file in any order by coordinate (samtools sort) or by read name (samtools sort -n), on the GPU, and\n"
            "writes them byte for byte in the new order.\n"
            "  -n               read-name order: samtools' natural order of the names, then READ1/READ2 flags, then input order\n"
            "  -o FILE          output file [standard output]\n"
            "  --write-index    also write FILE.bai (needs -o and coordinate order)\n"
            "  -t INT           inflate threads [1]\n"
            "  --window SIZE    uncompressed input bytes per window, suffix K, M or G [256M]\n"
            "  --sort-mem SIZE  uncompressed bytes per sorted run, suffix K, M or G [2G]\n");
}

// the value of a header line's tag ("ID:"), empty without it
std::string tag_of(const std::string &line, const char *tag) {
    const size_t at = line.find(std::string("\t") + tag);
    if (at == std::string::npos) return "";
    const size_t b = at + 4, e = line.find('\t', b);
    return line.substr(b, (e == std::string::npos ? line.size() : e) - b);
}

// what is wrong with record r (block_size first, at least 36 bytes), "" when nothing: the device key kernels read its QNAME and CIGAR without
// bounds, so a record must pass this before it reaches them
std::string record_problem(const uint8_t *r, int32_t n_ref) {
    const int32_t bs = bam_le32(r), lrn = r[12], n_cigar = (int32_t) bam_le16(r + 16), l_seq = bam_le32(r + 20);
    if (bs < 32) return "block_size " + std::to_string(bs) + " is below 32";
    if (lrn < 1) return "l_read_name is 0";
    if (l_seq < 0) return "l_seq " + std::to_string(l_seq) + " is negative";
    if (32 + (int64_t) lrn + 4 * (int64_t) n_cigar + ((int64_t) l_seq + 1) / 2 + l_seq > bs) return "its fields overrun its block_size";
    if (r[36 + lrn - 1]) return "its read name does not end with NUL";
    const int32_t rid = bam_le32(r + 4), pos = bam_le32(r + 8), mrid = bam_le32(r + 24);
    if (rid < -1 || rid >= n_ref) return "refID " + std::to_string(rid) + " is outside [-1, " + std::to_string(n_ref) + ")";
    if (mrid < -1 || mrid >= n_ref) return "next refID " + std::to_string(mrid) + " is outside [-1, " + std::to_string(n_ref) + ")";
    if (pos < -1) return "pos " + std::to_string(pos) + " is below -1";
    return "";
}

// the record's QNAME for a message, when it lies inside the record and ends with its NUL
std::string readable_name(const uint8_t *r) {
    const int32_t bs = bam_le32(r), lrn = r[12];
    if (lrn < 1 || 32 + lrn > bs || r[36 + lrn - 1]) return "";
    return std::string((const char *) r + 36);
}

}  // namespace

int main(int argc, char **argv) {
    const double t_start = now_s();
    const char *out_path = nullptr, *in_path = nullptr;
    bool by_name = false, write_index = false;
    long long threads = 1, window = 256LL << 20;        // 256M: a chosen figure, not a measured one
    long long sort_mem = 2LL << 30;                     // bm2_mem's --sort-mem default: a chosen figure, not a measured one
    for (int i = 1; i < argc; ++i) {
        const char *s = argv[i];
        auto value = [&](const char *opt) { if (i + 1 >= argc) { usage(); fail(1, std::string(opt) + " takes a value"); } return argv[++i]; };
        if (!strcmp(s, "-o")) out_path = value("-o");
        else if (!strcmp(s, "-n")) by_name = true;
        else if (!strcmp(s, "--write-index")) write_index = true;
        else if (!strcmp(s, "-t")) {
            char *e; threads = strtoll(value("-t"), &e, 10);
            if (*e || threads < 1 || threads > 1024) fail(1, "-t takes a number of threads from 1 to 1024");
        } else if (!strcmp(s, "--window")) {
            if (!parse_size(value("--window"), &window)) fail(1, "--window takes a size such as 64K, 256M or 1G");
        } else if (!strcmp(s, "--sort-mem")) {
            if (!parse_size(value("--sort-mem"), &sort_mem)) fail(1, "--sort-mem takes a positive byte count with an optional K, M or G suffix");
        } else if (s[0] == '-' && s[1]) { usage(); fail(1, std::string("unknown option ") + s); }
        else if (in_path) { usage(); fail(1, "more than one input"); }
        else in_path = s;
    }
    if (!in_path) { usage(); fail(1, "no input BAM"); }
    if (write_index && by_name) fail(1, "--write-index needs coordinate order: it cannot be given with -n");
    if (write_index && !out_path) fail(1, "--write-index needs -o");

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
    if (write_index)
        for (const auto &r : refs)
            if (r.second > (1 << 29) - 1)
                fail(1, "--write-index: contig " + r.first + " is longer than 2^29-1 bases, beyond what a BAI index addresses");
    while (!text.empty() && text.back() == '\0') text.pop_back();
    std::set<std::string> pg_ids;
    std::string last_pg;
    for (size_t b = 0; b < text.size();) {
        size_t en = text.find('\n', b); if (en == std::string::npos) en = text.size();
        const std::string line = text.substr(b, en - b);
        if (line.compare(0, 4, "@PG\t") == 0) { last_pg = tag_of(line, "ID:"); pg_ids.insert(last_pg); }
        b = en + 1;
    }
    std::string pg_id = "bm2_sort";
    for (int k = 1; pg_ids.count(pg_id); ++k) pg_id = "bm2_sort." + std::to_string(k);
    std::string out_text = header_with_sort_order(text, by_name ? "queryname" : "coordinate");
    out_text += "@PG\tID:" + pg_id + "\tPN:bm2_sort" + (last_pg.empty() ? "" : "\tPP:" + last_pg) + "\tVN:b200-r2\tCL:" + argv[0];
    for (int i = 1; i < argc; ++i) out_text += std::string(" ") + argv[i];
    out_text += "\n";

    // the device
    bm2_mem_opt_t opt;
    bm2_opt_init(&opt);
    bm2_ctx *ctx = nullptr;
    if (bm2_create(&ctx, 0, nullptr, &opt)) { fprintf(stderr, "bm2_sort: %s\n", bm2_last_error(nullptr)); return 3; }
    auto die = [&](const char *what) { fail(3, std::string(what) + ": " + bm2_last_error(ctx)); };
    int64_t device_bytes = 0;
    {
        int64_t avail = 0;
        if ((by_name ? bm2_bam_qname_sort_memory : bm2_bam_sort_memory)(ctx, sort_mem, &device_bytes, &avail)) die("bm2_bam_sort_memory");
        if (device_bytes > avail)
            fail(1, "--sort-mem " + std::to_string(sort_mem) + ": one run sort needs " + std::to_string(device_bytes) + " bytes of device memory, " +
                        std::to_string(avail) + " bytes free");
    }

    // the output header, in blocks of its own
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

    // the sink: calls come one at a time (the sorter thread's spills, then the merge on this thread)
    double stage_s[4] = {0, 0, 0, 0};
    BamSortSink sink;
    sink.sort = [ctx, by_name, &stage_s](const uint8_t *r, int64_t n, const int64_t *st, int64_t nr, const uint8_t *c, int64_t cl, int last,
                                         bm2_sort_out *o, double *device_s) {
        const int rc = (by_name ? bm2_bam_qname_sort_compress : bm2_bam_sort_compress)(ctx, r, n, st, nr, c, cl, last, o);
        double ms[4] = {0, 0, 0, 0};
        bm2_last_sort_stats(ctx, ms);
        for (int k = 0; k < 4; ++k) stage_s[k] += ms[k] / 1e3;
        *device_s = (ms[0] + ms[1] + ms[2] + ms[3]) / 1e3;
        return rc;
    };
    if (by_name) sink.cmp = bam_qname_rec_cmp;
    sink.fail = [ctx, by_name](const std::string &m) {
        if (m == "bm2_bam_sort_compress") fail(3, std::string(by_name ? "bm2_bam_qname_sort_compress" : m) + ": " + bm2_last_error(ctx));
        fail(m == "a malformed BAM record" ? 1 : 2, m);
    };
    sink.run_bytes = sort_mem; sink.threads = (int) threads;
    if (out_path) sink.tmp_prefix = std::string(out_path) + ".tmp.";
    else {
        const char *td = getenv("TMPDIR");
        sink.tmp_prefix = std::string(td && *td ? td : "/tmp") + "/bm2_sort." + std::to_string((long long) getpid()) + ".";
    }

    // the windows: the next one inflates while the records of the current one are checked and added
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
        for (size_t i = 0; i < S.size(); ++i) {
            const std::string p = record_problem(B.data() + S[i], (int32_t) refs.size());
            if (p.empty()) continue;
            next.join();
            const std::string name = readable_name(B.data() + S[i]);
            fail(1, rd.where() + "record " + std::to_string(n_records + (int64_t) i) + (name.empty() ? "" : " (read " + name + ")") + " is malformed: " + p);
        }
        sink.add(B.data(), (int64_t) B.size());
        n_records += (int64_t) S.size(); ++n_windows;
        next.join();
        if (!e_next.empty()) fail(1, e_next);
    }
    if (!rd.warning.empty()) fprintf(stderr, "[W::bm2_sort] %s\n", rd.warning.c_str());
    if (rd.f != stdin) fclose(rd.f);

    BaiBuilder bai((int) refs.size());
    sink.finish(out, (uint64_t) zl, write_index ? &bai : nullptr);
    static const uint8_t eof[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (fwrite(eof, 1, sizeof eof, out) != sizeof eof || fflush(out)) fail(2, "cannot write the output");
    double index_s = 0;
    if (out_path) {
        if (fclose(out)) fail(2, std::string("cannot write ") + g_tmp);
        if (write_index) {
            const double t0 = now_s();
            const std::string b = bai.bytes(), path = std::string(out_path) + ".bai", tmp = path + ".tmp";
            FILE *f = fopen(tmp.c_str(), "wb");
            if (!f || fwrite(b.data(), 1, b.size(), f) != b.size() || fclose(f) || rename(tmp.c_str(), path.c_str())) {
                unlink(tmp.c_str());
                fail(2, "cannot write " + path);
            }
            index_s = now_s() - t0;
        }
        if (rename(g_tmp.c_str(), out_path)) fail(2, std::string("cannot write ") + out_path);
        g_tmp.clear();
    }
    fprintf(stderr, "{\"records\": %lld, \"windows\": %lld, \"in_bytes\": %lld, \"inflate_s\": %.6f, \"sort_runs\": %lld, \"spill_bytes\": %lld, "
                    "\"sort_s\": %.6f, \"sort_stage_s\": [%.6f, %.6f, %.6f, %.6f], \"merge_s\": %.6f, \"merge_windows\": %lld, \"index_s\": %.6f, "
                    "\"device_bytes\": %lld, \"wall_s\": %.6f}\n",
            (long long) n_records, (long long) n_windows, (long long) rd.in_bytes, rd.inflate_s, (long long) std::max<size_t>(sink.runs.size(), 1),
            (long long) sink.spill_bytes, stage_s[0] + stage_s[1] + stage_s[2] + stage_s[3], stage_s[0], stage_s[1], stage_s[2], stage_s[3],
            sink.merge_s, (long long) sink.merge_windows, index_s, (long long) device_bytes, now_s() - t_start);
    bm2_destroy(ctx);
    return 0;
}

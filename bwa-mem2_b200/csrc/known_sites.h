// known_sites.h — the known-variant VCFs of bm2_mem --known-sites, read on the host into the two bitsets of bm2_bqsr_sites.
//   input     each file plain, gzip or BGZF (read_input.h's InputStream); lines starting with '#' are headers, empty lines are skipped
//   a record  at least the 8 tab-separated fixed columns; CHROM a contig of the index; POS a decimal integer >= 1; REF one or more letters.
//             It covers POS .. POS + len(REF) - 1 (1-based), whatever its FILTER; INFO/END is ignored
//   bitsets   over the forward strand's concatenated contigs: covered bit p for every base a record covers, junction bit p when one record
//             covers both p and p + 1
//   errors    a file that cannot be read, a CHROM that is not a contig, a record past its contig's end, a malformed line: named by file and
//             line number
#pragma once
#include "read_input.h"
#include <cctype>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

struct KnownSites {
    std::vector<uint64_t> covered, junction;
    int64_t records = 0;
};

inline void known_sites_set(std::vector<uint64_t> &b, int64_t beg, int64_t end) {
    for (int64_t p = beg; p < end;) {
        if ((p & 63) == 0 && p + 64 <= end) { b[(size_t) (p >> 6)] = ~(uint64_t) 0; p += 64; continue; }
        b[(size_t) (p >> 6)] |= (uint64_t) 1 << (p & 63); ++p;
    }
}

// one data line (without its newline) of file:line; returns "" or the error
inline std::string known_sites_line(const std::string &line, const std::string &where, const std::unordered_map<std::string, size_t> &contig,
                                    const std::vector<int64_t> &off, const std::vector<int64_t> &len, KnownSites &ks) {
    size_t f[4], nf = 0, tabs = 0;
    for (size_t i = 0; i < line.size(); ++i) if (line[i] == '\t') { if (nf < 4) f[nf++] = i; ++tabs; }
    if (tabs < 7) return where + ": a VCF data line needs the 8 tab-separated fixed columns";
    const std::string chrom = line.substr(0, f[0]), pos = line.substr(f[0] + 1, f[1] - f[0] - 1), ref = line.substr(f[2] + 1, f[3] - f[2] - 1);
    if (pos.empty() || pos.size() > 12) return where + ": POS is not a positive integer";
    for (char c : pos) if (!isdigit((unsigned char) c)) return where + ": POS is not a positive integer";
    const int64_t p = std::stoll(pos);
    if (p < 1) return where + ": POS is not a positive integer";
    if (ref.empty()) return where + ": REF is empty";
    for (char c : ref) if (!isalpha((unsigned char) c)) return where + ": REF is not a string of bases";
    const auto it = contig.find(chrom);
    if (it == contig.end()) return where + ": CHROM " + chrom + " is not a contig of the index";
    const int64_t e = p + (int64_t) ref.size() - 1;
    if (e > len[it->second])
        return where + ": the record ends at " + chrom + ":" + std::to_string(e) + ", past the contig's end (" + std::to_string(len[it->second]) + ")";
    const int64_t g = off[it->second] + p - 1;
    known_sites_set(ks.covered, g, g + (int64_t) ref.size());
    known_sites_set(ks.junction, g, g + (int64_t) ref.size() - 1);
    ++ks.records;
    return std::string();
}

// every file into ks (sized to l_pac bits); returns "" or the first error
inline std::string read_known_sites(const std::vector<std::string> &paths, const std::vector<std::string> &names, const std::vector<int64_t> &off,
                                    const std::vector<int64_t> &len, int64_t l_pac, KnownSites &ks) {
    std::unordered_map<std::string, size_t> contig;
    for (size_t i = 0; i < names.size(); ++i) contig.emplace(names[i], i);
    ks.covered.assign((size_t) ((l_pac + 63) / 64), 0);
    ks.junction.assign((size_t) ((l_pac + 63) / 64), 0);
    ks.records = 0;
    std::vector<char> buf((size_t) 1 << 20);
    for (const std::string &path : paths) {
        InputStream in;
        if (!in.open(path.c_str())) return in.error_msg;
        std::string line;
        int64_t ln = 0;
        auto take = [&]() -> std::string {
            ++ln;
            if (!line.empty() && line.back() == '\r') line.pop_back();
            std::string err;
            if (!line.empty() && line[0] != '#') err = known_sites_line(line, path + ":" + std::to_string(ln), contig, off, len, ks);
            line.clear();
            return err;
        };
        for (;;) {
            const int64_t r = in.read(buf.data(), buf.size());
            if (r < 0) return in.error_msg;
            if (r == 0) break;
            for (int64_t i = 0; i < r; ++i) {
                if (buf[(size_t) i] != '\n') { line += buf[(size_t) i]; continue; }
                const std::string err = take();
                if (!err.empty()) return err;
            }
        }
        if (!line.empty()) { const std::string err = take(); if (!err.empty()) return err; }
    }
    return std::string();
}

// bqsr_recal.h — the host side of bm2_baserecalibrator that is not the report (bqsr_report.h): the read groups of the inputs' headers, the
// read-group map the counting kernel looks IDs up in, and the placement check of a record.  Host only, so that
// tests/host_emul/baserecalibrator_emul.cpp compiles the same code.
//
//   read groups  the union of the inputs' @RG lines: each ID maps to its covariate, the line's PU, else its ID (bqsr_read_group); the first
//                line of an ID within one input is the one read.  An input without an @RG line, and one ID in two inputs with different
//                covariates, are errors.  The covariates are numbered in the byte order of their strings, which is the order of the report's
//                rows; several IDs with one covariate count into one row set.
//   map          n_ids BqsrRgEntry {offset of the ID's bytes from the map's start, length, value, 0}, then the IDs' bytes, padded to 16
//   placement    a record that passes bqsr_prep's filters must lie inside its contig (pos >= 0, pos + its CIGAR's reference length <= the
//                contig's length), or the kernel would read past the reference: such a record is malformed, which is an error naming it
#pragma once
#include "bqsr_report.h"
#include <algorithm>
#include <map>
#include <string>
#include <vector>

struct BqsrReadGroups {
    std::vector<std::string> ids;        // every @RG ID of the inputs, in order of first appearance
    std::vector<int32_t> id_cov;         // each ID's covariate index
    std::vector<std::string> covs;       // the covariates, in byte order
};

// texts: each input's header text; names: each input's name for the messages
inline std::string bqsr_read_groups(const std::vector<std::string> &texts, const std::vector<std::string> &names, BqsrReadGroups &out) {
    std::map<std::string, std::string> cov_of;           // ID -> covariate
    std::map<std::string, size_t> from;                  // ID -> the input it came from first
    std::vector<std::string> order;
    for (size_t i = 0; i < texts.size(); ++i) {
        std::map<std::string, std::string> here;
        for (size_t b = 0; b < texts[i].size();) {
            size_t e = texts[i].find('\n', b);
            if (e == std::string::npos) e = texts[i].size();
            const std::string line = texts[i].substr(b, e - b);
            b = e + 1;
            if (line.compare(0, 4, "@RG\t") != 0) continue;
            const std::string id = bqsr_rg_tag(line, "ID:");
            if (!here.count(id)) here[id] = bqsr_read_group(line);
            else continue;
            const auto it = cov_of.find(id);
            if (it == cov_of.end()) { cov_of[id] = here[id]; from[id] = i; order.push_back(id); }
            else if (it->second != here[id])
                return names[i] + ": read group " + id + " has covariate " + here[id] + " here and " + it->second + " in " + names[from[id]];
        }
        if (here.empty()) return names[i] + ": the header has no @RG line, so its reads have no read group";
    }
    out.ids = order;
    out.covs.clear();
    for (const auto &kv : cov_of) out.covs.push_back(kv.second);
    std::sort(out.covs.begin(), out.covs.end());
    out.covs.erase(std::unique(out.covs.begin(), out.covs.end()), out.covs.end());
    out.id_cov.clear();
    for (const std::string &id : order)
        out.id_cov.push_back((int32_t) (std::lower_bound(out.covs.begin(), out.covs.end(), cov_of[id]) - out.covs.begin()));
    return "";
}

// the map of ids with their values; "" or the error when it would be larger than kBqsrMapMax
inline std::string bqsr_rg_map(const std::vector<std::string> &ids, const std::vector<int32_t> &vals, std::vector<uint8_t> &blob) {
    int64_t bytes = 0;
    for (const std::string &s : ids) bytes += (int64_t) s.size();
    const int64_t total = (16 * (int64_t) ids.size() + bytes + 15) / 16 * 16;
    if (total > kBqsrMapMax)
        return "the read-group IDs take " + std::to_string(total) + " bytes with 16 per ID, more than " + std::to_string(kBqsrMapMax);
    blob.assign((size_t) total, 0);
    int32_t at = 16 * (int32_t) ids.size();
    for (size_t i = 0; i < ids.size(); ++i) {
        const BqsrRgEntry e{at, (int32_t) ids[i].size(), vals[i], 0};
        memcpy(blob.data() + 16 * i, &e, 16);
        memcpy(blob.data() + at, ids[i].data(), ids[i].size());
        at += (int32_t) ids[i].size();
    }
    return "";
}

// true when the record (rec: its block_size field) passes bqsr_prep's filters and does not lie inside its contig
inline bool bqsr_outside_contig(const uint8_t *rec, const int32_t *contig_len, int32_t n_seqs) {
    const int32_t rid = bqsr_le32(rec + 4), pos = bqsr_le32(rec + 8), l_seq = bqsr_le32(rec + 20);
    const int l_name = rec[12], mapq = rec[13], n_cigar = rec[16] | rec[17] << 8, flag = rec[18] | rec[19] << 8;
    if ((flag & (0x4 | 0x100 | 0x800 | 0x400 | 0x200)) || mapq == 0 || mapq == 255 || rid < 0 || rid >= n_seqs || n_cigar == 0 || l_seq <= 0) return false;
    int64_t rlen = 0;
    const uint32_t *cig = (const uint32_t *) (rec + 36 + l_name);
    for (int c = 0; c < n_cigar; ++c) {
        const uint32_t o = bqsr_cig(cig, c), op = o & 15;
        if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += o >> 4;
    }
    return pos < 0 || (int64_t) pos + rlen > contig_len[rid];
}

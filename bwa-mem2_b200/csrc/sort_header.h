// sort_header.h — what bm2_mem --sort and bm2_sort share on the host: the SIZE parser of --sort-mem and the @HD line of a sorted output.
#pragma once
#include <cctype>
#include <cerrno>
#include <cstdint>
#include <cstdlib>
#include <string>

// "SIZE" of --sort-mem: a positive decimal integer, optionally followed by one of K M G (binary multiples, either case)
inline bool parse_size(const char *s, long long *v) {
    char *e;
    if (!isdigit((unsigned char) *s)) return false;
    errno = 0;
    const unsigned long long x = strtoull(s, &e, 10);
    int shift = 0;
    if (*e == 'k' || *e == 'K') shift = 10, ++e;
    else if (*e == 'm' || *e == 'M') shift = 20, ++e;
    else if (*e == 'g' || *e == 'G') shift = 30, ++e;
    if (*e || errno || x == 0 || x > (unsigned long long) (INT64_MAX >> shift)) return false;
    *v = (long long) (x << shift);
    return true;
}

// the header text h with its first @HD line moved to the front and SO:<so> set in place of its SO field (or appended), its other fields kept;
// "@HD\tVN:1.6\tSO:<so>" when h has none.  Every line of the result ends with a newline.
inline std::string header_with_sort_order(const std::string &h, const std::string &so) {
    std::string hd, rest;
    for (size_t b = 0; b < h.size();) {
        size_t e = h.find('\n', b); if (e == std::string::npos) e = h.size();
        const std::string line = h.substr(b, e - b);
        if (hd.empty() && (line == "@HD" || line.compare(0, 4, "@HD\t") == 0)) {
            hd = "@HD";
            bool seen = false;
            for (size_t p = 3; p < line.size();) {
                size_t q = line.find('\t', p + 1); if (q == std::string::npos) q = line.size();
                const std::string f = line.substr(p + 1, q - p - 1);
                if (f.compare(0, 3, "SO:") == 0) { if (!seen) hd += "\tSO:" + so; seen = true; }
                else hd += "\t" + f;
                p = q;
            }
            if (!seen) hd += "\tSO:" + so;
        } else rest += line + "\n";
        b = e + 1;
    }
    return (hd.empty() ? "@HD\tVN:1.6\tSO:" + so : hd) + "\n" + rest;
}

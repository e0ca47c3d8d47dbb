// seq_emul.cpp — TEST ONLY: bm2_seq_encode's record resolution on the host, over the same grammar (bwa-mem2_b200/csrc/seq_grammar.cuh) and
// the same position tables as the kernels: candidates (the first '>' / '@' at or after each line start, deduplicated), next() by one
// seq_record walk each, the chain from the first candidate marked by pointer doubling, then every record walked again into a sink.
//   seq_emul <file>
// Output: "R <n>\n" and per record the fields of tests/host_emul/bseq_dump.cpp (qualities "-1:" when l_qual == 0, comment "-1:" when
// empty), or "E <record index>\n" at the first malformed record.  Last line "S <simple records> <mismatches>": on every simple record,
// fastq_spans_kernel's rules (fastq.cu) restated here must give the same name, comment, sequence and qualities, and kseq must leave
// qualities (the path of bm2_fastq_encode has no reads without them).
#include "seq_grammar.cuh"
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

struct StrSink {
    const char *raw; std::string *s_seq, *s_qual;
    void seq(int64_t b, int64_t k, int64_t at) const { put(*s_seq, b, k, at); }
    void qual(int64_t b, int64_t k, int64_t at) const { put(*s_qual, b, k, at); }
    void put(std::string &s, int64_t b, int64_t k, int64_t at) const {
        if (k <= 0) return;
        if ((int64_t) s.size() < at + k) s.resize((size_t) (at + k));
        memcpy(&s[(size_t) at], raw + b, (size_t) k);
    }
};

static void field(const char *p, int64_t n) { printf("%lld:", (long long) n); fwrite(p, 1, (size_t) n, stdout); }

// fastq_spans_kernel's rules on the four lines from h: name, comment, sequence, qualities (false: the kernel reports the record malformed)
static bool spans_rules(const std::vector<char> &raw, int64_t h, std::string f[4]) {
    const int64_t n = (int64_t) raw.size();
    int64_t ls[4], le[4], p = h;
    for (int k = 0; k < 4; ++k) {
        const void *q = p < n ? memchr(raw.data() + p, '\n', (size_t) (n - p)) : nullptr;
        ls[k] = p; le[k] = q ? (const char *) q - raw.data() : n; p = le[k] + 1;
    }
    int64_t e0 = le[0], e1 = le[1], e3 = le[3];
    if (e0 > ls[0] && raw[e0 - 1] == '\r') --e0;
    if (e1 > ls[1] && raw[e1 - 1] == '\r') --e1;
    if (e3 > ls[3] && raw[e3 - 1] == '\r') --e3;
    if (e0 <= ls[0] || raw[ls[0]] != '@' || le[2] <= ls[2] || raw[ls[2]] != '+' || e3 - ls[3] != e1 - ls[1]) return false;
    int64_t ne = ls[0] + 1;
    while (ne < e0 && raw[ne] != ' ' && raw[ne] != '\t') ++ne;
    int64_t cb = ne + 1, ce = le[0];
    if (ne >= e0) cb = ce = 0;
    else if (ce - cb > 1 && raw[ce - 1] == '\r') --ce;
    int64_t nl = ne - (ls[0] + 1);
    if (nl > 2 && raw[ls[0] + nl - 1] == '/' && raw[ls[0] + nl] >= '0' && raw[ls[0] + nl] <= '9') nl -= 2;
    f[0].assign(&raw[ls[0] + 1], (size_t) nl); f[1].assign(raw.data() + cb, (size_t) (ce - cb));
    f[2].assign(raw.data() + ls[1], (size_t) (e1 - ls[1])); f[3].assign(raw.data() + ls[3], (size_t) (e3 - ls[3]));
    return true;
}

int main(int argc, char **argv) {
    if (argc < 2) return 1;
    FILE *fp = fopen(argv[1], "rb");
    if (!fp) return 1;
    std::vector<char> raw;
    { char b[65536]; size_t r; while ((r = fread(b, 1, sizeof b, fp)) > 0) raw.insert(raw.end(), b, b + r); fclose(fp); }
    const int64_t n = (int64_t) raw.size();
    std::vector<int32_t> nl, hp;
    for (int64_t i = 0; i < n; ++i) { if (raw[i] == '\n') nl.push_back((int32_t) i); if (raw[i] == '>' || raw[i] == '@') hp.push_back((int32_t) i); }
    SeqTableSrc s = { raw.data(), n, nl.data(), (int) nl.size(), hp.data(), (int) hp.size(), 0 };
    // candidates
    std::vector<int32_t> cand;
    for (size_t k = 0; k <= nl.size(); ++k) {
        const int32_t c = (int32_t) s.hdr(k == 0 ? 0 : (int64_t) nl[k - 1] + 1);
        if (c < n && (cand.empty() || cand.back() != c)) cand.push_back(c);
    }
    const int K = (int) cand.size();
    std::vector<int32_t> nxt((size_t) K + 1, K);
    std::vector<SeqRec> rec((size_t) K);
    for (int i = 0; i < K; ++i) {
        s.k = 0;
        rec[i] = seq_record(s, cand[i], SeqNullSink());
        if (rec[i].status == SEQ_OK && rec[i].next < n) {
            const int j = (int) (std::lower_bound(cand.begin() + i + 1, cand.end(), (int32_t) rec[i].next) - cand.begin());
            if (j >= K || cand[j] != rec[i].next) { printf("X next %d is no candidate\n", i); return 2; }
            nxt[i] = j;
        }
    }
    // pointer doubling
    int T = 1; while ((1LL << T) <= K) ++T;
    std::vector<std::vector<int32_t>> J(T, nxt);
    for (int t = 1; t < T; ++t) for (int i = 0; i <= K; ++i) J[t][i] = J[t - 1][J[t - 1][i]];
    std::vector<uint8_t> mark((size_t) K + 1, 0);
    if (K) mark[0] = 1;
    for (int t = T - 1; t >= 0; --t) for (int i = 0; i <= K; ++i) if (mark[i]) mark[J[t][i]] = 1;
    std::vector<int> recs;
    for (int i = 0; i < K; ++i) if (mark[i] && rec[i].status != SEQ_NONE) recs.push_back(i);
    for (size_t r = 0; r < recs.size(); ++r) if (rec[recs[r]].status == SEQ_BAD) { printf("E %zu\n", r); return 0; }
    printf("R %zu\n", recs.size());
    long long n_simple = 0, n_bad = 0;
    for (int i : recs) {
        std::string sq, ql;
        s.k = 0;
        const SeqRec r = seq_record(s, cand[i], StrSink{ raw.data(), &sq, &ql });
        sq.resize((size_t) r.l_seq); ql.resize((size_t) r.l_qual);
        field(raw.data() + r.name_beg, r.name_len);
        if (r.cmt_len) field(raw.data() + r.cmt_beg, r.cmt_len); else fputs("-1:", stdout);
        field(sq.data(), (int64_t) sq.size());
        if (r.l_qual) field(ql.data(), (int64_t) ql.size()); else fputs("-1:", stdout);
        putchar('\n');
        if (r.simple) {
            ++n_simple;
            std::string f[4];
            const std::string want[4] = { std::string(raw.data() + r.name_beg, (size_t) r.name_len), std::string(raw.data() + r.cmt_beg, (size_t) r.cmt_len), sq, ql };
            // the kernel's path always has qualities: kseq must have them too (l_qual > 0)
            if (!spans_rules(raw, cand[i], f) || f[0] != want[0] || f[1] != want[1] || f[2] != want[2] || f[3] != want[3] || r.l_qual == 0) ++n_bad;
        }
    }
    printf("S %lld %lld\n", n_simple, n_bad);
    return 0;
}

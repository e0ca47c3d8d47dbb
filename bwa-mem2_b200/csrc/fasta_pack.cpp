// fasta_pack.cpp — bm2_fasta_pack: the first step of bm2_index, bns_fasta2bntseq(fp, prefix, 1) (reference src/bntseq.cpp:249-356): the
// records of a FASTA (or FASTQ) file, plain or gzip, packed into <prefix>.pac with the contigs in <prefix>.ann and the runs of ambiguous bases
// in <prefix>.amb.  Host code: the packing is one sequential pass whose random draws follow file order.
//
// Records are read by seq_record (seq_grammar.cuh), the restatement of kseq_read that bm2_mem uses, with the name as kseq returns it (no
// trim_readno: bseq_read applies that, the index builder does not).  Per base, as add1 does:
//   code   A C G T in either case -> 0-3, every other byte -> 4 (nst_nt4_table's rule)
//   hole   a byte of code 4 opens a new hole unless it equals the previous byte of the same contig (NNnn is two holes, NAN two); the previous
//          byte starts at 0 for each contig
//   base   code 4 becomes lrand48() & 3, drawn in file order after srand48(11) - here nrand48 on a private state equal to the one srand48(11)
//          sets, so the caller's drand48 state is untouched
#include "bm2_b200.h"
#include "seq_grammar.cuh"
#include "read_input.h"
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <vector>

void bm2_set_error(struct bm2_ctx *ctx, const std::string &msg);

namespace {

// nst_nt4_table's rule, written out: A C G T in either case are 0-3, every other byte is 4
struct Nt4 {
    uint8_t t[256];
    Nt4() {
        for (int i = 0; i < 256; ++i) t[i] = 4;
        const char *acgt = "ACGT";
        for (int c = 0; c < 4; ++c) { t[(unsigned char) acgt[c]] = (uint8_t) c; t[(unsigned char) acgt[c] + 32] = (uint8_t) c; }
    }
};

// the bytes seq_record keeps: each line written at the current length of the string (seq_grammar.cuh)
struct StringSink {
    std::string *s; const char *raw;
    void seq(int64_t p, int64_t k, int64_t at) const { s->resize((size_t) (at + k)); memcpy(&(*s)[(size_t) at], raw + p, (size_t) k); }
    void qual(int64_t, int64_t, int64_t) const {}
};

struct Hole { int64_t offset; int32_t len; char amb; };
struct Ann { std::string name, anno; int64_t offset; int32_t len, n_ambs; };

bool fail(const std::string &m) { bm2_set_error(nullptr, "bm2_fasta_pack: " + m); return false; }

bool write_all(const std::string &path, const void *p, size_t n) {
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = fwrite(p, 1, n, f) == n;
    return fclose(f) == 0 && ok;
}

}  // namespace

extern "C" int bm2_fasta_pack(const char *path, const char *prefix, bm2_fasta_pack_stats *stats) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!path || !prefix) return !fail("NULL argument");
    std::vector<char> buf;
    if (!read_file(path, buf)) return !fail(std::string("cannot read ") + path);
    static const Nt4 nt4;
    const SeqHostSrc src = { buf.data(), (int64_t) buf.size() };
    std::vector<uint8_t> pac;
    std::vector<Ann> anns; std::vector<Hole> holes;
    int64_t l_pac = 0;
    unsigned short xsubi[3] = { 0x330E, 11, 0 };     // srand48(11)
    std::string seq;
    for (int64_t h = src.hdr(0);;) {
        seq.clear();
        const SeqRec r = seq_record(src, h, StringSink{ &seq, buf.data() });
        if (r.status == SEQ_NONE) break;
        if (r.status == SEQ_BAD) {
            char m[160];
            snprintf(m, sizeof m, "malformed record %zu (a '+' line without qualities, or qualities of another length)", anns.size() + 1);
            return !fail(m);
        }
        seq.resize((size_t) r.l_seq);
        Ann a;
        a.name.assign(buf.data() + r.name_beg, (size_t) r.name_full_len);
        a.anno = r.cmt_len > 0 ? std::string(buf.data() + r.cmt_beg, (size_t) r.cmt_len) : std::string("(null)");
        a.offset = l_pac; a.len = r.l_seq; a.n_ambs = 0;
        pac.resize((size_t) ((l_pac + r.l_seq + 3) >> 2), 0);
        int lasts = 0;
        for (int32_t i = 0; i < r.l_seq; ++i) {
            const char ch = seq[(size_t) i];
            int c = nt4.t[(unsigned char) ch];
            if (c >= 4) {
                if (lasts == ch) { if (!holes.empty()) ++holes.back().len; }      // the run goes on (add1 lengthens its last hole)
                else { holes.push_back(Hole{ a.offset + i, 1, ch }); ++a.n_ambs; }
                c = (int) (nrand48(xsubi) & 3);
            }
            lasts = ch;
            pac[(size_t) (l_pac >> 2)] |= (uint8_t) (c << ((~l_pac & 3) << 1));
            ++l_pac;
        }
        anns.push_back(std::move(a));
        h = r.next;
    }
    if (l_pac == 0) return !fail(std::string("no sequence in ") + path + " (an empty reference cannot be indexed)");
    if (anns.size() > (size_t) INT_MAX) return !fail("more than INT_MAX sequences");
    // .pac: the packed bases, then a 0 byte when l_pac % 4 == 0, then l_pac % 4 (src/bntseq.cpp:338-351)
    if (l_pac % 4 == 0) pac.push_back(0);
    pac.push_back((uint8_t) (l_pac % 4));
    const std::string p(prefix);
    if (!write_all(p + ".pac", pac.data(), pac.size())) return !fail("cannot write " + p + ".pac");
    // .ann and .amb: bns_dump (src/bntseq.cpp:73-104)
    std::string ann = std::to_string(l_pac) + " " + std::to_string(anns.size()) + " 11\n";
    for (const Ann &a : anns)
        ann += "0 " + a.name + " " + a.anno + "\n" + std::to_string(a.offset) + " " + std::to_string(a.len) + " " + std::to_string(a.n_ambs) + "\n";
    std::string amb = std::to_string(l_pac) + " " + std::to_string(anns.size()) + " " + std::to_string(holes.size()) + "\n";
    for (const Hole &q : holes) amb += std::to_string(q.offset) + " " + std::to_string(q.len) + " " + q.amb + "\n";
    if (!write_all(p + ".ann", ann.data(), ann.size())) return !fail("cannot write " + p + ".ann");
    if (!write_all(p + ".amb", amb.data(), amb.size())) return !fail("cannot write " + p + ".amb");
    if (stats) {
        stats->l_pac = l_pac; stats->n_seqs = (int64_t) anns.size(); stats->n_holes = (int64_t) holes.size();
        stats->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    }
    return 0;
}

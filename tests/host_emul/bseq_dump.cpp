// bseq_dump.cpp — TEST ONLY: the records and chunks the unmodified reference reads from its input, through its own kseq_init +
// bseq_read_orig, declared by its own headers (compiled with -I <reference>/src) and linked from oracle/_ref/<isa>/libbwa.a.
//   bseq_dump <chunk_size> <file1|-> [file2]
// Output, per chunk: "C <n>\n", then per record four fields, each "<len>:<bytes>" or "-1:" when the reference leaves it NULL (comment,
// qualities): name, comment, sequence, qualities, then "\n".
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <zlib.h>
#include "bwa.h"
#include "kseq.h"
KSEQ_DECLARE(gzFile)

static void field(const char *s) {
    if (!s) { fputs("-1:", stdout); return; }
    const size_t n = strlen(s);
    printf("%zu:", n);
    fwrite(s, 1, n, stdout);
}

int main(int argc, char **argv) {
    if (argc < 3) { fprintf(stderr, "usage: bseq_dump <chunk_size> <file1|-> [file2]\n"); return 1; }
    const int64_t chunk = atoll(argv[1]);
    gzFile f1 = strcmp(argv[2], "-") ? gzopen(argv[2], "r") : gzdopen(0, "r");
    gzFile f2 = argc > 3 ? gzopen(argv[3], "r") : nullptr;
    if (!f1 || (argc > 3 && !f2)) { fprintf(stderr, "bseq_dump: cannot open the input\n"); return 1; }
    kseq_t *k1 = kseq_init(f1), *k2 = f2 ? kseq_init(f2) : nullptr;
    for (;;) {
        int n = 0; int64_t size = 0;
        bseq1_t *seqs = bseq_read_orig(chunk, &n, k1, k2, &size);
        if (n == 0) { free(seqs); break; }
        printf("C %d\n", n);
        for (int i = 0; i < n; ++i) {
            field(seqs[i].name); field(seqs[i].comment); field(seqs[i].seq); field(seqs[i].qual); putchar('\n');
            free(seqs[i].name); free(seqs[i].comment); free(seqs[i].seq); free(seqs[i].qual);
        }
        free(seqs);
    }
    return 0;
}

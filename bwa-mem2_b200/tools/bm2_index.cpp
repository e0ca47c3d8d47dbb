// bm2_index — `bwa-mem2 index` (bwa_index + bwa_idx_build, reference src/bwtindex.cpp:43-80) over the C ABI of libbm2b200.so:
//
//   bm2_index [-p prefix] <in.fasta>
//
// Same usage, default prefix (the input path) and exit codes as the reference: 1 with the usage line when no input is given, 1 on an unknown
// option.  Writes the five files of the reference, byte for byte: <prefix>.pac .ann .amb (bm2_fasta_pack, on the host) and .0123
// .bwt.2bit.64 (bm2_index_build, on GPU 0, with the working buffers sized from the free device memory).  A malformed record, an input without
// bases and a build that does not fit the device are errors with a message and exit code 1 (the reference stops silently or asserts).
// The stage times, the peak device bytes and the refinement rounds go to stderr as one JSON line.
#include "bm2_b200.h"
#include <cstdio>
#include <cstring>
#include <unistd.h>

int main(int argc, char **argv) {
    const char *prefix = nullptr;
    int c;
    while ((c = getopt(argc, argv, "p:")) >= 0) {
        if (c == 'p') prefix = optarg;
        else return 1;
    }
    if (optind + 1 > argc) {
        fprintf(stderr, "Usage: bm2_index [-p prefix] <in.fasta>\n");
        return 1;
    }
    const char *fa = argv[optind];
    if (!prefix) prefix = fa;
    bm2_fasta_pack_stats ps;
    if (bm2_fasta_pack(fa, prefix, &ps)) { fprintf(stderr, "[E::bm2_index] %s\n", bm2_last_error(nullptr)); return 1; }
    bm2_index_build_stats bs;
    if (bm2_index_build(0, prefix, 0, &bs)) { fprintf(stderr, "[E::bm2_index] %s\n", bm2_last_error(nullptr)); return 1; }
    fprintf(stderr, "{\"l_pac\": %lld, \"n_seqs\": %lld, \"n_holes\": %lld, \"pack_s\": %.3f, \"load_s\": %.3f, \"pass1_s\": %.3f, \"refine_s\": %.3f, "
                    "\"emit_s\": %.3f, \"build_s\": %.3f, \"peak_device_bytes\": %lld, \"rounds\": %d, \"groups\": %d, \"pieces\": %lld, \"windows\": %d, "
                    "\"unresolved\": %lld, \"unresolved_on_host\": %d}\n",
            (long long) ps.l_pac, (long long) ps.n_seqs, (long long) ps.n_holes, ps.seconds, bs.load_s, bs.pass1_s, bs.refine_s, bs.emit_s, bs.total_s,
            (long long) bs.peak_device_bytes, bs.rounds, bs.groups, (long long) bs.pieces, bs.windows, (long long) bs.unresolved, bs.unresolved_on_host);
    return 0;
}

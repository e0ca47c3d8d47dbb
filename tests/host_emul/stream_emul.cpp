// stream_emul.cpp — TEST ONLY: bm2_mem's chunker (chunk_stream, bwa-mem2_b200/csrc/read_input.h) over a fake source that delivers at most
// k bytes per read (k = 0: the whole file in one read), with a tiny starting window so that every refill, compaction and growth path runs.
//   stream_emul <K> <k> <file1> [file2]
// Output: one line per chunk as `bm2_mem --dump-chunks` prints it, or "E <message>" at an error.
#include "read_input.h"
#include <cstdio>
#include <vector>

struct FakeSource : ByteSource {
    std::vector<char> data; size_t at = 0, k = 0;
    int64_t read(char *dst, size_t cap) override {
        const size_t n = std::min({ cap, data.size() - at, k ? k : data.size() });
        memcpy(dst, data.data() + at, n); at += n;
        return (int64_t) n;
    }
};

static bool load(const char *path, std::vector<char> &d) {
    FILE *f = fopen(path, "rb");
    if (!f) return false;
    char b[65536]; size_t r;
    while ((r = fread(b, 1, sizeof b, f)) > 0) d.insert(d.end(), b, b + r);
    fclose(f);
    return true;
}

int main(int argc, char **argv) {
    if (argc < 4) return 1;
    const long long K = atoll(argv[1]);
    FakeSource s[2];
    for (int i = 0; i + 3 < argc && i < 2; ++i) { s[i].k = (size_t) atoll(argv[2]); if (!load(argv[3 + i], s[i].data)) return 1; }
    std::string err;
    const long long n = chunk_stream(s[0], argc > 4 ? &s[1] : nullptr, K, [&](Chunk &&ck) {
        printf("{\"first_read\": %lld, \"offset1\": %lld, \"bytes1\": %zu, \"offset2\": %lld, \"bytes2\": %zu, \"simple\": %s}\n", ck.first_read,
               (long long) ck.off1, ck.n1, (long long) ck.off2, ck.n2, ck.simple ? "true" : "false");
        // the chunk's own copy holds the input's bytes
        if (memcmp(ck.c1, s[0].data.data() + ck.off1, ck.n1) || (ck.n2 && memcmp(ck.c2, s[1].data.data() + ck.off2, ck.n2))) printf("X bytes\n");
    }, err, 64);
    if (n < 0) printf("E %s\n", err.c_str());
    return 0;
}

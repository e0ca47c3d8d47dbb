"""The input grammar of bm2_seq_encode and bm2_mem (bwa-mem2_b200/csrc/seq_grammar.cuh) against the unmodified reference, without a GPU.

The reference side, tests/host_emul/bseq_dump.cpp, is compiled against the reference's own headers, linked against oracle/_ref/<isa>/libbwa.a,
and reads its input through the reference's kseq_init + bseq_read_orig, dumping every chunk's records.  tests/golden/seq_corpus_bseq.json holds
the SHA-256 of each corpus file's records as that dump gives them (sequences as nt4 codes, seq_corpus.digest), so that the record checks
also run where the reference is absent, and the GPU test compares with it; test_golden_digests_are_the_reference keeps it honest.  Our side:
- tests/host_emul/seq_emul.cpp runs bm2_seq_encode's resolution on the host (candidates, next(), pointer doubling, the record walk into a sink)
  over the same grammar: every record must equal the reference's, and on every "simple" record fastq_spans_kernel's rules must give the same
  record (the condition under which bm2_mem sends a chunk through bm2_fastq_encode);
- `bm2_mem --dump-chunks` runs the program's chunker: its chunks must hold the reference's records chunk for chunk, each chunk's bytes parsed
  on their own giving that chunk's records, at several chunk sizes, single-end and paired, from files and from standard input (plain, gzip)."""
import gzip, json, os, subprocess
import pytest
import seq_corpus as sc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
CSRC = os.path.join(ROOT, "bwa-mem2_b200", "csrc")
HOST = os.path.join(ROOT, "tests", "host_emul")
CORPUS = sc.corpus()
CHUNKS = [1, 2000, 100_000_000]
REF = os.environ.get("REF", "/root/reference")           # the reference's sources, as oracle/Makefile names them
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "seq_corpus_bseq.json")))


@pytest.fixture(scope="module")
def tools(tmp_path_factory):
    d = tmp_path_factory.mktemp("seq_input")
    emul = str(d / "seq_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-w", "-I" + CSRC, os.path.join(HOST, "seq_emul.cpp"), "-o", emul])
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    ref = os.path.join(ROOT, "oracle", "_ref")
    dump = None
    if os.path.exists(os.path.join(ref, isa, "libbwa.a")) and os.path.exists(os.path.join(REF, "src", "bwa.h")):
        dump = str(d / "bseq_dump")
        subprocess.check_call(["g++", "-O2", "-w", "-I" + os.path.join(REF, "src"), "-I" + os.path.join(REF, "ext", "safestringlib", "include"),
                               os.path.join(HOST, "bseq_dump.cpp"), os.path.join(ref, isa, "libbwa.a"),
                               os.path.join(ref, "libsafestring.a"), "-lz", "-lpthread", "-lm", "-o", dump])
    files = {}
    for name, (a, b) in CORPUS.items():
        files[name] = []
        for k, data in enumerate((a, b)):
            if data is not None:
                p = d / ("%s_%d" % (name, k)); p.write_bytes(data); files[name].append(str(p))
    return dict(d=d, emul=emul, dump=dump, files=files)


def _bseq(tools, chunk, paths, stdin=None):
    if tools["dump"] is None:
        pytest.skip("the reference or oracle/_ref is absent")
    o = subprocess.run([tools["dump"], str(chunk)] + paths, input=stdin, capture_output=True, timeout=120)
    assert o.returncode == 0, o.stderr
    return sc.parse_dump(o.stdout)[0]


def _emul(tools, data):
    p = tools["d"] / "emul_in"
    p.write_bytes(data)
    o = subprocess.run([tools["emul"], str(p)], capture_output=True, timeout=120)
    assert o.returncode == 0, o.stdout[-500:]
    chunks, extra = sc.parse_dump(o.stdout)
    return (chunks[0] if chunks else None), extra


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_golden_digests_are_the_reference(tools, name):
    recs = [r for c in _bseq(tools, 1 << 40, tools["files"][name]) for r in c]
    assert {"records": len(recs), "sha256": sc.digest(sc.encoded(recs))} == GOLDEN[name]


@pytest.mark.parametrize("name", sorted(n for n in CORPUS if CORPUS[n][1] is None))
def test_records_equal_the_reference(tools, name):
    data = CORPUS[name][0]
    got, extra = _emul(tools, data)
    assert "E" not in extra
    assert len(got) == GOLDEN[name]["records"] > 0
    assert sc.digest(sc.encoded(got)) == GOLDEN[name]["sha256"]
    if tools["dump"] is not None:                  # the raw bytes too (the digest holds the sequences as codes), record by record
        want = [r for c in _bseq(tools, 1 << 40, tools["files"][name]) for r in c]
        for i, (g, w) in enumerate(zip(got, want)):
            assert g == w, (i, g, w)
    n_simple, n_mismatch = extra["S"]
    assert n_mismatch == 0
    if name == "fq_4line":
        assert n_simple == len(got)
    if name.startswith("fa_"):
        assert n_simple == 0


@pytest.mark.parametrize("name", sorted(sc.MALFORMED))
def test_malformed_record_is_an_error_naming_it(tools, name):
    data, index = sc.MALFORMED[name]
    _, extra = _emul(tools, data)
    assert extra["E"] == [index]
    p = tools["d"] / ("bad_" + name); p.write_bytes(data)
    o = subprocess.run([TOOL, "--dump-chunks", "idx", str(p)], capture_output=True, text=True, timeout=60)
    assert o.returncode != 0 and ("malformed record %d of the 1st file" % index) in o.stderr
    if tools["dump"] is not None:                  # the reference stops there without a message: the records before it
        assert sum(len(c) for c in _bseq(tools, 1 << 40, [str(p)])) == index


def _dump_chunks(paths, K, extra=(), stdin=None):
    o = subprocess.run([TOOL, "--dump-chunks", "-K", str(K)] + list(extra) + ["idx"] + paths, input=stdin, capture_output=True, timeout=120)
    assert o.returncode == 0, o.stderr
    return [json.loads(l) for l in o.stdout.decode().splitlines()]


@pytest.mark.parametrize("K", CHUNKS)
@pytest.mark.parametrize("name", sorted(CORPUS))
def test_chunks_equal_the_reference(tools, name, K):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    paths = tools["files"][name]
    want = _bseq(tools, K, paths)
    got = _dump_chunks(paths, K)
    assert len(got) == len(want)
    data = [CORPUS[name][0], CORPUS[name][1]]
    paired = len(paths) == 2
    for ck, wc in zip(got, want):
        piece = [data[k][ck["offset%d" % (k + 1)]:ck["offset%d" % (k + 1)] + ck["bytes%d" % (k + 1)]] for k in range(len(paths))]
        parsed = [_emul(tools, b) for b in piece]
        per = [p[0] for p in parsed]
        recs = [r for pair in zip(*per) for r in pair] if paired else per[0]
        assert recs == wc
        if ck["simple"]:                           # bm2_fastq_encode takes the bytes whole: four lines per record, every record simple
            for b, (rs, extra) in zip(piece, parsed):
                assert b.count(b"\n") + (not b.endswith(b"\n")) == 4 * len(rs)
                assert extra["S"] == [len(rs), 0]
    if name in ("fq_4line", "header_at_eof"):
        assert all(c["simple"] for c in got)
    if name == "header_at_eof":                    # the '@' at the end of the file is in no chunk
        assert sum(c["bytes1"] for c in got) == len(data[0]) - 1
    elif name in ("fa_60", "fq_wrapped_at", "mixed", "corners", "pe_fa_60"):
        assert not all(c["simple"] for c in got)


@pytest.mark.parametrize("how", ["plain", "gzip", "gzip_two_members"])
def test_standard_input(tools, how):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    data = CORPUS["mixed"][0]
    stdin = data if how == "plain" else gzip.compress(data) if how == "gzip" else gzip.compress(data[:5000]) + gzip.compress(data[5000:])
    want = _dump_chunks(tools["files"]["mixed"], 2000)
    assert _dump_chunks(["-"], 2000, stdin=stdin) == want
    gz = tools["d"] / "mixed.gz"; gz.write_bytes(stdin)
    assert _dump_chunks([str(gz)], 2000) == want
    assert _bseq(tools, 2000, ["-"], stdin=stdin) == _bseq(tools, 2000, tools["files"]["mixed"])


def test_sam_quality_star_where_absent(pkg):
    """bm2_sam_format_ex prints QUAL '*' for exactly the reads whose qual_present is 0"""
    import numpy as np
    capi = pkg.capi
    n, L = 4, 6
    codes = np.tile(np.arange(L, dtype=np.uint8) % 4, n); offs = (np.arange(n + 1) * L).astype(np.int64)
    quals = np.frombuffer(b"ABCDEF" * n, np.uint8)
    recs = np.zeros(n, capi.SAM_REC_DT)
    recs["read"] = np.arange(n); recs["flag"] = 4; recs["rid"] = -1; recs["rnext"] = -1; recs["score"] = -1; recs["sub"] = -1; recs["reg"] = -1
    qp = np.array([1, 0, 1, 0], np.uint8)
    text = capi.sam_format(recs, np.zeros(0, capi.SAM_XA_DT), np.zeros(0, np.uint32), np.zeros(0, np.uint8), codes, offs, ["c"],
                           read_names=["a", "b", "c", "d"], quals=quals, qual_present=qp).decode()
    cols = [l.split("\t") for l in text.splitlines()]
    assert [c[10] for c in cols] == ["ABCDEF", "*", "ABCDEF", "*"]
    assert all(c[9] == "ACGTAC" for c in cols)
    base = capi.sam_format(recs, np.zeros(0, capi.SAM_XA_DT), np.zeros(0, np.uint32), np.zeros(0, np.uint8), codes, offs, ["c"],
                           read_names=["a", "b", "c", "d"], quals=quals).decode()
    assert [l.split("\t")[10] for l in base.splitlines()] == ["ABCDEF"] * 4

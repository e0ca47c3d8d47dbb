"""The streaming input of bm2_mem (bwa-mem2_b200/csrc/read_input.h), without a GPU.

- tests/host_emul/stream_emul.cpp runs bm2_mem's chunker (read_input.h chunk_stream) over a fake source that delivers 1, 7 or 4096 bytes per
  read: its chunks equal the whole-input chunks on every corpus file, single-end and paired, at every chunk size.
- bm2_mem --dump-chunks streams: BGZF files (written by the small BGZF writer below), BGZF mixed with plain gzip members and bytes after
  the last member cut like the plain file; an input cut inside a member read as far as it goes (gzread's rule, the reference's too),
  by bm2_mem and by bm2_fasta_pack; a corrupt member an error; standard input answered before it ends, and its memory
  bounded far below the size of its input."""
import gzip, json, os, struct, subprocess, threading, zlib
import numpy as np
import pytest
import seq_corpus as sc
from test_seq_input_cpu import CHUNKS, CORPUS, TOOL, _bseq, _dump_chunks, tools  # noqa: F401  (tools is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bwa-mem2_b200", "csrc")
HOST = os.path.join(ROOT, "tests", "host_emul")
_ISA = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
REF_INDEX = os.path.join(ROOT, "oracle", "_ref", _ISA, "bwa-mem2")      # the unmodified reference, where built
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def bgzf_member(payload: bytes, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=()) -> bytes:
    """one BGZF member: gzip header with the BC subfield (BSIZE = member length - 1), raw deflate, CRC32, ISIZE; flushes: payload offsets
    where a Z_FULL_FLUSH ends a block"""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    body, at = b"", 0
    for f in list(flushes) + [len(payload)]:
        body += c.compress(payload[at:f]) + (c.flush(zlib.Z_FULL_FLUSH) if f < len(payload) else b"")
        at = f
    body += c.flush()
    hdr = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00"
    return hdr + struct.pack("<H", len(hdr) + 2 + len(body) + 8 - 1) + body + struct.pack("<II", zlib.crc32(payload), len(payload))


def bgzf(data: bytes, level=6, block=65280, eof=True, strategy=zlib.Z_DEFAULT_STRATEGY) -> bytes:
    """data as BGZF (bgzip's block size), with the EOF block"""
    return b"".join(bgzf_member(data[i:i + block], level, strategy) for i in range(0, len(data), block)) + (BGZF_EOF if eof else b"")


@pytest.fixture(scope="module")
def stream_emul(tmp_path_factory):
    d = tmp_path_factory.mktemp("stream")
    exe = str(d / "stream_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-w", "-I" + CSRC, os.path.join(HOST, "stream_emul.cpp"), "-o", exe, "-lz"])
    files = {}
    for name, (a, b) in list(CORPUS.items()) + [("bad_" + k, (v[0], None)) for k, v in sc.MALFORMED.items()]:
        files[name] = []
        for k, data in enumerate((a, b)):
            if data is not None:
                p = d / ("%s_%d" % (name, k)); p.write_bytes(data); files[name].append(str(p))
    return exe, files


@pytest.mark.parametrize("name", sorted(CORPUS) + sorted("bad_" + k for k in sc.MALFORMED))
def test_streamed_chunks_equal_whole_input_chunks(stream_emul, name):
    exe, files = stream_emul
    for K in CHUNKS:
        def run(k):
            o = subprocess.run([exe, str(K), str(k)] + files[name], capture_output=True, text=True, timeout=300)
            assert o.returncode == 0 and "X bytes" not in o.stdout
            return o.stdout
        whole = run(0)
        assert whole
        if name.startswith("bad_"):
            assert whole.splitlines()[-1] == "E malformed record %d of the 1st file (a '+' line without qualities, or qualities of another length)" \
                % sc.MALFORMED[name[4:]][1]
        for k in (1, 7, 4096):
            assert run(k) == whole, (K, k)
        if not name.startswith("bad_") and os.path.exists(TOOL):       # and the program's own chunks, from the whole file
            assert [json.loads(l) for l in whole.splitlines()] == _dump_chunks(files[name], K)


@pytest.mark.parametrize("how", ["bgzf", "bgzf_then_gzip", "gzip_then_bgzf", "bgzf_trailing_bytes"])
def test_dump_chunks_of_bgzf_files_equal_the_plain_file(tmp_path, how):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    data = CORPUS["mixed"][0] * 3
    cut = len(data) // 2
    enc = {"bgzf": bgzf(data, block=5000),
           "bgzf_then_gzip": bgzf(data[:cut], block=3000, eof=False) + gzip.compress(data[cut:]),
           "gzip_then_bgzf": gzip.compress(data[:cut]) + bgzf(data[cut:], block=7000),
           "bgzf_trailing_bytes": bgzf(data, block=5000) + b"trailing bytes"}[how]
    plain = tmp_path / "plain.fq"; plain.write_bytes(data)
    gz = tmp_path / "in.gz"; gz.write_bytes(enc)
    for K in (2000, 100_000_000):
        want = _dump_chunks([str(plain)], K)
        assert _dump_chunks([str(gz)], K) == want
        assert _dump_chunks(["-"], K, stdin=enc) == want


def _gzread(enc: bytes) -> bytes:
    """what gzread hands kseq: every member inflated, a member cut by the end of the input as far as it goes, bytes after the last member
    ignored"""
    out = b""
    while enc[:2] == b"\x1f\x8b":
        d = zlib.decompressobj(31)
        out += d.decompress(enc)
        if not d.eof:
            break
        enc = d.unused_data
    return out


def _truncations():
    # FASTA: a record cut anywhere is still a record, so the cut input has chunks to compare
    reads_fa = sc.fasta(sc.records(np.random.default_rng(8), 600, 50, 400), 70, b"\r\n")
    fa = sc.fasta(sc.records(np.random.default_rng(9), 200, 50, 400, b"ACGTN"), 60)
    whole = bgzf(reads_fa, block=5000)
    two = gzip.compress(reads_fa[:30000], mtime=0) + gzip.compress(reads_fa[30000:], mtime=0)
    return {
        "gzip_body": (gzip.compress(reads_fa, mtime=0)[:-100], reads_fa),
        "gzip_trailer": (gzip.compress(reads_fa, mtime=0)[:-3], reads_fa),
        "second_member_body": (two[:len(two) - 2000], reads_fa),
        "second_member_header": (two[:len(gzip.compress(reads_fa[:30000], mtime=0)) + 5], reads_fa),
        "bgzf_mid": (whole[:len(whole) // 2 + 77], reads_fa),
        "fasta_gzip_body": (gzip.compress(fa, mtime=0)[:-500], fa),
    }


@pytest.mark.parametrize("name", sorted(_truncations()))
def test_truncated_gzip_reads_as_far_as_it_goes(pkg, tools, tmp_path, name):
    """a gzip input cut inside a member is read as gzread reads it - the bytes inflated so far, then the end - by bm2_mem (files and standard
    input, with a warning) and by bm2_fasta_pack, as the reference reads it"""
    enc, text = _truncations()[name]
    want = _gzread(enc)
    assert 0 < len(want) <= len(text) and text.startswith(want)
    gz = tmp_path / "cut.gz"; gz.write_bytes(enc)
    plain = tmp_path / "plain"; plain.write_bytes(want)
    if os.path.exists(TOOL):
        for K in (2000, 100_000_000):
            chunks = _dump_chunks([str(plain)], K)
            assert chunks and _dump_chunks([str(gz)], K) == chunks
            assert _dump_chunks(["-"], K, stdin=enc) == chunks
        o = subprocess.run([TOOL, "--dump-chunks", "idx", str(gz)], capture_output=True, text=True, timeout=60)
        assert o.returncode == 0 and "ends inside a gzip member" in o.stderr
    if tools["dump"] is not None:                  # the reference reads the same records from the cut file
        assert _bseq(tools, 2000, [str(gz)]) == _bseq(tools, 2000, [str(plain)])
    if name.startswith("fasta"):
        pkg.capi.fasta_pack(str(gz), str(tmp_path / "cut")); pkg.capi.fasta_pack(str(plain), str(tmp_path / "plain"))
        ref = None
        if os.path.exists(REF_INDEX):
            # the reference packs what gzread gave, writes .pac / .ann / .amb, then stops at gzclose's Z_BUF_ERROR ("[gzclose] buffer error")
            subprocess.run([REF_INDEX, "index", "-p", str(tmp_path / "ref"), str(gz)], capture_output=True, timeout=300)
            ref = "ref"
        for ext in (".pac", ".ann", ".amb"):
            got = (tmp_path / ("cut" + ext)).read_bytes()
            assert got == (tmp_path / ("plain" + ext)).read_bytes(), ext
            if ref:
                assert got == (tmp_path / (ref + ext)).read_bytes(), ext


def test_corrupt_gzip_member_is_an_error(tmp_path):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    enc = bytearray(bgzf(CORPUS["fq_4line"][0], block=5000, eof=False))
    enc[-8] ^= 1                                   # the last member's CRC32: zlib's "incorrect data check", gzread returns -1
    p = tmp_path / "bad.gz"; p.write_bytes(bytes(enc))
    o = subprocess.run([TOOL, "--dump-chunks", "idx", str(p)], capture_output=True, text=True, timeout=60)
    assert o.returncode == 2 and "cannot read the input files" in o.stderr


def test_standard_input_streams():
    """the first chunk is cut and printed while the writer still holds back the rest of the input"""
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    data = CORPUS["fq_4line"][0]
    for enc in (data, gzip.compress(data)):
        p = subprocess.Popen([TOOL, "--dump-chunks", "-K", "2000", "idx", "-"], stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        half = len(enc) // 2
        p.stdin.write(enc[:half]); p.stdin.flush()
        first = []
        t = threading.Thread(target=lambda: first.append(p.stdout.readline()), daemon=True)
        t.start(); t.join(timeout=30)
        ok = bool(first) and first[0].startswith(b"{")
        p.stdin.write(enc[half:]); p.stdin.close()
        rest = p.stdout.read(); p.wait(timeout=60)
        assert ok, "no chunk before the end of the input"
        assert p.returncode == 0
        assert [json.loads(l) for l in (first[0] + rest).decode().splitlines()] == _dump_chunks(["-"], 2000, stdin=data)


# runs argv[2:] from a small process and writes its peak RSS (KiB) to argv[1]: a child forked straight from the test process would count the
# test process's pages in its ru_maxrss until it execs
_RSS = "import os, subprocess, sys; p = subprocess.Popen(sys.argv[2:]); _, s, ru = os.wait4(p.pid, 0); open(sys.argv[1], 'w').write(str(ru.ru_maxrss)); sys.exit(os.waitstatus_to_exitcode(s))"


def peak_rss(argv, feed, rss_path, stdout=subprocess.PIPE):
    """argv with feed() writing its standard input: (exit code, standard output, standard error, peak RSS in bytes)"""
    import sys
    p = subprocess.Popen([sys.executable, "-c", _RSS, str(rss_path)] + argv, stdin=subprocess.PIPE, stdout=stdout, stderr=subprocess.PIPE)
    res = {}
    threads = [threading.Thread(target=lambda: res.__setitem__("out", p.stdout.read() if p.stdout else b""), daemon=True),
               threading.Thread(target=lambda: res.__setitem__("err", p.stderr.read()), daemon=True)]
    for t in threads:
        t.start()
    feed(p.stdin); p.stdin.close()
    for t in threads:
        t.join()
    rc = p.wait()
    return rc, res["out"], res["err"], int(open(rss_path).read()) * 1024


def test_memory_is_bounded_on_a_large_pipe(tmp_path):
    """about 500 MB of FASTQ through a pipe: the child's peak RSS stays far below the input's size"""
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    rng = np.random.default_rng(5)
    block = sc.fastq(sc.records(rng, 4000, 100, 151))
    reps = 500_000_000 // len(block) + 1

    def feed(f):
        for _ in range(reps):
            f.write(block)
    rc, out, err, rss = peak_rss([TOOL, "--dump-chunks", "idx", "-"], feed, tmp_path / "rss")
    assert rc == 0, err[-2000:]
    chunks = [json.loads(l) for l in out.decode().splitlines()]
    assert sum(c["bytes1"] for c in chunks) == reps * len(block)
    assert rss < 200_000_000, rss

"""bm2_seq_encode and bm2_mem's FASTA / multi-line FASTQ / standard-input paths on the GPU.

- Context.seq_encode on the corpus of tests/seq_corpus.py: codes, qualities, offsets, names, comments and qual_present must equal the records
  of the host emulation (tests/host_emul/seq_emul.cpp) field by field, and their digest must equal that of the records the reference's
  kseq_init + bseq_read_orig read (tests/golden/seq_corpus_bseq.json, checked against the reference by tests/test_seq_input_cpu.py); on
  four-line FASTQ the batch must equal bm2_fastq_encode's field for field.
- bm2_mem against the unmodified reference run live (oracle/_ref/<isa>/ref_driver mem, as tests/test_zz_mem_cli_gpu.py runs it): the whole SAM
  file, header included, byte-identical except @PG, at two -K values with 1 and 2 chunks in flight."""
import gzip, json, os, subprocess
import numpy as np
import pytest
import seq_corpus as sc
import test_mem_cli_cpu as cli
from test_seq_input_cpu import tools, _emul, CORPUS, GOLDEN  # noqa: F401  (tools is a fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNS = [(100_000_000, 1), (40_000, 2)]
ALL_FASTA = {"pe_fa60", "smart_fa", "C_fa", "gz_fa", "stdin", "stdin_gz", "stdin_smart", "intractg"}


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_seq_encode_equals_the_reference(pkg, tools, name):
    a, b = CORPUS[name]
    if b is None:
        want = _emul(tools, a)[0]
    else:                                          # the records of a pair of files, interleaved
        want = [r for pair in zip(_emul(tools, a)[0], _emul(tools, b)[0]) for r in pair]
    ctx = pkg.capi.Context(0)
    got = ctx.seq_encode(a, b)
    cb, cl = ctx.fastq_comments()
    assert got["n_reads"] == len(want)
    bufs = (a, b if b is not None else a)
    stride = 2 if b is not None else 1
    mine = []
    for r, (nm, cmt, seq, qual) in enumerate(want):
        o0, o1 = got["offsets"][r], got["offsets"][r + 1]
        assert got["names"][r] == nm, r
        assert (bufs[r % stride][cb[r]:cb[r] + cl[r]] if cl[r] else None) == cmt, r
        assert got["codes"][o0:o1].tobytes() == sc.nt4(seq), r
        assert got["qual_present"][r] == (qual is not None), r
        if qual is not None:
            assert bytes(got["quals"][o0:o1]) == qual, r
        mine.append((got["names"][r], bufs[r % stride][cb[r]:cb[r] + cl[r]] if cl[r] else None, got["codes"][o0:o1].tobytes(), bytes(got["quals"][o0:o1]) if got["qual_present"][r] else None))
    assert len(mine) == GOLDEN[name]["records"] and sc.digest(mine) == GOLDEN[name]["sha256"]
    if name == "fq_4line":
        fq = ctx.fastq_encode(a)
        for k in ("codes", "offsets", "quals", "names"):
            assert (fq[k] == got[k]) if k == "names" else np.array_equal(fq[k], got[k]), k
        assert np.array_equal(ctx.fastq_comments()[1], cl) and got["qual_present"].all()
    ctx.close()


@pytest.mark.parametrize("name", sorted(sc.MALFORMED))
def test_seq_encode_rejects_a_malformed_record(pkg, name):
    data, index = sc.MALFORMED[name]
    ctx = pkg.capi.Context(0)
    with pytest.raises(pkg.capi.Bm2Error, match="malformed record %d" % index):
        ctx.seq_encode(data)
    ctx.close()


@pytest.mark.parametrize("name", sorted(sc.MALFORMED))
def test_seq_encode_names_a_malformed_record_of_the_2nd_file(pkg, name):
    """a malformed record ends its file early: the error names it rather than the unequal record counts"""
    data, index = sc.MALFORMED[name]
    good = b"".join(b"@g%d\nACGT\n+\nIIII\n" % i for i in range(4))
    ctx = pkg.capi.Context(0)
    with pytest.raises(pkg.capi.Bm2Error, match="malformed record %d of the 2nd file" % index):
        ctx.seq_encode(good, data)
    ctx.close()


def _contigs(index_prefix, rng, n):
    """n pieces of 1-5 kb of the index's reference (forward strand, from <prefix>.pac), a few bases changed"""
    ann = open(index_prefix + ".ann").read().split("\n")
    spans = [tuple(int(x) for x in ann[2 + 2 * i].split()[:2]) for i in range(int(ann[0].split()[1]))]
    pac = np.fromfile(index_prefix + ".pac", np.uint8)
    out = []
    for k in range(n):
        off, ln = spans[k % len(spans)]
        L = int(rng.integers(1000, 5000)); L = min(L, ln - 1)
        s = off + int(rng.integers(0, ln - L))
        i = np.arange(s, s + L)
        codes = (pac[i >> 2] >> ((~i & 3) << 1)) & 3
        codes[rng.integers(0, L, L // 200)] = rng.integers(0, 4, L // 200)
        out.append((b"ctg%d len=%d" % (k, L), bytes(np.frombuffer(b"ACGT", np.uint8)[codes]), None))
    return out


@pytest.fixture(scope="module")
def inputs(tmp_path_factory, golden_dir):
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    drv = os.path.join(ROOT, "oracle", "_ref", isa, "ref_driver")
    if not os.path.exists(cli.TOOL) or not os.path.exists(drv):
        pytest.skip("bm2_mem / oracle/_ref not built")
    d = tmp_path_factory.mktemp("seq_input_gpu")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    rng = np.random.default_rng(11)
    L = reads.shape[1]
    qual = [bytes(rng.integers(35, 74, L).astype(np.uint8)) for _ in range(len(reads))]
    seq = [bytes(np.frombuffer(b"ACGTN", np.uint8)[r]) for r in reads]
    mate = [[(b"p%d/%d" % (i // 2, w + 1), seq[i], qual[i]) for i in range(w, len(reads), 2)] for w in (0, 1)]
    cmt = [[(h + (b" BC:Z:%d x" % k if k % 2 else b"\tCO:Z:t%d" % k), s, q) for k, (h, s, q) in enumerate(m)] for m in mate]
    files = {}

    def put(name, data):
        p = d / name; p.write_bytes(data); files[name] = str(p)
    put("1.fa", sc.fasta(mate[0], 60)); put("2.fa", sc.fasta(mate[1], 60))
    put("1c.fa", sc.fasta(cmt[0], 60)); put("2c.fa", sc.fasta(cmt[1], 60))
    put("1w.fq", sc.fastq(mate[0], 60))
    put("1.fq", sc.fastq(mate[0])); put("2.fq", sc.fastq(mate[1]))
    put("1at.fq", sc.fastq(mate[0]) + b"@")
    parts = [sc.fasta, lambda r: sc.fastq(r, 70), lambda r: sc.fasta(r, 80, b"\r\n"), sc.fastq, lambda r: b"junk\n" + sc.fastq(r, 50, b"\r\n")]
    put("mixed", b"".join(parts[k % 5](mate[0][k * 50:(k + 1) * 50]) for k in range(10)))
    inter = []
    for k, (a, b) in enumerate(zip(mate[0], mate[1])):
        inter += [a, b] if k % 7 else [a]
    put("inter.fa", sc.fasta(inter, 60))
    put("1.fa.gz", gzip.compress(sc.fasta(mate[0], 60)))
    idx = golden_dir + "/c0_index/ref.fa"
    put("ctg.fa", sc.fasta(_contigs(idx, rng, 40), 60))
    return dict(drv=drv, d=d, f=files, idx=idx)


# (name, arguments of both programs, files, standard input, seq_encode_chunks > 0)
CASES = [
    ("pe_fa60", [], ["1.fa", "2.fa"], None, True),
    ("se_fq_wrapped", [], ["1w.fq"], None, True),
    ("se_mixed", [], ["mixed"], None, True),
    ("smart_fa", ["-p"], ["inter.fa"], None, True),
    ("C_fa", ["-C"], ["1c.fa", "2c.fa"], None, True),
    ("gz_fa", [], ["1.fa.gz"], None, True),
    ("stdin", [], ["-"], "1.fa", True),
    ("stdin_gz", [], ["-"], "1.fa.gz", True),
    ("stdin_smart", ["-p"], ["-"], "inter.fa", True),
    ("stdin_pe", [], ["-", "2.fq"], "1w.fq", True),
    ("intractg", ["-x", "intractg"], ["ctg.fa"], None, True),
    ("fq_4line", [], ["1.fq", "2.fq"], None, False),
    ("fq_header_at_eof", [], ["1at.fq"], None, False),             # a stray '@' after the last record: in no chunk
]


@pytest.mark.parametrize("K,workers", RUNS, ids=["K100M_w1", "K40k_w2"])
@pytest.mark.parametrize("name,args,files,stdin,seq", CASES, ids=[c[0] for c in CASES])
def test_bm2_mem_equals_the_reference(inputs, name, args, files, stdin, seq, K, workers):
    paths = [f if f == "-" else inputs["f"][f] for f in files]
    data = open(inputs["f"][stdin], "rb").read() if stdin else None
    out = str(inputs["d"] / ("%s_%d_%d.sam" % (name, K, workers)))
    o = subprocess.run([cli.TOOL, "-t", "4", "-K", str(K)] + args + ["-p", str(workers), "-o", out, inputs["idx"]] + paths, input=data,
                       capture_output=True, timeout=600)
    assert o.returncode == 0, o.stderr[-2000:]
    ref = subprocess.run([inputs["drv"], "mem", "-t", "4", "-K", str(K)] + args + [inputs["idx"]] + paths, input=data,
                         env=dict(os.environ, BM2_MODE="ref"), capture_output=True, timeout=600)
    assert ref.returncode == 0, ref.stderr[-2000:]
    got = [l for l in open(out, "rb").read().split(b"\n") if not l.startswith(b"@PG")]
    want = [l for l in ref.stdout.split(b"\n") if not l.startswith(b"@PG")]
    assert len(got) == len(want) and len(got) > 40
    diff = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    assert diff == [], (len(diff), got[diff[0]], want[diff[0]])
    st = json.loads(o.stderr.decode().strip().splitlines()[-1])
    assert (st["seq_encode_chunks"] > 0) == seq
    if name in ALL_FASTA:                          # no qualities anywhere: QUAL '*' on every record
        assert all(l.split(b"\t")[10] == b"*" for l in got if l and not l.startswith(b"@"))

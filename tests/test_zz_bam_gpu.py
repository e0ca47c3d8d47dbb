"""BAM out on the GPU: bm2_bgzf_compress is byte-identical to the host emulation of its per-block logic, and `bm2_mem --bam`, decoded by
tests/bam_util.py, equals the SAM bm2_mem writes from the same call - paired, single-end, smart pairing, FASTA input, -R -C -V -M -a -5, an
ALT index and -x ont2d long reads - with the same bytes at 1, 2 and 3 chunks in flight, an EOF block last and every member within BSIZE's
rules.  -C on comments that are not SAM tags is an error naming the read."""
import os, shutil, subprocess
import numpy as np
import pytest
import bam_util as bu
import bam_inputs
import test_bam_cpu as tb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
INDEX_TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_index")
RG = r"@RG\tID:g1\tSM:s1"


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return tb.build_emul(tmp_path_factory)


def test_kernel_equals_emulation(gpu_ctx, emul):
    cases = dict(tb.corpus())
    cases["bam_stream"] = bam_inputs.bam_records(60_000, seed=3)                  # about 25 MB: several hundred blocks, several per CTA
    for name, (data, cut) in cases.items():
        got, ms, members = gpu_ctx.bgzf_compress(data, cut)
        want, starts = tb.emul_stream(emul, data, cut)
        assert got == want, name
        assert members == len(starts) - 1 and bu.inflate(got) == data, name


def _fq(recs, eol=b"\n"):
    return b"".join(b"@" + h + eol + bytes(b"ACGTN"[c] for c in r) + eol + b"+" + eol + q + eol for h, r, q in recs)


@pytest.fixture(scope="module")
def inputs(pkg, tmp_path_factory, golden_dir):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    d = tmp_path_factory.mktemp("bam_gpu")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    qual = [bytes(q) for q in bam_inputs.illumina_quals(len(reads), reads.shape[1], np.random.default_rng(5))]
    f = {}
    for which in (0, 1):
        plain = [(b"p%d/%d" % (i // 2, which + 1), reads[i], qual[i]) for i in range(which, len(reads), 2)]
        tags = [(h + (b"" if k % 5 == 0 else b"\tBX:Z:ACGT%d\tXI:i:%d" % (k, k - 300)), r, q) for k, (h, r, q) in enumerate(plain)]
        illumina = [(h + b" %d:N:0:ACGT" % (which + 1), r, q) for h, r, q in plain]
        for name, recs in (("r%d.fq", plain), ("t%d.fq", tags), ("i%d.fq", illumina)):
            p = d / (name % (which + 1)); p.write_bytes(_fq(recs)); f[name % (which + 1)] = str(p)
        fa = b"".join(b">" + h + b"\n" + bytes(b"ACGTN"[c] for c in r) + b"\n" for h, r, _ in plain)
        (d / ("a%d.fa" % (which + 1))).write_bytes(fa); f["a%d.fa" % (which + 1)] = str(d / ("a%d.fa" % (which + 1)))
    inter = []
    for k in range(len(reads) // 2):
        a, b = 2 * k, 2 * k + 1
        if k % 10 == 3:
            inter.append((b"p%d/1" % k, reads[a], qual[a]))
        else:
            inter += [(b"p%d/1" % k, reads[a], qual[a]), (b"p%d/2" % k, reads[b], qual[b])]
    (d / "inter.fq").write_bytes(_fq(inter)); f["inter"] = str(d / "inter.fq")
    for sub in ("idx", "alt", "anno"):
        t = d / sub; t.mkdir()
        for x in os.listdir(golden_dir + "/c0_index"):
            shutil.copy(os.path.join(golden_dir, "c0_index", x), t / x)
    (d / "alt" / "ref.fa.alt").write_text("chr3\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\nchr4\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\n")
    lines = open(d / "anno" / "ref.fa.ann").read().split("\n")
    for k, a in enumerate(["first contig", "", "with\ta tab", "(null)"]):
        gi, name = lines[1 + 2 * k].split()[:2]
        lines[1 + 2 * k] = ("%s %s %s" % (gi, name, a)) if a else "%s %s" % (gi, name)
    (d / "anno" / "ref.fa.ann").write_text("\n".join(lines))
    # long reads (-x ont2d) on a 1 Mbp genome indexed by bm2_index
    from bwa_mem2_b200 import synth
    lr = d / "long"; lr.mkdir()
    ctg = synth.make_reference(1_000_000, seed=9, n_contigs=3)
    synth.write_fasta(str(lr / "ref.fa"), ctg)
    subprocess.run([INDEX_TOOL, str(lr / "ref.fa")], check=True, capture_output=True, timeout=600)
    long_reads = synth.make_long_reads(ctg, 12, read_len=6000, seed=4)
    lq = bam_inputs.illumina_quals(len(long_reads), max(len(r) for r in long_reads), np.random.default_rng(8))
    (lr / "reads.fq").write_bytes(_fq([(b"long%d" % i, r, bytes(lq[i][:len(r)])) for i, r in enumerate(long_reads)]))
    f["long"] = str(lr / "reads.fq")
    return d, f


def _run(args, out, bam):
    r = subprocess.run([TOOL] + (["--bam"] if bam else []) + ["-o", out] + args, capture_output=True, timeout=900)
    return r


def _same(d, name, args, files, idx="idx"):
    prefix = str(d / idx / "ref.fa") if not os.path.isabs(idx) else idx
    sam, bam = str(d / (name + ".sam")), str(d / (name + ".bam"))
    a = _run(args + [prefix] + files, sam, False); b = _run(args + [prefix] + files, bam, True)
    assert a.returncode == 0 and b.returncode == 0, (a.stderr[-2000:], b.stderr[-2000:])
    text = open(sam).read()
    hdr_text, refs, lines, ms = bu.read_bam_file(open(bam, "rb").read())
    want_hdr = [l for l in text.split("\n") if l.startswith("@") and not l.startswith("@PG")]
    assert [l for l in hdr_text.split("\n") if l.startswith("@") and not l.startswith("@PG")] == want_hdr
    assert [n for n, _ in refs] == [l.split()[1] for i, l in enumerate(open(prefix + ".ann")) if i % 2 == 1]
    want = [bu.norm(l) for l in text.split("\n") if l and not l.startswith("@")]
    assert len(lines) == len(want) and [bu.norm(l) for l in lines] == want
    assert all(len(m) <= 65536 for m, _ in ms)
    return text


@pytest.mark.parametrize("name,args,files,idx", [
    ("pe", [], ["r1.fq", "r2.fq"], "idx"),
    ("se", [], ["r1.fq"], "idx"),
    ("smart", ["-p"], ["inter"], "idx"),
    ("fasta", [], ["a1.fa", "a2.fa"], "idx"),
    ("R_C_V_M_a_5", ["-R", RG, "-C", "-V", "-M", "-a", "-5"], ["t1.fq", "t2.fq"], "anno"),
    ("alt", [], ["r1.fq", "r2.fq"], "alt"),
    ("ont2d", ["-x", "ont2d"], ["long"], "long"),
])
def test_bam_equals_sam(inputs, name, args, files, idx):
    d, f = inputs
    text = _same(d, name, args + ["-K", "40000"], [f[x] for x in files], idx if idx != "long" else str(d / "long" / "ref.fa"))
    if name == "R_C_V_M_a_5":
        assert "\tBX:Z:" in text and "\tXR:Z:" in text and "\tRG:Z:g1" in text
    if name == "fasta":
        assert "\t*\tNM:i:" in text or "\t*\tAS:i:" in text


def _records_part(data):
    """The members after the header's (the header carries the @PG command line)."""
    ms = bu.members(data)
    raw = b"".join(r for _, r in ms)
    _, _, used = bu.parse_header(raw)
    at = 0
    for k, (_, r) in enumerate(ms):
        at += len(r)
        if at == used:
            return b"".join(m for m, _ in ms[k + 1:])
    raise AssertionError("the header does not end a member")


def test_bam_bytes_do_not_depend_on_workers(inputs):
    d, f = inputs
    got = []
    for w in (1, 2, 3):
        out = str(d / ("w%d.bam" % w))
        r = _run(["-p", str(w), "-K", "30000", str(d / "idx" / "ref.fa"), f["r1.fq"], f["r2.fq"]], out, True)
        assert r.returncode == 0, r.stderr[-2000:]
        data = open(out, "rb").read()
        assert data.endswith(bu.EOF_BLOCK)
        got.append(_records_part(data))
    assert got[0] == got[1] == got[2] and len(bu.members(got[0])) > 3


def test_bam_C_on_illumina_comments_is_an_error(inputs):
    d, f = inputs
    r = _run(["-C", str(d / "idx" / "ref.fa"), f["i1.fq"], f["i2.fq"]], str(d / "ill.bam"), True)
    assert r.returncode != 0 and b"p0" in r.stderr and b"1:N:0:ACGT" in r.stderr
    assert _run(["-C", str(d / "idx" / "ref.fa"), f["i1.fq"], f["i2.fq"]], str(d / "ill.sam"), False).returncode == 0

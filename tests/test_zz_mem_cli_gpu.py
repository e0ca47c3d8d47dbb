"""bm2_mem with the options of `bwa-mem2 mem` against the unmodified reference run live with the same arguments: the whole SAM file, header
included, must be byte-identical except the @PG line.  Every case runs at two -K values (one chunk / several chunks) with 1 and 2 chunks in
flight.  Then the GPU split of smart pairing (bm2_fastq_smart_pair) against the host model of bseq_classify in tests/test_mem_cli_cpu.py."""
import os, shutil, subprocess
import numpy as np
import pytest
import test_mem_cli_cpu as cli

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RG = r"@RG\tID:g1\tSM:s1"

CASES = [
    ("M_R", ["-M", "-R", RG], "pe"),
    ("5SP", ["-5SP"], "pe"),
    ("Y_q", ["-Y", "-q"], "pe"),
    ("a", ["-a"], "pe"),
    ("S", ["-S"], "pe"),
    ("I400,40", ["-I", "400,40"], "pe"),
    ("k15_w60_T20_h3,50", ["-k", "15", "-w", "60", "-T", "20", "-h", "3,50"], "pe"),
    ("A2", ["-A", "2"], "pe"),
    ("x_intractg", ["-x", "intractg"], "pe"),
    ("H_file_R", ["-H", "{hdr}", "-R", RG], "pe"),
    ("C", ["-C"], "pe_cmt"),
    ("C_crlf", ["-C"], "pe_cmt_crlf"),
    ("V", ["-V"], "pe_anno"),
    ("alt", [], "pe_alt"),
    ("alt_j", ["-j"], "pe_alt"),
    ("se_M_C", ["-M", "-C"], "se_cmt"),
    ("smart", ["-p"], "inter"),
    ("smart_M_C", ["-p", "-M", "-C"], "inter"),
    ("smart_second_file", ["-p"], "inter+"),
]
RUNS = [(100_000_000, 1), (40_000, 2)]


def _fq(recs, eol=b"\n"):
    return b"".join(b"@" + h + eol + bytes(b"ACGTN"[c] for c in r) + eol + b"+" + eol + q + eol for h, r, q in recs)


@pytest.fixture(scope="module")
def inputs(tmp_path_factory, golden_dir):
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    drv = os.path.join(ROOT, "oracle", "_ref", isa, "ref_driver")
    if not os.path.exists(cli.TOOL) or not os.path.exists(drv):
        pytest.skip("bm2_mem / oracle/_ref not built")
    d = tmp_path_factory.mktemp("mem_cli_gpu")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    L = reads.shape[1]
    rng = np.random.default_rng(5)
    qual = [bytes(rng.integers(35, 74, L).astype(np.uint8)) for _ in range(len(reads))]
    files = {}
    for which in (0, 1):
        plain = [(b"p%d/%d" % (i // 2, which + 1), reads[i], qual[i]) for i in range(which, len(reads), 2)]
        cmt = [(h + (b"" if k % 5 == 0 else b"\tBX:Z:ACGT%d" % k if k % 2 else b" CB:Z:%d comment" % k), r, q) for k, (h, r, q) in enumerate(plain)]
        for name, recs, eol in (("r%d.fq", plain, b"\n"), ("c%d.fq", cmt, b"\n"), ("crlf%d.fq", cmt, b"\r\n")):
            p = d / (name % (which + 1)); p.write_bytes(_fq(recs, eol)); files[name % (which + 1)] = str(p)
    # interleaved: pairs, orphans (one mate only) and runs of three reads with one name
    inter = []
    for k in range(len(reads) // 2):
        a, b = 2 * k, 2 * k + 1
        if k % 10 == 3:
            inter.append((b"p%d/1" % k, reads[a], qual[a]))
        elif k % 10 == 7:
            inter += [(b"p%d/1" % k, reads[a], qual[a]), (b"p%d/2" % k, reads[b], qual[b]), (b"p%d/3" % k, reads[(b + 6) % len(reads)], qual[b])]
        else:
            inter += [(b"p%d/1 c%d" % (k, k), reads[a], qual[a]), (b"p%d/2" % k, reads[b], qual[b])]
    (d / "inter.fq").write_bytes(_fq(inter)); files["inter"] = str(d / "inter.fq")
    (d / "hdr.txt").write_text("@CO\tfrom a file\n@CO\tsecond\\tline\n")
    for sub in ("alt", "anno"):
        t = d / sub; t.mkdir()
        for f in os.listdir(golden_dir + "/c0_index"):
            shutil.copy(os.path.join(golden_dir, "c0_index", f), t / f)
    (d / "alt" / "ref.fa.alt").write_text("chr3\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\nchr4\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\n")
    lines = open(d / "anno" / "ref.fa.ann").read().split("\n")
    for k, a in enumerate(["first contig", "", "with\ta tab", "(null)"]):
        gi, name = lines[1 + 2 * k].split()[:2]
        lines[1 + 2 * k] = ("%s %s %s" % (gi, name, a)) if a else "%s %s" % (gi, name)
    (d / "anno" / "ref.fa.ann").write_text("\n".join(lines))
    idx = golden_dir + "/c0_index/ref.fa"
    inp = {"pe": [idx, files["r1.fq"], files["r2.fq"]], "pe_cmt": [idx, files["c1.fq"], files["c2.fq"]],
           "pe_cmt_crlf": [idx, files["crlf1.fq"], files["crlf2.fq"]], "pe_anno": [str(d / "anno" / "ref.fa"), files["r1.fq"], files["r2.fq"]],
           "pe_alt": [str(d / "alt" / "ref.fa"), files["r1.fq"], files["r2.fq"]], "se_cmt": [idx, files["c1.fq"]],
           "inter": [idx, files["inter"]], "inter+": [idx, files["inter"], files["r2.fq"]]}
    return dict(drv=drv, d=d, inp=inp, hdr=str(d / "hdr.txt"))


@pytest.mark.parametrize("K,workers", RUNS, ids=["K100M_w1", "K40k_w2"])
@pytest.mark.parametrize("name,args,inp", CASES, ids=[c[0] for c in CASES])
def test_bm2_mem_equals_the_reference(inputs, name, args, inp, K, workers):
    args = [inputs["hdr"] if a == "{hdr}" else a for a in args]
    files = inputs["inp"][inp]
    out = str(inputs["d"] / ("%s_%d_%d.sam" % (name, K, workers)))
    o = subprocess.run([cli.TOOL, "-t", "4", "-K", str(K)] + args + ["-p", str(workers), "-o", out] + files, capture_output=True, text=True, timeout=600)
    assert o.returncode == 0, o.stderr[-2000:]
    ref = subprocess.run([inputs["drv"], "mem", "-t", "4", "-K", str(K)] + args + files, env=dict(os.environ, BM2_MODE="ref"),
                         capture_output=True, timeout=600)
    assert ref.returncode == 0, ref.stderr[-2000:]
    got = [l for l in open(out, "rb").read().split(b"\n") if not l.startswith(b"@PG")]
    want = [l for l in ref.stdout.split(b"\n") if not l.startswith(b"@PG")]
    assert len(got) == len(want) and len(got) > 500
    diff = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    assert diff == [], (len(diff), got[diff[0]], want[diff[0]])
    if inp == "inter+":
        assert "second query file is ignored" in o.stderr
    if "-C" in args:
        assert any(b"\tBX:Z:" in l or b"\tc1" in l for l in got)
    if K == 40_000:
        import json
        assert json.loads(o.stderr.strip().splitlines()[-1])["chunks"] > 1


@pytest.mark.parametrize("pattern", sorted(cli.name_patterns()))
def test_smart_pair_split_equals_bseq_classify(pkg, pattern):
    capi = pkg.capi
    names = cli.name_patterns()[pattern]
    rng = np.random.default_rng(len(names))
    lens = rng.integers(1, 200, len(names))
    seqs = [rng.integers(0, 5, n).astype(np.uint8) for n in lens]
    quals = [bytes(rng.integers(33, 74, n).astype(np.uint8)) for n in lens]
    heads = [nm + b"/%d" % (i % 3) + (b" cmt %d" % i if i % 4 else b"") for i, nm in enumerate(names)]
    buf = _fq(list(zip(heads, seqs, quals)))
    ctx = capi.Context(0)
    fq = ctx.fastq_encode(buf)
    assert fq["n_reads"] == len(names)
    cb, cl = ctx.fastq_comments()
    sets = ctx.fastq_smart_pair()
    se, pe = cli.classify([fq["names"][i] for i in range(len(names))])
    assert sets[0]["read_index"].tolist() == se and sets[1]["read_index"].tolist() == pe
    for s, want_idx in zip(sets, (se, pe)):
        assert s["n_reads"] == len(want_idx)
        for j, i in enumerate(want_idx):
            a, b = s["offsets"][j], s["offsets"][j + 1]
            assert np.array_equal(s["codes"][a:b], seqs[i]) and bytes(s["quals"][a:b]) == quals[i]
            assert buf[s["name_beg"][j]:s["name_beg"][j] + s["name_len"][j]] == names[i]
            assert (s["comment_beg"][j], s["comment_len"][j]) == (cb[i], cl[i])
            want_c = heads[i].split(b" ", 1)[1] if b" " in heads[i] else b""
            assert buf[cb[i]:cb[i] + cl[i]] == want_c
    with pytest.raises(capi.Bm2Error):           # a paired-end batch cannot be split
        ctx.fastq_encode(buf, buf)
        ctx.fastq_smart_pair()
    ctx.close()

"""bm2_wgsmetrics on the GPU: bm2_wgs_set / bm2_wgs_add / bm2_wgs_finish equal the host emulation (tests/host_emul/wgsmetrics_emul.cpp) on
crafted and random records at several window sizes, read errors included; `bm2_wgsmetrics` writes the file Python computes (Picard's loop,
tests/wgsmetrics_util.py) from the BAM of `bm2_mem --markdup` (paired, single-end, smart pairing) against an index built by bm2_index from a
FASTA with N, n and IUPAC runs, from the BAM of `bm2_applybqsr`, and with every option changed; the bytes do not depend on -t, --window or
standard input; the error cases exit 1 and leave no file.  The references are small: no test allocates a genome-sized counter array."""
import json, os, subprocess
import numpy as np
import pytest
import bam_util as bu
import bqsr_util as bq
import markdup_util as mu
import wgsmetrics_util as wm
import test_wgsmetrics_cpu as tc
import test_zz_markdup_gpu as tmg

pytestmark = pytest.mark.gpu

TOOL = wm.TOOL
ROOT = wm.ROOT
MEM = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
INDEX = os.path.join(ROOT, "bwa-mem2_b200", "bm2_index")
APPLY = os.path.join(ROOT, "bwa-mem2_b200", "bm2_applybqsr")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return wm.build_emul(tmp_path_factory)


def _device(ctx, ref, wins, min_mapq=20, min_baseq=20, cap=250, count_unpaired=False):
    ctx.wgs_set(ref.off, ref.lens, ref.l_pac, ref.nocall_ranges(), min_mapq, min_baseq, cap, count_unpaired)
    for w in wins:
        data, starts = bq.flatten(w)
        ctx.wgs_add(data, starts)
    return ctx.wgs_finish()


def test_kernels_equal_emulation(gpu_ctx, emul):
    rng = np.random.default_rng(91)
    ref = tc.REF
    for recs in (tc.crafted(), wm.random_pairs(ref, rng, 2000), []):
        for kw in ({}, dict(min_mapq=0, min_baseq=0, cap=10, count_unpaired=True)):
            for sizes in ([max(len(recs), 1)], [1], [7], [333]):
                wins = wm.windows(recs, sizes)
                want = wm.emul_run(emul, ref, wins, **kw)
                got = _device(gpu_ctx, ref, wins, **kw)
                assert want[3] is None and np.array_equal(got["hist"], want[0]) and got["exc"] == want[1], (kw, sizes)
                assert (got["counted_records"], got["records"], got["carried_max"]) == (want[2], want[4], want[5])
                assert got["add_ms"] >= 0 and got["finish_ms"] >= 0
        assert not recs or _device(gpu_ctx, ref, [recs])["exc"][4] > 0
    P = 0x1 | 0x40 | 0x20
    ok = wm.rec("ok", P, 0, 100, [(10, 0)], [30] * 10)
    for bad, msg in ((wm.rec("noq", P, 0, 200, [(10, 0)], None), "read noq (record 3) has no base qualities"),
                     (wm.rec("past", P, 0, 2995, [(10, 0)], [30] * 10), "read past (record 3) does not lie inside a contig"),
                     (wm.rec("badcig", P, 0, 200, [(10, 0), (2, 1)], [30] * 10, seq="A" * 10), "read badcig (record 3) has a CIGAR")):
        wins = [[ok, ok], [ok, bad, ok]]
        want = wm.emul_run(emul, ref, wins, check_order=False)
        assert msg in want[3]
        gpu_ctx.wgs_set(ref.off, ref.lens, ref.l_pac, ref.nocall_ranges())
        gpu_ctx.wgs_add(*bq.flatten(wins[0]))
        with pytest.raises(Exception, match=msg.replace("(", r"\(").replace(")", r"\)")):
            gpu_ctx.wgs_add(*bq.flatten(wins[1]))
        got = gpu_ctx.wgs_finish()                                                       # nothing of the failed window was counted
        assert got["records"] == 2 and np.array_equal(got["hist"], _device(gpu_ctx, ref, [wins[0]])["hist"])


def _genome(rng):
    """A FASTA of three contigs with runs of N, n, R, y and a short contig."""
    def s(n):
        return "".join("ACGT"[int(x)] for x in rng.integers(0, 4, n))
    c1 = s(30000) + "N" * 200 + s(20000) + "RRRRRR" + s(15000) + "n" * 50 + s(10000)
    c2 = s(25000) + "yyyy" + s(5000) + "NNNNNNNNNN" + s(20000)
    return ">chrA\n%s\n>chrB desc\n%s\n>chrC\n%s\n" % (c1, c2, s(800))


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    for t in (TOOL, MEM, INDEX, APPLY):
        if not os.path.exists(t):
            pytest.skip(os.path.basename(t) + " not built")
    d = tmp_path_factory.mktemp("wgs_gpu")
    rng = np.random.default_rng(92)
    (d / "ref.fa").write_text(_genome(rng))
    subprocess.run([INDEX, str(d / "ref.fa")], check=True, capture_output=True, timeout=900)
    prefix = str(d / "ref.fa")
    ref = wm.Ref.read(prefix)
    assert ref.nocall.any() and any(c not in wm.NOCALL for _, _, c in ref.holes)
    pairs = mu.planted_pairs(mu.load_reference(prefix), rng, n_base=400)
    files, _ = tmg._write_pairs(d, pairs, "p")
    bams = {}
    for mode in ("pe", "se", "smart"):
        out = str(d / ("md_%s.bam" % mode))
        r = subprocess.run([MEM, "--markdup", "-R", r"@RG\tID:g1\tSM:s", prefix] + files[mode] + (["-p"] if mode == "smart" else []) + ["-o", out],
                           capture_output=True, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        bams[mode] = out
    return d, prefix, ref, files, bams


def _tool(args, stdin=None):
    r = subprocess.run([TOOL] + args, capture_output=True, timeout=900, stdin=stdin)
    assert r.returncode == 0, r.stderr[-3000:]
    return r, json.loads(r.stderr.decode().strip().split("\n")[-1])


def _want(bam, ref, args, **kw):
    raw = bu.inflate(open(bam, "rb").read())
    _, _, used = bu.parse_header(raw)
    recs = [r for _, r in bu.records(raw[used:])]
    hist, exc, counted, err = wm.metrics(recs, ref, **kw)
    assert err is None
    return wm.text(hist, exc, " ".join(args)), len(recs), counted


@pytest.mark.parametrize("mode", ["pe", "se", "smart"])
def test_markdup_bam_equals_python(inputs, mode):
    d, prefix, ref, files, bams = inputs
    out = str(d / ("w_%s.txt" % mode))
    args = ["-o", out, prefix, bams[mode]]
    _, st = _tool(args)
    want, n, counted = _want(bams[mode], ref, args)
    assert open(out).read() == want and st["records"] == n and st["counted_records"] == counted and st["windows"] == 1
    v = dict(zip(*[l.split("\t") for l in want.split("\n")[4:6]]))
    assert float(v["PCT_EXC_DUPE"]) > 0
    if mode == "se":                                                                   # single-end reads are unpaired: nothing counts
        assert float(v["MEAN_COVERAGE"]) == 0 and float(v["PCT_EXC_UNPAIRED"]) > 0
    else:
        assert float(v["MEAN_COVERAGE"]) > 0
    assert not os.path.exists(out + ".tmp")


def test_applybqsr_bam_and_options(inputs):
    d, prefix, ref, files, bams = inputs
    bref = bq.Ref(prefix)
    (d / "s.vcf").write_text(bq.vcf_text(bref, bq.random_sites(bref, np.random.default_rng(93), every=50)))
    r = subprocess.run([MEM, "--recal-file", str(d / "t.txt"), "--known-sites", str(d / "s.vcf"), "-R", r"@RG\tID:g1\tSM:s", prefix] + files["pe"] +
                       ["-o", str(d / "rc.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([APPLY, "--bqsr-recal-file", str(d / "t.txt"), "-o", str(d / "ap.bam"), str(d / "rc.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    args = ["-o", str(d / "ap.txt"), prefix, str(d / "ap.bam")]
    _tool(args)
    assert open(d / "ap.txt").read() == _want(str(d / "ap.bam"), ref, args)[0]
    args = ["--min-mapq", "0", "--min-baseq", "0", "--coverage-cap", "10", "--count-unpaired", "-o", str(d / "opt.txt"), prefix, bams["pe"]]
    _tool(args)
    want = _want(bams["pe"], ref, args, min_mapq=0, min_baseq=0, cap=10, count_unpaired=True)[0]
    assert open(d / "opt.txt").read() == want and want.endswith("\n10\t" + want.rsplit("\t", 1)[1])


def test_bytes_do_not_depend_on_threads_windows_or_stdin(inputs):
    d, prefix, ref, files, bams = inputs
    bodies, stats = [], []
    for k, extra in enumerate((["-t", "1"], ["-t", "8"], ["-t", "8", "--window", "16K"], ["-t", "3", "--window", "100K"])):
        out = str(d / ("b%d.txt" % k))
        stats.append(_tool(extra + ["-o", out, prefix, bams["pe"]])[1])
        bodies.append(open(out).read().split("\n", 2)[2])
    with open(bams["pe"], "rb") as f:
        r, st = _tool([prefix, "-"], stdin=f)
    bodies.append(r.stdout.decode().split("\n", 2)[2])
    assert all(b == bodies[0] for b in bodies)
    assert stats[2]["windows"] > 10 and stats[2]["carried_max"] > 0 and stats[0]["windows"] == 1
    assert len({s["counted_records"] for s in stats + [st]}) == 1


def test_errors(inputs, tmp_path):
    d, prefix, ref, files, bams = inputs
    r = subprocess.run([MEM, "--markdup", "-R", r"@RG\tID:g1", prefix] + files["fasta"] + ["-o", str(tmp_path / "fa.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([MEM, "--bam", "-R", r"@RG\tID:g1", prefix] + files["pe"] + ["-o", str(tmp_path / "un.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    raw = bu.inflate(open(bams["pe"], "rb").read())
    text, refs, used = bu.parse_header(raw)
    recs = [x for _, x in bu.records(raw[used:])]
    (tmp_path / "rev.bam").write_bytes(wm.bam_bytes(ref, recs[::-1], text=text))
    golden = os.path.join(ROOT, "tests", "golden", "c0_index", "ref.fa")
    for args, msg in (([prefix, str(tmp_path / "fa.bam")], "has no base qualities"),
                      ([prefix, str(tmp_path / "un.bam")], "is not coordinate-sorted"),
                      ([prefix, str(tmp_path / "rev.bam")], "is out of coordinate order"),
                      ([golden, bams["pe"]], "in the header, chr1 of length")):
        out = str(tmp_path / "e.txt")
        r = subprocess.run([TOOL, "-o", out] + args, capture_output=True, timeout=900)
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr[-2000:])
        assert not os.path.exists(out) and not os.path.exists(out + ".tmp")

"""Recalibration tables on the GPU: bm2_bqsr_count equals the host emulation (tests/host_emul/bqsr_emul.cpp) on the crafted records of each
rule and on random ones, read errors included; `bm2_mem --recal-file` on reads with planted mismatches, indels and duplicates, with a synthetic
VCF over part of them, writes the report Python computes from the output BAM's records, the reference and the VCF - paired, single-end,
smart pairing, -R with and without PU, gzip known sites - while its BAM records, BAI layout and metrics equal --markdup's; the report is the same at
-p 1, -p 3 and --sort-mem 100K; reads without qualities are an error."""
import gzip, json, os, subprocess
import numpy as np
import pytest
import bam_util as bu
import bqsr_util as bq
import markdup_util as mu
import test_zz_bam_gpu as tg
import test_zz_markdup_gpu as tmg

pytestmark = pytest.mark.gpu

TOOL = tg.TOOL


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return bq.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def ref(golden_dir):
    return bq.Ref(os.path.join(golden_dir, "c0_index", "ref.fa"))


def test_kernel_equals_emulation(pkg, golden_dir, emul, ref):
    idx = pkg.capi.Index(os.path.join(golden_dir, "c0_index", "ref.fa"))
    ctx = pkg.capi.Context(0, index=idx)
    try:
        rng = np.random.default_rng(51)
        crafted = bq.crafted(ref, rng)
        cases = [(crafted, bq.random_sites(ref, rng, 40)), (bq.random_records(ref, rng, 4000), bq.random_sites(ref, rng)),
                 (bq.random_records(ref, rng, 2000), []), ([], [])]
        for recs, sites in cases:
            cov, jun = bq.sites_bits(ref, sites)
            ctx.bqsr_sites(bq.pack_bits(cov), bq.pack_bits(jun), ref.l_pac, ref.holes, "rg.1")
            for part in (recs[: len(recs) // 3], recs[len(recs) // 3:]):                  # two calls add up
                data, starts = bq.flatten(part)
                ctx.bqsr_count(data, starts)
            got = ctx.bqsr_tables()
            data, starts = bq.flatten(recs)
            want = bq.emul_count(emul, data, starts, ref, cov, jun)
            assert bq.same_tables(got, want) and got["err_kind"] == 0 and got["read_group"] == "rg.1" and got["ms"] >= 0
            assert bq.emul_report(emul, got, "rg.1") == bq.emul_report(emul, want, "rg.1")
        ok = bq.make_rec("ok", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50)
        for bad, kind in ((bq.make_rec("noq", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), None), 1),
                          (bq.make_rec("long", 0, 0, 100, [(501, 0)], ref.seq(0, 100, 501), [30] * 501), 2),
                          (bq.make_rec("hiq", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [94] * 50), 3)):
            ctx.bqsr_sites(bq.pack_bits(np.zeros(ref.l_pac, bool)), bq.pack_bits(np.zeros(ref.l_pac, bool)), ref.l_pac, ref.holes, "g")
            data, starts = bq.flatten([ok, ok, bad, ok])
            ctx.bqsr_count(data, starts)
            t = ctx.bqsr_tables()
            assert (t["err_kind"], t["err_index"], t["reads"]) == (kind, 2, 3) and t["err_name"] == bu.fields(bad)["qname"]
    finally:
        ctx.close(); idx.close()


@pytest.fixture(scope="module")
def planted(golden_dir, tmp_path_factory, ref):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    d = tmp_path_factory.mktemp("bqsr_gpu")
    prefix = os.path.join(golden_dir, "c0_index", "ref.fa")
    rng = np.random.default_rng(53)
    pairs = mu.planted_pairs(mu.load_reference(prefix), rng, n_base=150)
    out = []
    for n, r1, q1, r2, q2 in pairs:                                               # planted mismatches and indels
        r1 = bq.mutate(r1, rng, 0.01)
        if rng.random() < 0.2:
            k = int(rng.integers(20, 80))
            r1 = r1[:k] + "".join("ACGT"[int(x)] for x in rng.integers(0, 4, 2)) + r1[k:-2] if rng.random() < 0.5 else r1[:k] + r1[k + 3:] + "ACG"
        out.append((n, r1, q1, bq.mutate(r2, rng, 0.01), q2))
    files, _ = tmg._write_pairs(d, out, "p")
    sites = bq.random_sites(ref, rng, every=30)
    (d / "a.vcf").write_text(bq.vcf_text(ref, sites[::2]))
    (d / "b.vcf.gz").write_bytes(gzip.compress(bq.vcf_text(ref, sites[1::2]).encode()))
    return d, prefix, files, sites


def _run(args, timeout=900):
    r = subprocess.run([TOOL] + args, capture_output=True, timeout=timeout)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1])


def _want(out, ref, sites, rg):
    cov, jun = bq.sites_bits(ref, sites)
    return bq.report_text(bq.count(tmg._records(out), ref, cov, jun), rg)


@pytest.mark.parametrize("mode,rg", [("pe", r"@RG\tID:g1\tSM:s"), ("se", r"@RG\tID:g1\tSM:s\tPU:fc.1"), ("smart", r"@RG\tID:g7\tPU:x.2"),
                                     ("pe", r"@RG\tID:g1\tPU:fc.3\tLB:l")])
def test_report_equals_python(planted, ref, mode, rg):
    d, prefix, files, sites = planted
    w = d / ("r_%s_%d" % (mode, len(rg))); w.mkdir()
    known = ["--known-sites", str(d / "a.vcf"), "--known-sites", str(d / "b.vcf.gz")]
    common = ["-R", rg, "-K", "100000000" if mode == "smart" else "20000", prefix] + files[mode] + (["-p"] if mode == "smart" else [])
    st = _run(["--recal-file", str(w / "t.txt"), "--markdup-metrics", str(w / "m.txt")] + known + ["--write-index"] + common + ["-o", str(w / "r.bam")])
    plain = _run(["--markdup-metrics", str(w / "pm.txt"), "--write-index"] + common + ["-o", str(w / "p.bam")])
    assert sorted(os.listdir(w)) == ["m.txt", "p.bam", "p.bam.bai", "pm.txt", "r.bam", "r.bam.bai", "t.txt"]
    assert tg._records_part(open(w / "r.bam", "rb").read()) == tg._records_part(open(w / "p.bam", "rb").read())
    # the BAI's virtual offsets move with the header's @PG command line, so the two indexes agree in layout, not in bytes
    assert len(open(w / "r.bam.bai", "rb").read()) == len(open(w / "p.bam.bai", "rb").read())
    assert open(w / "m.txt").read().split("\n", 2)[2] == open(w / "pm.txt").read().split("\n", 2)[2]
    assert "bqsr_s" not in plain and st["known_sites"] == len(sites) and st["bqsr_reads"] > 0 and st["bqsr_bases"] > 0 and st["bqsr_s"] > 0
    text = open(w / "t.txt").read()
    assert text == _want(str(w / "r.bam"), ref, sites, bq.read_group(rg))
    rows2 = [l for l in text.split("\n") if " Cycle " in l]
    assert rows2 and (mode == "se") == all(int(l.split()[2]) > 0 for l in rows2)


def test_report_does_not_depend_on_workers_or_budgets(planted):
    d, prefix, files, sites = planted
    w = d / "budgets"; w.mkdir()
    common = ["-R", r"@RG\tID:g1\tSM:s", "--known-sites", str(d / "a.vcf"), "--known-sites", str(d / "b.vcf.gz"), "-K", "20000", prefix] + files["pe"]
    texts, stats = [], []
    for k, extra in enumerate((["-p", "1"], ["-p", "3"], ["-p", "2", "--sort-mem", "100K"])):
        stats.append(_run(["--recal-file", str(w / ("t%d.txt" % k))] + extra + common + ["-o", str(w / ("r%d.bam" % k))]))
        texts.append(open(w / ("t%d.txt" % k)).read())
    assert texts[0] == texts[1] == texts[2]
    assert stats[2]["sort_runs"] >= 3 and stats[2]["merge_windows"] >= 1 and stats[0]["sort_runs"] == 1
    assert stats[0]["bqsr_bases"] == stats[1]["bqsr_bases"] == stats[2]["bqsr_bases"]
    r = subprocess.run([TOOL, "--recal-file", str(w / "s.txt"), "-R", r"@RG\tID:g1", "--known-sites", str(d / "a.vcf"), "-K", "20000", prefix] + files["pe"],
                       capture_output=True, timeout=900)                              # standard output as the BAM destination
    assert r.returncode == 0 and r.stdout[:4] == b"\x1f\x8b\x08\x04" and open(w / "s.txt").read().startswith("#:GATKReport.v1.1:5\n")


def test_read_and_vcf_errors(planted, tmp_path):
    d, prefix, files, sites = planted
    r = subprocess.run([TOOL, "--recal-file", str(tmp_path / "t.txt"), "-R", r"@RG\tID:g1", "--known-sites", str(d / "a.vcf"), prefix] + files["fasta"]
                       + ["-o", str(tmp_path / "o.bam")], capture_output=True, timeout=900)
    assert r.returncode == 1 and b"has no base qualities" in r.stderr and not os.path.exists(tmp_path / "t.txt"), r.stderr[-2000:]
    (tmp_path / "bad.vcf").write_text("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\nnochrom\t5\t.\tA\tG\t.\t.\t.\n")
    r = subprocess.run([TOOL, "--recal-file", str(tmp_path / "t.txt"), "-R", r"@RG\tID:g1", "--known-sites", str(tmp_path / "bad.vcf"), prefix]
                       + files["pe"] + ["-o", str(tmp_path / "o2.bam")], capture_output=True, timeout=900)
    assert r.returncode == 1 and b"bad.vcf:2: CHROM nochrom is not a contig" in r.stderr, r.stderr[-2000:]

"""bm2_baserecalibrator on the GPU: bm2_recal_add equals the host emulation (tests/host_emul/baserecalibrator_emul.cpp) on crafted and random
records at covariate counts on both sides of the shared/global threshold and at it, over several calls, each read error named; the table of a
bm2_mem --markdup BAM is byte for byte bm2_mem --recal-file's; three lanes of bm2_mem --sort merged and marked by bm2_markdup give Python's
per-read-group table, which bm2_applybqsr applies as tests/applybqsr_util.py does; the bytes do not depend on -t, --window, standard input,
the inputs' split or their order; errors exit with their code and leave no table."""
import json, os, random, subprocess
import numpy as np
import pytest
import applybqsr_util as au
import bam_util as bu
import baserecalibrator_util as br
import bqsr_util as bq
import markdup_bam_util as mb
import markdup_util as mu
import test_baserecalibrator_cpu as tc
import test_zz_bam_gpu as tg
import test_zz_markdup_gpu as tmg
from test_zz_bqsr_gpu import planted, ref  # noqa: F401  (fixtures: bm2_mem's planted reads and sites, the c0 reference)

pytestmark = pytest.mark.gpu

MEM = tg.TOOL
TOOL = tc.TOOL
APPLY = os.path.join(bq.ROOT, "bwa-mem2_b200", "bm2_applybqsr")
SHARED_MAX = 2                                       # kBqsrSharedCovMax (bqsr_device.cuh)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return br.build_rg_emul(tmp_path_factory)


def _set(ctx, ref, cov, jun, ids, id_cov, n_cov):
    ctx.recal_set(ref.off, ref.lens, ref.l_pac, br.pac_of(ref), ref.holes, bq.pack_bits(cov), bq.pack_bits(jun), ids, id_cov, n_cov)


@pytest.mark.parametrize("n_cov", [1, SHARED_MAX, SHARED_MAX + 1, 12])
def test_kernel_equals_emulation(gpu_ctx, emul, ref, n_cov):
    rng = np.random.default_rng(60 + n_cov)
    n_ids = 800 if n_cov == SHARED_MAX else n_cov + 2                                    # at the threshold, a map of 28 KB: above 48 KB in all
    ids = ["r%d%s" % (k, "x" * 16 if n_cov == SHARED_MAX else "") for k in range(n_ids)]
    id_cov = [k % n_cov for k in range(n_ids)]
    pick = lambda: ids[int(rng.integers(0, len(ids)))]
    crafted = [br.with_rg(r, pick()) for r in bq.crafted(ref, rng)] + [bq.make_rec("dup_no_tag", 0x400, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50)]
    for recs, sites in ((crafted, bq.random_sites(ref, rng, 40)), ([br.with_rg(r, pick()) for r in bq.random_records(ref, rng, 3000)], bq.random_sites(ref, rng)),
                        ([], [])):
        cov, jun = bq.sites_bits(ref, sites)
        _set(gpu_ctx, ref, cov, jun, ids, id_cov, n_cov)
        for part in (recs[: len(recs) // 3], recs[len(recs) // 3:]):                      # two calls add up
            gpu_ctx.recal_add(*bq.flatten(part))
        data, starts = bq.flatten(recs)
        want, err, _ = br.emul_count_rg(emul, data, starts, ref, cov, jun, ids, id_cov, n_cov)
        assert err is None
        for c in range(n_cov):
            got = gpu_ctx.recal_tables(c)
            assert bq.same_tables(got, want[c]) and got["err_kind"] == 0 and got["ms"] >= 0, (n_cov, c)
    ok = br.with_rg(bq.make_rec("ok", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50), ids[0])
    plain = lambda name, q, n=50: bq.make_rec(name, 0, 0, 100, [(n, 0)], ref.seq(0, 100, n), q)
    for bad, kind in ((br.with_rg(plain("noq", None), ids[0]), 1), (br.with_rg(plain("long", [30] * 501, 501), ids[0]), 2),
                      (br.with_rg(plain("hiq", [94] * 50), ids[0]), 3), (plain("notag", [30] * 50), 4), (br.with_rg(plain("unknown", [30] * 50), "zz"), 5)):
        _set(gpu_ctx, ref, *bq.sites_bits(ref, []), ids, id_cov, n_cov)
        with pytest.raises(Exception) as e:
            gpu_ctx.recal_add(*bq.flatten([ok, ok, bad, ok]))
        t = gpu_ctx.recal_tables(0)
        assert (t["err_kind"], t["err_index"], t["reads"]) == (kind, 2, 3) and t["err_name"] == bu.fields(bad)["qname"] and t["err_name"] in str(e.value)


def _tool(args, code=0):
    r = subprocess.run([TOOL] + args, capture_output=True, timeout=900)
    assert r.returncode == code, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1]) if code == 0 else r.stderr.decode()


@pytest.mark.parametrize("mode,rg", [("pe", r"@RG\tID:g1\tSM:s"), ("se", r"@RG\tID:g1\tSM:s\tPU:fc.1"), ("pe", r"@RG\tID:g1\tPU:fc.3\tLB:l")])
def test_table_equals_bm2_mem_recal_file(planted, mode, rg):  # noqa: F811
    d, prefix, files, sites = planted
    w = d / ("brc_%s_%d" % (mode, len(rg))); w.mkdir()
    known = ["--known-sites", str(d / "a.vcf"), "--known-sites", str(d / "b.vcf.gz")]
    r = subprocess.run([MEM, "--recal-file", str(w / "mem.txt")] + known + ["-R", rg, "-K", "20000", prefix] + files[mode] + ["-o", str(w / "r.bam")],
                       capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    st = _tool(["-o", str(w / "t.txt")] + known + [prefix, str(w / "r.bam")])
    assert open(w / "t.txt").read() == open(w / "mem.txt").read()
    assert st["read_groups"] == 1 and st["known_sites"] == len(sites) and st["counted_reads"] > 0 and st["recal_s"] > 0


@pytest.fixture(scope="module")
def chain(planted, ref):  # noqa: F811
    """Three lanes of bm2_mem --sort, two of one library, merged and marked by bm2_markdup."""
    d, prefix, files, sites = planted
    w = d / "chain"; w.mkdir()
    rng = np.random.default_rng(71)
    pairs = mu.planted_pairs(mu.load_reference(prefix), rng, n_base=150)
    lanes = [r"@RG\tID:l1\tSM:s\tLB:a\tPU:fc.1", r"@RG\tID:l2\tSM:s\tLB:a\tPU:fc.2", r"@RG\tID:l3\tSM:s\tLB:b"]
    ins = []
    for k, rg in enumerate(lanes):
        fs, _ = tmg._write_pairs(w, [p for i, p in enumerate(pairs) if i % 3 == k], "lane%d" % k)
        ins.append(str(w / ("lane%d.bam" % k)))
        r = subprocess.run([MEM, "--sort", "-R", rg, "-K", "20000", prefix] + fs["pe"] + ["-o", ins[-1]], capture_output=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
    merged = str(w / "merged.bam")
    r = subprocess.run([mb.TOOL, "-M", str(w / "m.txt"), "-o", merged] + ins, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return w, prefix, ins, merged, sites, ["--known-sites", str(d / "a.vcf"), "--known-sites", str(d / "b.vcf.gz")]


def test_multi_lane_chain(chain, ref):  # noqa: F811
    w, prefix, ins, merged, sites, known = chain
    st = _tool(["-o", str(w / "t.txt")] + known + [prefix, merged])
    text, _, recs = mb.read_bam(merged)
    ids, id_cov, covs = br.read_groups([text])
    assert covs == ["fc.1", "fc.2", "l3"] and st["read_groups"] == 3 and st["records"] == len(recs)
    cov, jun = bq.sites_bits(ref, sites)
    tabs, err = br.count_rg(recs, ref, cov, jun, ids, id_cov, 3)
    table = open(w / "t.txt").read()
    assert err is None and table == br.report_text_rg(tabs, covs) and all(t["reads"] for t in tabs)
    # the duplicates bm2_markdup found (bm2_mem --sort marks none) are not counted
    assert not any(bu.fields(r)["flag"] & 0x400 for p in ins for r in mb.read_bam(p)[2])
    undup = [r[:18] + bytes([r[18], r[19] & ~0x04]) + r[20:] for r in recs]
    assert sum(bu.fields(r)["flag"] & 0x400 != 0 for r in recs) > 0
    assert sum(t["reads"] for t in br.count_rg(undup, ref, cov, jun, ids, id_cov, 3)[0]) > st["counted_reads"] == sum(t["reads"] for t in tabs)
    # bm2_applybqsr applies the table as Python does
    r = subprocess.run([APPLY, "--bqsr-recal-file", str(w / "t.txt"), "-o", str(w / "recal.bam"), merged], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    rgs, P, Cx, Y = au.dense(table)
    hids, id_table = au.header_map(text, rgs)
    want, aerr, *_ = au.apply_all(recs, hids, id_table, (rgs, P, Cx, Y))
    assert aerr is None and mb.read_bam(str(w / "recal.bam"))[2] == want


def test_same_bytes_in_every_setting(chain):
    w, prefix, ins, merged, sites, known = chain
    s = w / "settings"; s.mkdir()
    text, refs, recs = mb.read_bam(merged)
    mb.write_bam(str(s / "a.bam"), text, refs, recs[: len(recs) // 2])
    mb.write_bam(str(s / "b.bam"), text, refs, recs[len(recs) // 2:])
    shuffled = list(recs)
    random.Random(5).shuffle(shuffled)
    mb.write_bam(str(s / "shuf.bam"), text.replace("SO:coordinate", "SO:unsorted"), refs, shuffled)
    base = None
    for k, (args, stdin) in enumerate(((["-t", "1", merged], None), (["-t", "4", merged], None), (["--window", "64K", merged], None),
                                       (["--window", "256M", merged], None), (["-"], merged), ([str(s / "a.bam"), str(s / "b.bam")], None),
                                       ([str(s / "shuf.bam")], None))):
        out = str(s / ("t%d.txt" % k))
        argv = [TOOL, "-o", out] + known + [prefix] + args
        r = subprocess.run(argv, stdin=open(stdin, "rb") if stdin else None, capture_output=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        st = json.loads(r.stderr.decode().strip().split("\n")[-1])
        base = base or open(out).read()
        assert open(out).read() == base, args
        if "64K" in args:
            assert st["windows"] > 1


def test_errors_exit_with_their_code_and_leave_no_table(chain, ref, tmp_path):  # noqa: F811
    w, prefix, ins, merged, sites, known = chain
    text, refs, recs = mb.read_bam(merged)
    lost = bq.make_rec("lost", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50)
    mb.write_bam(str(tmp_path / "notag.bam"), text, refs, recs[:100] + [lost])
    (tmp_path / "bad.vcf").write_text("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\nnochrom\t5\t.\tA\tG\t.\t.\t.\n")
    out = str(tmp_path / "t.txt")
    for args, code, msg in (([prefix, str(tmp_path / "notag.bam")] + known, 1, "read lost has no RG tag"),
                            ([prefix, merged, "--known-sites", str(tmp_path / "bad.vcf")], 1, "bad.vcf:2: CHROM nochrom is not a contig"),
                            ([prefix, ins[0], str(tmp_path / "notag.bam")] + known, 1, "read lost has no RG tag")):
        err = _tool(["-o", out] + args, code)
        assert msg in err and not os.path.exists(out) and not os.path.exists(out + ".tmp"), err
    err = _tool(["-o", str(tmp_path / "nodir" / "t.txt"), prefix, merged] + known, 2)
    assert "cannot open" in err and not os.path.exists(tmp_path / "nodir")

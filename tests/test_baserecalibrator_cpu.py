"""bm2_baserecalibrator without a GPU: the host emulation (tests/host_emul/baserecalibrator_emul.cpp: bqsr_device.cuh's rule with the shared
read-group lookup, bqsr_recal.h's read groups, bqsr_report.h's report of several covariates, the tool's window loop) equals the rule restated
in Python (tests/baserecalibrator_util.py, over tests/bqsr_util.py's per-record rule) on crafted records for each read-group case and on
random records over 1, 3 and 12 covariates; the report of one covariate is bm2_mem --recal-file's byte for byte; the tool's usage,
reference, header, VCF and read errors."""
import os, struct, subprocess
import numpy as np
import pytest
import baserecalibrator_util as br
import bqsr_util as bq

ROOT = bq.ROOT
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_baserecalibrator")
IDX = os.path.join(ROOT, "tests", "golden", "c0_index", "ref.fa")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return br.build_rg_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def old_emul(tmp_path_factory):
    return bq.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def ref():
    return bq.Ref(IDX)


def header(ref, rgs, so="unsorted"):
    return "@HD\tVN:1.6\tSO:%s\n" % so + "".join("@SQ\tSN:%s\tLN:%d\n" % (n, l) for n, l in zip(ref.names, ref.lens)) + "".join(r + "\n" for r in rgs)


def write_bam(path, ref, text, recs, refs=None):
    refs = refs if refs is not None else list(zip(ref.names, ref.lens))
    h = b"BAM\x01" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for n, ln in refs:
        h += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", ln)
    with open(path, "wb") as f:
        f.write(bq.bgzf(h + b"".join(recs)))
    return str(path)


RGS = ["@RG\tID:a\tSM:s\tPU:fc.1", "@RG\tID:b\tSM:s\tPU:fc.1", "@RG\tID:c\tSM:s", "@RG\tID:d\tSM:s\tPU:c", "@RG\tID:e\tSM:t\tPU:fc.2"]


def check(emul, ref, recs, sites, texts):
    ids, id_cov, covs = br.read_groups(texts)
    assert br.emul_read_groups(emul, texts, ["in%d" % k for k in range(len(texts))]) == (ids, id_cov, covs)
    cov, jun = bq.sites_bits(ref, sites)
    data, starts = bq.flatten(recs)
    got, err, msg = br.emul_count_rg(emul, data, starts, ref, cov, jun, ids, id_cov, len(covs))
    want, werr = br.count_rg(recs, ref, cov, jun, ids, id_cov, len(covs))
    assert err == werr
    for g, w in zip(got, want):
        assert bq.same_tables(g, w)
    assert br.emul_report_rg(emul, got, covs) == br.report_text_rg(want, covs)
    return got, err, msg, covs


def test_read_group_cases(emul, ref):
    rng = np.random.default_rng(21)
    ok = lambda name, v, pos=100, flag=0: br.with_rg(bq.make_rec(name, flag, 0, pos, [(50, 0)], bq.mutate(ref.seq(0, pos, 50), rng, 0.05),
                                                                   [30] * 50), v)
    texts = [header(ref, RGS)]
    assert br.read_groups(texts)[2] == ["c", "fc.1", "fc.2"]                                  # PU, else ID, in byte order
    recs = [ok("a1", "a"), ok("b1", "b", 300), ok("c1", "c", 500), ok("d1", "d", 700), ok("e1", "e", 900)]
    filtered = bq.make_rec("dup_no_tag", 0x400, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50)
    got, err, _, covs = check(emul, ref, recs + [filtered, br.with_rg(bq.make_rec("unm", 4, -1, -1, [], "ACGT", None), "zz")], [], texts)
    assert err is None and [t["reads"] for t in got] == [2, 2, 1]                           # a and b share fc.1, c and d share c
    no_tag = bq.make_rec("no_tag", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50)
    unknown = ok("unknown", "zz")
    noq_unknown = br.with_rg(bq.make_rec("noq", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), None), "zz")
    empty_no_tag = bq.make_rec("empty", 0, 0, 3500, [(50, 4), (10, 2), (50, 4)], "A" * 100, [30] * 100)
    for bad, kind, text in ((no_tag, 4, "has no RG tag"), (unknown, 5, "not an @RG ID"), (noq_unknown, 5, "not an @RG ID"),
                            (empty_no_tag, 4, "has no RG tag"), (br.with_rg(bq.make_rec("noq2", 0, 0, 100, [(50, 0)], "A" * 50, None), "a"), 1, "qualities")):
        _, err, msg, _ = check(emul, ref, recs[:2] + [bad] + recs[2:], [], texts)
        assert err == (2, kind) and bq.bu.fields(bad)["qname"] in msg and text in msg, (kind, msg)
    # the same ID in two headers: one entry; an ID with two covariates, or a header without @RG, is an error
    assert br.read_groups([header(ref, RGS[:2]), header(ref, RGS[1:])])[0] == ["a", "b", "c", "d", "e"]
    for texts, msg in (([header(ref, RGS), header(ref, ["@RG\tID:a\tPU:other"])], "read group a has covariate other here and fc.1 in in0"),
                       ([header(ref, RGS), header(ref, [])], "in1: the header has no @RG line")):
        with pytest.raises(ValueError) as e:
            br.emul_read_groups(emul, texts, ["in0", "in1"])
        assert msg in str(e.value)
        with pytest.raises(ValueError):
            br.read_groups(texts)


@pytest.mark.parametrize("n_cov", [1, 3, 12])
def test_random_records_over_covariates(emul, ref, n_cov):
    rng = np.random.default_rng(30 + n_cov)
    rgs = ["@RG\tID:r%d\tSM:s\tPU:u.%d" % (k, k % n_cov) for k in range(n_cov + 2)]
    ids = ["r%d" % k for k in range(n_cov + 2)]
    recs = [br.with_rg(r, ids[int(rng.integers(0, len(ids)))]) for r in bq.random_records(ref, rng, 1200)]
    got, err, _, covs = check(emul, ref, recs, bq.random_sites(ref, rng), [header(ref, rgs)])
    assert err is None and len(covs) == n_cov and all(t["reads"] > 0 for t in got)


def test_one_covariate_report_is_recal_file_report(emul, old_emul, ref):
    rng = np.random.default_rng(41)
    recs = bq.random_records(ref, rng, 800)
    cov, jun = bq.sites_bits(ref, bq.random_sites(ref, rng))
    t = bq.count(recs, ref, cov, jun)
    for name in ("g1", "flow.cell.3"):
        want = bq.report_text(t, name)
        assert br.emul_report_rg(emul, [t], [name]) == want == bq.emul_report(old_emul, t, name) == br.report_text_rg([t], [name])
    assert br.emul_report_rg(emul, [t, br.empty_tables()], ["a", "b"]) == bq.report_text(t, "a")     # a covariate with no rows


def _inputs(ref, d, rng, n=1500):
    ids = ["l1", "l2", "l3"]
    rgs = ["@RG\tID:l1\tSM:s\tPU:fc.1", "@RG\tID:l2\tSM:s\tPU:fc.2", "@RG\tID:l3\tSM:s\tLB:x"]
    recs = [br.with_rg(r, ids[int(rng.integers(0, 3))]) for r in bq.random_records(ref, rng, n)]
    sites = bq.random_sites(ref, rng)
    (d / "a.vcf").write_text(bq.vcf_text(ref, sites[::2]))
    (d / "b.vcf.bgz").write_bytes(bq.bgzf(bq.vcf_text(ref, sites[1::2]).encode()))
    return recs, rgs, sites, [str(d / "a.vcf"), str(d / "b.vcf.bgz")]


def test_tool_emulation_equals_python(emul, ref, tmp_path):
    rng = np.random.default_rng(43)
    recs, rgs, sites, vcfs = _inputs(ref, tmp_path, rng)
    one = write_bam(tmp_path / "one.bam", ref, header(ref, rgs), recs)
    a = write_bam(tmp_path / "a.bam", ref, header(ref, rgs[:2]), recs[:700])
    b = write_bam(tmp_path / "b.bam", ref, header(ref, rgs[1:]), recs[700:])
    ids, id_cov, covs = br.read_groups([header(ref, rgs)])
    cov, jun = bq.sites_bits(ref, sites)
    want = br.report_text_rg(br.count_rg(recs, ref, cov, jun, ids, id_cov, len(covs))[0], covs)
    for inputs, window in (([one], 1 << 28), ([one], 1 << 16), ([one], 1), ([a, b], 1 << 16)):
        text, st = br.emul_run(emul, IDX, inputs, vcfs, window)
        assert text == want and st["records"] == len(recs) and st["read_groups"] == 3 and st["known_sites"] == len(sites)
    assert br.emul_run(emul, IDX, [one], vcfs, 1 << 14)[1]["windows"] > 3


def test_tool_emulation_errors(emul, ref, tmp_path):
    rng = np.random.default_rng(47)
    recs, rgs, sites, vcfs = _inputs(ref, tmp_path, rng, 50)
    text = header(ref, rgs)
    good = write_bam(tmp_path / "good.bam", ref, text, recs)
    no_tag = bq.make_rec("lost", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50)
    past = br.with_rg(bq.make_rec("past", 0, 0, ref.lens[0] - 20, [(50, 0)], "A" * 50, [30] * 50), "l1")
    (tmp_path / "bad.vcf").write_text("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\nnochrom\t5\t.\tA\tG\t.\t.\t.\n")
    cases = [([str(tmp_path / "nope.bam")], vcfs, "cannot open"),
             ([write_bam(tmp_path / "norg.bam", ref, header(ref, []), recs)], vcfs, "the header has no @RG line"),
             ([good, write_bam(tmp_path / "clash.bam", ref, header(ref, ["@RG\tID:l1\tPU:zz"]), [])], vcfs, "read group l1 has covariate zz"),
             ([write_bam(tmp_path / "sq.bam", ref, text, recs, refs=[("chrX", 10)])], vcfs, "reference 0 is chrX of length 10 in the header"),
             ([good], [str(tmp_path / "bad.vcf")], "bad.vcf:2: CHROM nochrom is not a contig"),
             ([write_bam(tmp_path / "notag.bam", ref, text, recs[:5] + [no_tag])], vcfs, "read lost has no RG tag"),
             ([write_bam(tmp_path / "unk.bam", ref, text, [br.with_rg(no_tag, "l9")])], vcfs, "read lost has an RG tag that is not an @RG ID"),
             ([write_bam(tmp_path / "past.bam", ref, text, [past])], vcfs, "read past is malformed: its alignment is not inside contig 0"),
             ([str(tmp_path / "a.vcf")], vcfs, "not BGZF")]
    for inputs, v, msg in cases:
        with pytest.raises(ValueError) as e:
            br.emul_run(emul, IDX, inputs, v)
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(ValueError) as e:
        br.emul_run(emul, str(tmp_path / "noindex"), [good], vcfs)
    assert "cannot open" in str(e.value) and ".ann" in str(e.value)


def _run(args):
    return subprocess.run([TOOL] + args, capture_output=True, timeout=120)


@pytest.mark.skipif(not os.path.exists(TOOL), reason="bm2_baserecalibrator not built")
def test_usage_reference_and_header_errors(ref, tmp_path):
    rng = np.random.default_rng(49)
    recs, rgs, sites, vcfs = _inputs(ref, tmp_path, rng, 20)
    good = write_bam(tmp_path / "good.bam", ref, header(ref, rgs), recs)
    norg = write_bam(tmp_path / "norg.bam", ref, header(ref, []), recs)
    o = str(tmp_path / "t.txt")
    ks = ["--known-sites", vcfs[0]]
    for args, msg in (([], "no index prefix"), ([IDX], "no input BAM"), ([IDX, good] + ks, "no output table (-o)"),
                      (["-o", o, IDX, good], "at least one --known-sites is required"), (["-o", o, IDX, "-", "-"] + ks, "standard input (-) can be only one"),
                      (["-o", o, "-t", "0", IDX, good] + ks, "-t takes"), (["-o", o, "--window", "1X", IDX, good] + ks, "--window takes"),
                      (["-o", o, "--bogus", IDX, good] + ks, "unknown option --bogus"), (["-o", o, IDX, good, "--known-sites"], "takes a value"),
                      (["-o", o, str(tmp_path / "noidx"), good] + ks, "cannot open"), (["-o", o, IDX, norg] + ks, "has no @RG line"),
                      (["-o", o, IDX, str(tmp_path / "missing.bam")] + ks, "cannot open")):
        r = _run(args)
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr)
    assert sorted(os.listdir(tmp_path)) == sorted(["a.vcf", "b.vcf.bgz", "good.bam", "norg.bam"])

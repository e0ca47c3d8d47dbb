"""bm2_mem --recal-file without a GPU: the host emulation (tests/host_emul/bqsr_emul.cpp: bqsr_device.cuh's per-record rule, bqsr_report.h's
empirical quality and report text, known_sites.h's VCF reader) equals the rule restated in Python (tests/bqsr_util.py) on crafted records for
each rule and on random ones; the empirical quality equals Python's on a grid including n > 2^31; the VCF reader takes plain, gzip and BGZF
files, several files and header-only ones, and names each error by file and line.  Plus the option errors and --dump-opt."""
import gzip, json, os, subprocess
import numpy as np
import pytest
import bqsr_util as bq

ROOT = bq.ROOT
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
IDX = os.path.join(ROOT, "tests", "golden", "c0_index", "ref.fa")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return bq.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def ref():
    return bq.Ref(IDX)


def _sites(ref, recs, rng):
    """Sites over part of the records' spans, single- and multi-base, plus random ones."""
    sites = bq.random_sites(ref, rng, every=40)
    for r in recs[::3]:
        f = bq.bu.fields(r)
        if f["rid"] >= 0 and not f["flag"] & 4:
            sites.append((f["rid"], f["pos"] + 20, 1))
            sites.append((f["rid"], f["pos"] + 41, 3))
    return sites


def _check(emul, ref, recs, cov, jun, rg="g1"):
    data, starts = bq.flatten(recs)
    got = bq.emul_count(emul, data, starts, ref, cov, jun)
    want = bq.count(recs, ref, cov, jun)
    assert bq.same_tables(got, want) and got["err"] == want["err"]
    assert bq.emul_report(emul, got, rg) == bq.report_text(want, rg)
    return got


def test_crafted_records_equal_python(emul, ref):
    rng = np.random.default_rng(5)
    recs = bq.crafted(ref, rng)
    cov, jun = bq.sites_bits(ref, _sites(ref, recs, rng))
    t = _check(emul, ref, recs, cov, jun)
    by = {bq.bu.fields(r)["qname"]: bq.record_bases(r, ref, cov, jun) for r in recs}
    for name in ("flag_4", "flag_100", "flag_800", "flag_400", "flag_200", "mapq0", "mapq255"):
        assert by[name][0] == 4, name
    assert by["clipped_to_nothing"][0] == 5 and len(by["adapt_rev_two_left"][1]) <= 2
    assert len(by["adapt_fwd"][1]) <= 90 and len(by["adapt_rev"][1]) <= 90                 # clipped at the mate's end
    assert len(by["adapt_t0"][1]) > 80 and len(by["adapt_same_strand"][1]) > 80
    assert all(c < 0 for _, _, c, _ in by["second_of_pair"][1]) and all(c > 0 for _, _, c, _ in by["first_of_pair"][1])
    assert any(e for *_, e in by["hole"][1])                                                 # the hole's N is an error
    assert all(q >= 6 for q, *_ in by["low_quals"][1])
    assert t["reads"] > 20 and t["bases"] > 1000 and t["err"] is None
    # with no sites, more bases; a site under every base: none
    t0 = _check(emul, ref, recs, np.zeros(ref.l_pac, bool), np.zeros(ref.l_pac, bool))
    assert t0["bases"] > t["bases"]
    ta = _check(emul, ref, recs, np.ones(ref.l_pac, bool), np.ones(ref.l_pac, bool))
    assert ta["bases"] == 0 and ta["reads"] == t["reads"]


def test_sites_next_to_and_inside_indels(emul, ref):
    rng = np.random.default_rng(6)
    recs = [bq.make_rec("ins", 0, 0, 9000, [(30, 0), (3, 1), (30, 0)], ref.seq(0, 9000, 30) + "GGG" + ref.seq(0, 9030, 30), [30] * 63),
            bq.make_rec("del", 16, 0, 9100, [(30, 0), (4, 2), (30, 0)], ref.seq(0, 9100, 30) + ref.seq(0, 9134, 30), [30] * 60)]
    for sites in ([(0, 9030, 1)], [(0, 9031, 1)], [(0, 9030, 2)], [(0, 9029, 3)], [(0, 9128, 6)], [(0, 9131, 2)], [(0, 9125, 12)]):
        cov, jun = bq.sites_bits(ref, sites)
        _check(emul, ref, recs, cov, jun)
    base = len(bq.record_bases(recs[0], ref, *bq.sites_bits(ref, []))[1])
    assert len(bq.record_bases(recs[0], ref, *bq.sites_bits(ref, [(0, 9030, 2)]))[1]) == base - 2 - 3   # the junction 9029|9030 (0-based)
    assert len(bq.record_bases(recs[0], ref, *bq.sites_bits(ref, [(0, 9030, 1)]))[1]) == base - 1       # one base: no junction


def test_read_errors_equal_python(emul, ref):
    rng = np.random.default_rng(7)
    ok = bq.make_rec("ok", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50)
    noq = bq.make_rec("noq", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), None)
    long_ = bq.make_rec("long", 0, 0, 100, [(501, 0)], ref.seq(0, 100, 501), [30] * 501)
    long_clipped = bq.make_rec("long_clipped", 0, 0, 100, [(2, 4), (500, 0), (3, 4)], "A" * 2 + ref.seq(0, 100, 500) + "A" * 3, [30] * 505)
    hiq = bq.make_rec("hiq", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 49 + [94])
    unm_noq = bq.make_rec("unm", 4, -1, -1, [], "ACGT", None)
    cov, jun = bq.sites_bits(ref, [])
    for recs, want in (([ok, noq, long_], (1, 1)), ([ok, long_], (1, 2)), ([hiq, noq], (0, 3)), ([ok, long_clipped, unm_noq], None)):
        t = _check(emul, ref, recs, cov, jun)
        assert t["err"] == want


def test_random_records_equal_python(emul, ref):
    rng = np.random.default_rng(8)
    recs = bq.random_records(ref, rng, 1500)
    cov, jun = bq.sites_bits(ref, bq.random_sites(ref, rng))
    t = _check(emul, ref, recs, cov, jun, rg="unit.1")
    assert t["bases"] > 50_000 and t["cyc_obs"][:, :bq.MAXC].sum() > 0


def test_empirical_quality_equals_python(emul):
    for n in (0, 1, 2, 10, 37, 100, 1000, 123_456, 10**7, 2**31 - 3, 2**31 - 2, 2**31, 3 * 2**31 + 7, 10**12):
        for frac in (0, 1e-6, 1e-4, 1e-3, 0.01, 0.1, 0.5, 1.0):
            e = int(n * frac)
            for prior in (0, 2, 6, 12, 20.5, 30, 37, 41, 60, 93, 27.183):
                assert emul.bqsr_emul_empirical(n, e, prior) == bq.empirical_q(n, e, prior), (n, e, prior)
    assert bq.empirical_q(10**6, 1000, 30) == 30 and bq.empirical_q(10**6, 10**5, 30) in (10, 11)


def test_read_group_covariate(emul):
    for line in (r"@RG\tID:g1\tSM:s", r"@RG\tID:g1\tPU:flow.3\tSM:s", r"@RG\tPU:x\tID:y"):
        assert bq.emul_read_group(emul, line.replace("\\t", "\t")) == bq.read_group(line)


def test_vcf_reader(emul, ref, tmp_path):
    rng = np.random.default_rng(9)
    sites = bq.random_sites(ref, rng)
    a, b = sites[::2], sites[1::2]
    text_a, text_b = bq.vcf_text(ref, a), bq.vcf_text(ref, b)
    (tmp_path / "a.vcf").write_text(text_a)
    (tmp_path / "b.vcf.gz").write_bytes(gzip.compress(text_b.encode()))
    (tmp_path / "b.vcf.bgz").write_bytes(bq.bgzf(text_b.encode()))
    (tmp_path / "h.vcf").write_text(bq.vcf_text(ref, [], header=True))
    (tmp_path / "crlf.vcf").write_text(text_a.replace("\n", "\r\n"))
    want = bq.sites_bits(ref, sites)
    for files in (["a.vcf", "b.vcf.gz"], ["a.vcf", "b.vcf.bgz", "h.vcf"], ["b.vcf.bgz", "crlf.vcf"]):
        cov, jun, n = bq.emul_sites(emul, [str(tmp_path / f) for f in files], ref)
        assert np.array_equal(cov, want[0]) and np.array_equal(jun, want[1]) and n == len(sites)
    cov, jun, n = bq.emul_sites(emul, [str(tmp_path / "h.vcf")], ref)
    assert n == 0 and not cov.any() and not jun.any()
    hdr = "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n"
    name, ln = ref.names[1], ref.lens[1]
    bad = {"chrom": ("chrZ\t10\t.\tA\tG\t.\t.\t.\n", "CHROM chrZ is not a contig"),
           "past_end": ("%s\t%d\t.\tAC\tG\t.\t.\t.\n" % (name, ln), "past the contig's end"),
           "columns": ("%s\t10\t.\tA\tG\n" % name, "8 tab-separated fixed columns"),
           "pos": ("%s\t1x\t.\tA\tG\t.\t.\t.\n" % name, "POS is not a positive integer"),
           "pos0": ("%s\t0\t.\tA\tG\t.\t.\t.\n" % name, "POS is not a positive integer"),
           "ref": ("%s\t10\t.\t\tG\t.\t.\t.\n" % name, "REF is empty")}
    for k, (line, msg) in bad.items():
        p = tmp_path / ("bad_%s.vcf" % k)
        p.write_text(hdr + "%s\t5\t.\tA\tG\t.\t.\t.\n" % name + line)
        with pytest.raises(ValueError) as e:
            bq.emul_sites(emul, [str(tmp_path / "a.vcf"), str(p)], ref)
        assert str(p) + ":4: " in str(e.value) and msg in str(e.value), (k, str(e.value))
    ok = "%s\t%d\t.\tAC\tG\t.\t.\t.\n" % (name, ln - 1)                                 # ends on the contig's last base
    (tmp_path / "edge.vcf").write_text(hdr + ok)
    assert bq.emul_sites(emul, [str(tmp_path / "edge.vcf")], ref)[2] == 1
    with pytest.raises(ValueError):
        bq.emul_sites(emul, [str(tmp_path / "missing.vcf")], ref)


def _run(args):
    return subprocess.run([TOOL] + args, capture_output=True, timeout=120)


@pytest.mark.skipif(not os.path.exists(TOOL), reason="bm2_mem not built")
def test_options_and_dump_opt(tmp_path):
    fq = tmp_path / "r.fq"
    fq.write_text("@a\nACGT\n+\nIIII\n")
    rg = r"@RG\tID:g1\tSM:s"
    for args, msg in ((["--known-sites", "a.vcf"], "--known-sites needs --recal-file"),
                      (["--recal-file", "x.txt"], "needs at least one --known-sites"),
                      (["--recal-file", "x.txt", "--known-sites", "a.vcf"], "needs a read group (-R)"),
                      ([IDX, str(fq), "--recal-file"], "--recal-file takes a file name"),
                      ([IDX, str(fq), "-R", rg, "--recal-file", "x", "--known-sites"], "takes a VCF")):
        r = _run(args + ([] if args[0] == IDX else [IDX, str(fq)]))
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr)
    r = _run(["--recal-file", "t.txt", "--known-sites", "a.vcf", "--known-sites", "b.vcf.gz", "-R", rg, "--dump-opt", IDX, str(fq)])
    assert r.returncode == 0, r.stderr
    d = json.loads(r.stdout)
    assert d["recal_file"] == "t.txt" and d["known_sites"] == ["a.vcf", "b.vcf.gz"] and d["markdup"] and d["sort"] and d["bam"]
    r = _run(["--markdup", "--dump-opt", IDX, str(fq)])
    d = json.loads(r.stdout)
    assert "recal_file" not in d and "known_sites" not in d

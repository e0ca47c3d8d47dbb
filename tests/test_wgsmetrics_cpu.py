"""bm2_wgsmetrics without a GPU: the host emulation (tests/host_emul/wgsmetrics_emul.cpp: wgs.cu's check, count and overlap phases with the
carry between windows over wgs_device.cuh's rule, wgs_metrics.h's reference reader, checks and text) equals Picard's per-locus loop restated
in Python (tests/wgsmetrics_util.py) on crafted records for each filter and overlap case, under a forced hash collision, on 2 000 random
pairs at every window size down to one record per window, and on the metrics of small histograms; every read, header and order error is
named; the tool rejects every bad option."""
import os, subprocess
import numpy as np
import pytest
import wgsmetrics_util as wm

M, I, D, N, S, H, EQ, X = 0, 1, 2, 3, 4, 5, 7, 8
REF = wm.Ref([("c1", 3000), ("c2", 2000), ("empty", 500)], holes=[(100, 20, "N"), (300, 10, "n"), (400, 5, "R"), (3100, 8, "."), (3200, 4, "Y")])


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return wm.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def emul_collide(tmp_path_factory):
    return wm.build_emul(tmp_path_factory, collide=True)


def q(n, v=30):
    return [v] * n


def crafted():
    """Records for each filter, overlap and locus case, coordinate-sorted."""
    P = 0x1 | 0x40 | 0x20
    P2 = 0x1 | 0x80 | 0x10
    r = [
        wm.rec("sec_mapq0", 0x100 | P, 0, 500, [(50, M)], q(50), mapq=0),          # MAPQ first: EXC_MAPQ
        wm.rec("dup_lowmapq", 0x400 | P, 0, 510, [(40, M)], q(40), mapq=10),       # EXC_MAPQ, not EXC_DUPE
        wm.rec("dup", 0x400 | P, 0, 520, [(40, M)], q(40)),                        # EXC_DUPE
        wm.rec("dup_nomate", 0x400, 0, 530, [(40, M)], q(40)),                     # EXC_DUPE before EXC_UNPAIRED
        wm.rec("unpaired", 0, 0, 540, [(40, M)], q(40)),
        wm.rec("mate_unmapped", 0x1 | 0x8 | 0x40, 0, 550, [(40, M)], q(40)),
        wm.rec("secondary", 0x100 | P, 0, 560, [(40, M)], q(40)),                 # dropped
        wm.rec("qcfail", 0x200 | P, 0, 570, [(40, M)], q(40)),                    # skipped
        wm.rec("suppl", 0x800 | P, 0, 580, [(40, M)], q(40)),                     # counted
        # overlapping mates: plain, inside a deletion / insertion, soft clips at the ends
        wm.rec("ov", P, 0, 1000, [(100, M)], q(100)), wm.rec("ov", P2, 0, 1050, [(100, M)], q(100)),
        wm.rec("ovdel", P, 0, 1200, [(40, M), (10, D), (40, M)], q(80)), wm.rec("ovdel", P2, 0, 1230, [(5, S), (60, M)], q(65)),
        wm.rec("ovins", P, 0, 1400, [(30, M), (5, I), (30, M)], q(65)), wm.rec("ovins", P2, 0, 1420, [(20, M), (3, I), (20, M), (7, S)], q(50)),
        wm.rec("ovskip", P, 0, 1500, [(20, M), (30, N), (20, EQ)], q(40)), wm.rec("ovskip", P2, 0, 1510, [(10, S), (40, X)], q(50)),
        # one mate low-quality where they overlap: the other counts
        wm.rec("lowq", P, 0, 1600, [(60, M)], q(30, 10) + q(30)), wm.rec("lowq", P2, 0, 1600, [(60, M)], q(60)),
        # three records of one name
        wm.rec("three", P, 0, 1700, [(60, M)], q(60)), wm.rec("three", 0x800 | P, 0, 1720, [(60, M)], q(60)),
        wm.rec("three", P2, 0, 1740, [(60, M)], q(60)),
        # read base N and a quality exactly at the threshold
        wm.rec("nbase", P, 0, 1800, [(20, M)], q(20), seq="ACGTN" * 4), wm.rec("atq", P, 0, 1810, [(20, M)], [19, 20] * 10),
        # holes: N and n are no-call, R is not; a read ending on the contig's last base; hard clips
        wm.rec("hole_n", P, 0, 90, [(50, M)], q(50)), wm.rec("hole_lc", P, 0, 295, [(20, M)], q(20)), wm.rec("hole_r", P, 0, 398, [(10, M)], q(10)),
        wm.rec("lastbase", P, 0, 2950, [(5, H), (50, M)], q(50)),
        wm.rec("c2_dot", P, 1, 95, [(20, M)], q(20)), wm.rec("c2_y", P, 1, 198, [(10, M)], q(10)),
        wm.rec("unmapped", 0x4, -1, -1, [], q(30), seq="A" * 30),
    ]
    # a pile deeper than the cap, with duplicates and secondaries mixed in
    r += [wm.rec("deep%d" % k, P, 0, 2000 + (k % 3), [(30, M)], q(30)) for k in range(40)]
    return wm.sort_recs(r)


def _py(recs, **kw):
    return wm.metrics(recs, REF, **kw)


def _same(e, p):
    return e[3] is None and p[3] is None and np.array_equal(e[0], p[0]) and e[1] == p[1] and e[2] == p[2]


@pytest.mark.parametrize("kw", [{}, dict(count_unpaired=True), dict(min_mapq=0, min_baseq=0, cap=10, count_unpaired=True), dict(cap=1)])
def test_crafted_equals_python(emul, kw):
    recs = crafted()
    want = _py(recs, **kw)
    for sizes in ([len(recs)], [1], [2, 3], [7]):
        got = wm.emul_run(emul, REF, wm.windows(recs, sizes), **kw)
        assert _same(got, want), (kw, sizes)
    hist, exc = want[0], want[1]
    if not kw:
        assert all(x > 0 for x in exc[:5]) and exc[5] == 0                        # the cap of 250 is not reached
        assert hist[0] > 0 and (REF.nocall.sum() == 20 + 10 + 8)
    if kw.get("cap") == 10:
        assert exc[5] > 0 and exc[0] == 0 and exc[2] == 0 and hist[10] >= 30
    assert wm.emul_text(emul, hist, exc, "a b") == wm.text(hist, exc, "a b")


def test_each_rule(emul):
    P, P2 = 0x1 | 0x40 | 0x20, 0x1 | 0x80 | 0x10
    one = lambda recs, **kw: _py(wm.sort_recs(recs), **kw)
    assert one([wm.rec("s", 0x100 | P, 0, 500, [(50, M)], q(50), mapq=0)])[1][0] == 50
    assert one([wm.rec("s", 0x400 | P, 0, 500, [(50, M)], q(50), mapq=19)])[1][:2] == [50, 0]
    assert one([wm.rec("s", 0x400, 0, 500, [(50, M)], q(50))])[1][1:3] == [50, 0]
    assert one([wm.rec("s", 0x1 | 0x8, 0, 500, [(50, M)], q(50))])[1][2] == 50
    assert one([wm.rec("s", 0x1 | 0x8, 0, 500, [(50, M)], q(50))], count_unpaired=True)[1][2] == 0
    assert sum(one([wm.rec("s", 0x100 | P, 0, 500, [(50, M)], q(50))])[0][1:]) == 0
    assert one([wm.rec("a", P, 0, 500, [(50, M)], q(50)), wm.rec("a", P2, 0, 520, [(50, M)], q(50))])[1][4] == 30
    assert one([wm.rec("a", P, 0, 500, [(50, M)], q(50)), wm.rec("b", P2, 0, 520, [(50, M)], q(50))])[1][4] == 0
    assert one([wm.rec("a", P, 0, 500, [(10, M)], [19] * 5 + [20] * 5)])[1][3] == 5
    assert one([wm.rec("a", P, 0, 95, [(10, M)], q(10))])[1][0] == 0 and one([wm.rec("a", P, 0, 95, [(10, M)], q(10))])[0][1] == 5
    h = one([wm.rec("a", P, 0, 400, [(5, M)], q(5))])[0]
    assert h[1] == 5                                                            # an R hole is an ordinary locus
    deep = one([wm.rec("d%d" % k, P, 0, 600, [(10, M)], q(10)) for k in range(30)], cap=25)
    assert deep[1][5] == 50 and deep[0][25] == 10


def test_hash_collision(emul_collide, emul):
    recs = crafted() + [wm.rec("zz%d" % k, 0x1 | 0x40, 1, 900, [(30, M)], q(30)) for k in range(5)]
    recs = wm.sort_recs(recs)
    want = _py(recs)
    for lib in (emul, emul_collide):
        for sizes in ([len(recs)], [1], [5]):
            assert _same(wm.emul_run(lib, REF, wm.windows(recs, sizes)), want)
    assert want[1][4] > 0


def test_random_pairs_every_window(emul):
    rng = np.random.default_rng(81)
    recs = wm.random_pairs(REF, rng, 2000)
    for kw in ({}, dict(min_mapq=0, min_baseq=0, cap=10, count_unpaired=True)):
        want = _py(recs, **kw)
        assert want[3] is None and want[1][4] > 1000
        carried = []
        for sizes in ([len(recs)], [1], [2], [17], [1000], [3, 1, 250]):
            got = wm.emul_run(emul, REF, wm.windows(recs, sizes), **kw)
            assert _same(got, want), (kw, sizes)
            carried.append(got[5])
        assert carried[0] == 0 and max(carried) > 1


def test_metrics_text_small_histograms(emul):
    for hist in ([0, 0, 0], [4, 0, 0], [0, 1, 0], [1, 1, 0], [1, 2, 3], [5, 0, 1], [2, 2, 2, 2], [0, 0, 0, 7], [3, 1, 0, 0, 0, 9]):
        for exc in ([0] * 6, [1, 2, 3, 4, 5, 6]):
            assert wm.emul_text(emul, np.array(hist), exc, "") == wm.text(np.array(hist), exc, "")
    t = wm.text(np.array([1, 1, 0]), [0] * 6, "x").split("\n")
    cols, vals = t[4].split("\t"), t[5].split("\t")
    v = dict(zip(cols, vals))
    assert (v["GENOME_TERRITORY"], v["MEAN_COVERAGE"], v["MEDIAN_COVERAGE"], v["MAD_COVERAGE"]) == ("2", "0.5", "0.5", "0.5")
    assert v["SD_COVERAGE"] == "0.707107" and v["HET_SNP_Q"] == "" and len(cols) == len(vals) == 28
    v = dict(zip(cols, wm.text(np.array([1, 2, 3]), [0] * 6, "").split("\n")[5].split("\t")))
    assert (v["MEDIAN_COVERAGE"], v["MAD_COVERAGE"], v["PCT_1X"]) == ("1.5", "0.5", "0.833333")
    v = dict(zip(cols, wm.text(np.array([0, 1, 0]), [0] * 6, "").split("\n")[5].split("\t")))
    assert (v["MEDIAN_COVERAGE"], v["SD_COVERAGE"]) == ("1", "0")


def test_read_errors(emul):
    P = 0x1 | 0x40 | 0x20
    ok = wm.rec("ok", P, 0, 100, [(10, M)], q(10))
    cases = [(wm.rec("noq", P, 0, 200, [(10, M)], None), "read noq (record 1) has no base qualities"),
             (wm.rec("lseq0", P, 0, 200, [(10, D)], [], seq=""), "read lseq0 (record 1) has no base qualities"),
             (wm.rec("past", P, 0, 2995, [(10, M)], q(10)), "read past (record 1) does not lie inside a contig"),
             (wm.rec("badrid", P, 3, 5, [(10, M)], q(10)), "read badrid (record 1) does not lie inside a contig"),
             (wm.rec("badcig", P, 0, 200, [(10, M), (2, I)], q(10) + [], seq="A" * 10), "read badcig (record 1) has a CIGAR that does not match")]
    for bad, msg in cases:
        recs = [ok, bad, ok]
        want = _py(recs)
        assert want[3] is not None and want[3][0] == 1
        got = wm.emul_run(emul, REF, [recs], check_order=False)
        assert got[3] is not None and msg in got[3], (msg, got[3])
    # a filtered record without qualities is not an error; one past its contig's end is
    assert _py([wm.rec("f", 0x400 | P, 0, 200, [(10, M)], None)])[3] is None
    assert _py([wm.rec("f", 0x400 | P, 0, 2995, [(10, M)], q(10))])[3][1] == 2
    got = wm.emul_run(emul, REF, [[wm.rec("b", P, 0, 500, [(10, M)], q(10)), wm.rec("a", P, 0, 400, [(10, M)], q(10))]])
    assert "read a is out of coordinate order" in got[3]


def test_tool_emulation_over_files(emul, tmp_path):
    rng = np.random.default_rng(82)
    REF.write(str(tmp_path / "ref.fa"))
    assert wm.Ref.read(str(tmp_path / "ref.fa")).holes == REF.holes
    recs = wm.random_pairs(REF, rng, 600)
    (tmp_path / "in.bam").write_bytes(wm.bam_bytes(REF, recs))
    hist, exc, _, _ = _py(recs)
    want = wm.text(hist, exc, "x")
    for window in (1, 4096, 1 << 30):
        t, st = wm.emul_tool(emul, str(tmp_path / "ref.fa"), str(tmp_path / "in.bam"), window=window, args="x")
        assert t == want and st["records"] == len(recs)
    (tmp_path / "empty.bam").write_bytes(wm.bam_bytes(REF, []))                     # header only: every locus at depth 0
    t, _ = wm.emul_tool(emul, str(tmp_path / "ref.fa"), str(tmp_path / "empty.bam"))
    h0 = np.zeros(251, np.int64); h0[0] = REF.l_pac - REF.nocall.sum()
    assert t == wm.text(h0, [0] * 6, "")
    bad = {"unsorted.bam": (wm.bam_bytes(REF, recs, text="@HD\tVN:1.6\tSO:queryname\n"), "not coordinate-sorted (@HD SO:queryname)"),
           "nohd.bam": (wm.bam_bytes(REF, recs, text="@CO\tx\n"), "not coordinate-sorted"),
           "names.bam": (wm.bam_bytes(REF, recs, refs=[("c1", 3000), ("cX", 2000), ("empty", 500)]), "reference 1 is cX of length 2000 in the header"),
           "lens.bam": (wm.bam_bytes(REF, recs, refs=[("c1", 3000), ("c2", 2001), ("empty", 500)]), "reference 1 is c2 of length 2001"),
           "count.bam": (wm.bam_bytes(REF, recs, refs=[("c1", 3000), ("c2", 2000)]), "the header has 2 references, the index 3 contigs"),
           "order.bam": (wm.bam_bytes(REF, recs[::-1]), "out of coordinate order")}
    for name, (data, msg) in bad.items():
        (tmp_path / name).write_bytes(data)
        with pytest.raises(ValueError) as e:
            wm.emul_tool(emul, str(tmp_path / "ref.fa"), str(tmp_path / name))
        assert msg in str(e.value), (name, str(e.value))
    with pytest.raises(ValueError, match="cannot open .*nothere.ann"):
        wm.emul_tool(emul, str(tmp_path / "nothere"), str(tmp_path / "in.bam"))


def _run(args):
    return subprocess.run([wm.TOOL] + args, capture_output=True, timeout=120)


@pytest.mark.skipif(not os.path.exists(wm.TOOL), reason="bm2_wgsmetrics not built")
def test_option_errors(tmp_path):
    REF.write(str(tmp_path / "ref.fa"))
    (tmp_path / "u.bam").write_bytes(wm.bam_bytes(REF, [], text="@HD\tVN:1.6\tSO:unsorted\n"))
    pre, bam = str(tmp_path / "ref.fa"), str(tmp_path / "u.bam")
    for args, msg in (([], "no index prefix"), ([pre], "no input BAM"), ([pre, bam, "x"], "more than one input"),
                      (["--min-mapq", "256", pre, bam], "--min-mapq takes a whole number from 0 to 255"),
                      (["--min-mapq", "-1", pre, bam], "--min-mapq takes"), (["--min-baseq", "94", pre, bam], "--min-baseq takes a whole number from 0 to 93"),
                      (["--coverage-cap", "0", pre, bam], "--coverage-cap takes a whole number from 1 to 10000"),
                      (["--coverage-cap", "10001", pre, bam], "--coverage-cap takes"), (["--coverage-cap", "1x", pre, bam], "--coverage-cap takes"),
                      (["-t", "0", pre, bam], "-t takes"), (["--window", "12Q", pre, bam], "--window takes a size"),
                      (["--bogus", pre, bam], "unknown option --bogus"), (["--min-mapq"], "--min-mapq takes a value"),
                      ([str(tmp_path / "none"), bam], "cannot open"), ([pre, str(tmp_path / "none.bam")], "cannot open"),
                      (["-o", str(tmp_path / "o.txt"), pre, bam], "not coordinate-sorted (@HD SO:unsorted)")):
        r = _run(args)
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr)
    assert sorted(os.listdir(tmp_path)) == ["ref.fa.amb", "ref.fa.ann", "u.bam"]

"""GC bias of bm2_multiplemetrics without a GPU: Picard's calculateGc restated literally and the numpy cumulative sums give the same reference
windows on random references with N, n and IUPAC holes, and so do the host emulation's scan and mm_gc_word's bitsets; the host emulation
(tests/host_emul/gcbias_emul.cpp: mm.cu's scan, check and count with GC on, mm_gcbias.h's text) writes byte for byte the detail and summary
files that Python (tests/gcbias_util.py) gives, on crafted records for each edge of the rule and on 2 000 random pairs in windows of every
size; the tool's --program errors exit 1 before anything is read."""
import os, subprocess
import numpy as np
import pytest
import gcbias_util as gu
import multiplemetrics_util as mu

M, I, D, N, S, H, EQ, X = 0, 1, 2, 3, 4, 5, 7, 8
# g1: a 4-N hole (450..453) and a 5-N hole (750..754), an n hole, an S run, an R pair; g2..g4: contigs of length W, W + 1 and W + 2
REF = mu.Ref([("g1", 3000), ("g2", 100), ("g3", 101), ("g4", 102), ("g5", 1500)],
             holes=[(450, 4, "N"), (750, 5, "N"), (1200, 3, "n"), (1600, 10, "S"), (2000, 2, "R"), (3400, 30, "N")], seed=11)
P1, P2 = 0x1 | 0x40, 0x1 | 0x80


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return gu.build_emul(tmp_path_factory)


def crafted():
    """Records for each edge of the GC rule, on several contigs, not sorted."""
    r = mu.rec
    L1, L5 = 3000, 1500
    out = [
        # forward and reverse at the contig's start: p = 1 (binned), p <= 0 and p = 0 (not)
        r("f_start", 0, 0, 0, [(50, M)]), r("r_neg", 0x10, 0, 0, [(50, M)]), r("r_zero", 0x10, 0, 50, [(50, M)]), r("r_one", 0x10, 0, 51, [(50, M)]),
        # at the contig's end: p = L - W - 1 (the last counted window), p = L - W, p > L - W
        r("f_last", 0, 0, L1 - 102, [(30, M)]), r("f_lw", 0, 0, L1 - 101, [(30, M)]), r("f_past", 0, 0, L1 - 30, [(30, M)]),
        r("r_end", 0x10, 0, L1 - 40, [(40, M)]), r("r_last", 0x10, 0, L1 - 41, [(40, M)]), r("r_g5", 0x10, 4, L5 - 60, [(60, M)]),
        # windows with exactly 4 and 5 Ns
        r("n4", 0, 0, 420, [(40, M)]), r("n5", 0, 0, 700, [(40, M)]), r("n5r", 0x10, 0, 760, [(40, M)]),
        # contigs of length W, W + 1 and W + 2
        r("w100", 0, 1, 0, [(50, M)]), r("w101", 0, 2, 0, [(50, M)]), r("w102", 0, 3, 0, [(50, M)]), r("w102r", 0x10, 3, 52, [(50, M)]),
        # I / D / S / H, read N and = bases, QUAL '*'
        r("indel", 0, 0, 1000, [(3, H), (5, S), (20, M), (2, I), (20, M), (3, D), (10, M), (30, N), (5, M), (4, S)]),
        r("indel_r", 0x10, 4, 200, [(10, M), (4, D), (10, M), (3, I), (10, M)]),
        r("readN", 0, 0, 1100, [(20, M)], seq="ACGTNNNNNACGTACGTACG"), r("eq", 0, 0, 1150, [(20, EQ)], seq="=" * 20),
        r("ex", 0, 4, 300, [(20, X)], seq=mu.ref_seq(REF, 4, 300, 20)), r("noqual", 0, 0, 1190, [(30, M)], None),
        r("hole_n", 0, 0, 1180, [(40, M)]), r("hole_s", 0x10, 0, 1650, [(40, M)]), r("hole_r", 0, 0, 1990, [(40, M)]),
        # unmapped records placed at their mate's position
        r("um", P1 | 0x8, 0, 1300, [(40, M)], mpos=1300), r("um", P2 | 0x4, 0, 1300, [], seq="A" * 40, mpos=1300),
        r("umr", P1 | 0x4 | 0x20, 4, 500, [], seq="C" * 30, mpos=500), r("umr", P2 | 0x10 | 0x8, 4, 500, [(30, M)], mpos=500),
        # flags: secondary and supplementary not counted; QC fail and duplicates counted and placed
        r("sec", 0x100, 0, 1400, [(40, M)]), r("supp", 0x800 | P1, 0, 1400, [(40, M)]), r("qc", 0x200, 0, 1400, [(40, M)]),
        r("qc_r", 0x200 | 0x10, 4, 800, [(40, M), (2, D), (5, M)]), r("dup", 0x400, 0, 1400, [(40, M)]), r("dup_p", 0x400 | P2, 4, 900, [(40, M)]),
        r("qc_um", 0x200 | 0x4, -1, -1, [], seq="G" * 30),
        # pairs: first, second; unpaired
        r("p", P1 | 0x2 | 0x20, 0, 2500, [(50, M)], mpos=2600, tlen=150), r("p", P2 | 0x2 | 0x10, 0, 2600, [(50, M)], mpos=2500, tlen=-150),
        r("q", P1 | 0x10, 4, 1000, [(50, M)], mrid=0, mpos=10), r("q", P2, 0, 10, [(50, M)], mrid=4, mpos=1000),
        r("u", 0, 4, 1100, [(50, M)]), r("u_unmapped", 0x4, -1, -1, [], seq="ACGT" * 10),
    ]
    rng = np.random.default_rng(5)
    return [out[i] for i in rng.permutation(len(out))]


SIZES = ([10 ** 9], [1], [7], [333])


def _cmp(emul, recs, sizes_list=SIZES):
    want = gu.files(recs, REF, "a b")
    for sizes in sizes_list:
        got = gu.emul_run(emul, REF, mu.windows(recs, sizes), "a b")
        assert got[4] is None, got[4]
        assert (got[0], got[1]) == want, sizes
    return want


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_restatements_agree(emul, seed):
    rng = np.random.default_rng(seed)
    ref = gu.random_ref(rng, 12, 60, 4000, hole_every=150, extra_lens=(100, 101, 102, 103))
    lit = gu.ref_windows_literal(ref)
    assert list(gu.ref_windows_numpy(ref)) == lit and sum(lit) > 0
    assert {c for _, _, c in ref.holes} >= {"N", "n", "S"}
    h = gu.emul_new(emul, ref)
    try:
        bins, totals = np.zeros((4, gu.BINS), np.int64), np.zeros(2, np.int64)
        emul.gce_counts(h, bins.ctypes.data, totals.ctypes.data)
        assert list(bins[0]) == lit
        g, n = gu.classes(ref)
        a, b = np.zeros(1, np.uint32), np.zeros(1, np.uint32)
        for w in range((ref.l_pac + 31) // 32 + 1):                      # mm_gc_word: the scan's bitsets, past the end included
            emul.gce_word(h, w, a.ctypes.data, b.ctypes.data)
            want = [sum(int(v[32 * w + k]) << k for k in range(32) if 32 * w + k < ref.l_pac) for v in (g, n)]
            assert [int(a[0]), int(b[0])] == want, w
    finally:
        emul.gce_free(h)


def test_window_edges():
    """The Python rule at each edge, against the letters directly."""
    assert gu.window_bin(REF, 450 - 50) == (REF.text[400:500].count("G") + REF.text[400:500].count("C"))   # 4 Ns: binned
    assert gu.window_bin(REF, 700) == -1                                                                    # 5 Ns: not
    x, err = gu.reads(crafted(), REF)
    assert err is None
    one = lambda rec: gu.reads([rec], REF)[0]
    assert sum(one(mu.rec("a", 0, 0, 0, [(50, M)]))["reads"]) == 1
    for name, flag, rid, pos in (("r_neg", 0x10, 0, 0), ("r_zero", 0x10, 0, 50), ("f_lw", 0, 0, 2899), ("f_past", 0, 0, 2970), ("n5", 0, 0, 700),
                                 ("w101", 0, 2, 0), ("w100", 0, 1, 0)):
        y = one(mu.rec(name, flag, rid, pos, [(30 if name in ("f_lw", "f_past") else 50, M)]))
        assert sum(y["reads"]) == 0 and y["aligned"] == 1, name
    assert sum(one(mu.rec("w102", 0, 3, 0, [(50, M)]))["reads"]) == 1
    assert sum(one(mu.rec("f_last", 0, 0, 2898, [(30, M)]))["reads"]) == 1
    y = one(mu.rec("id", 0, 0, 1000, [(10, M), (2, I), (10, M), (3, D), (8, M)], seq=mu.ref_seq(REF, 0, 1000, 10) + "AA" + mu.ref_seq(REF, 0, 1010, 10) +
                   mu.ref_seq(REF, 0, 1023, 8)))
    assert sum(y["errors"]) == 5 and sum(y["bases"]) == 30
    # duplicates and QC fails count; secondary and supplementary do not; unmapped records are clusters, not aligned
    assert (x["clusters"], x["aligned"]) == (sum(1 for r in crafted() if not mu.bu.fields(r)["flag"] & 0x900 and
                                                 (not mu.bu.fields(r)["flag"] & 1 or mu.bu.fields(r)["flag"] & 0x40)),
                                             sum(1 for r in crafted() if not mu.bu.fields(r)["flag"] & 0x904))


def test_crafted_equals_python(emul):
    detail, summary = _cmp(emul, crafted())
    d = gu.rows(detail)
    assert [int(r["GC"]) for r in d] == list(range(101)) and all(r["ACCUMULATION_LEVEL"] == "All Reads" and r["READS_USED"] == "ALL" for r in d)
    assert sum(int(r["READ_STARTS"]) for r in d) > 10 and any(int(r["MEAN_BASE_QUALITY"]) > 0 for r in d)
    s = gu.rows(summary)
    assert len(s) == 1 and s[0]["WINDOW_SIZE"] == "100" and s[0]["SAMPLE"] == ""


def test_empty_and_windows_only(emul):
    detail, summary = _cmp(emul, [], ([1],))
    assert all(r["READ_STARTS"] == "0" and r["NORMALIZED_COVERAGE"] == "0" for r in gu.rows(detail))
    assert gu.rows(summary)[0]["TOTAL_CLUSTERS"] == "0" and gu.rows(summary)[0]["GC_NC_0_19"] == "0"


def test_random_pairs_every_window(emul):
    rng = np.random.default_rng(201)
    # mates drawn onto the short contigs do not fit there; those records are left out
    recs = [r for r in mu.random_records(REF, rng, 3000) if gu.reads([r], REF)[1] is None]
    assert len(recs) >= 2000
    want = gu.files(recs, REF, "x")
    assert sum(int(r["READ_STARTS"]) for r in gu.rows(want[0])) > 500
    for sizes in SIZES:
        got = gu.emul_run(emul, REF, mu.windows(recs, sizes), "x")
        assert got[4] is None and (got[0], got[1]) == want, sizes


def test_read_errors(emul):
    """With GC bias on, a placed QC-fail record gets the checks of an aligned one."""
    ok = mu.rec("ok", 0, 0, 100, [(10, M)])
    for bad, msg in ((mu.rec("qc_past", 0x200, 0, 2995, [(10, M)]), "read qc_past (record 1) does not lie inside a contig"),
                     (mu.rec("qc_cig", 0x200, 0, 200, [(10, M), (2, I)], seq="A" * 10), "read qc_cig (record 1) has a CIGAR that does not match"),
                     (mu.rec("past", 0, 0, 2995, [(10, M)]), "read past (record 1) does not lie inside a contig")):
        recs = [ok, bad, ok]
        assert gu.reads(recs, REF)[1][0] == 1
        got = gu.emul_run(emul, REF, [recs])
        assert got[4] is not None and msg in got[4], (msg, got[4])
    assert mu.metrics([mu.rec("qc_past", 0x200, 0, 2995, [(10, M)])], REF)[2] is None   # not an error without GC bias


@pytest.mark.skipif(not os.path.exists(mu.TOOL), reason="bm2_multiplemetrics not built")
def test_program_errors(tmp_path):
    o = str(tmp_path / "o")
    missing = str(tmp_path / "none")                                     # neither index nor BAM exists: the option fails first
    for args, msg in ((["--program", "Bogus"], "--program Bogus is not a program of this tool"),
                      (["--program", "QualityScoreDistribution"], "--program QualityScoreDistribution is not a program"),
                      (["--program", "CollectGcBiasMetrics", "--program", "MeanQualityByCycle"], "--program MeanQualityByCycle is not"),
                      (["--program", "collectgcbiasmetrics"], "--program collectgcbiasmetrics is not"),
                      (["--program"], "--program takes a value")):
        r = subprocess.run([mu.TOOL] + args + ["-o", o, missing, missing + ".bam"] if args != ["--program"] else [mu.TOOL] + args,
                           capture_output=True, timeout=120)
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr)
        assert "CollectGcBiasMetrics" in r.stderr.decode() or args == ["--program"]
    assert os.listdir(tmp_path) == []

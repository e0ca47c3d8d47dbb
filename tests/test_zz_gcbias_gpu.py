"""GC bias of bm2_multiplemetrics on the GPU: bm2_mm_gc_set / bm2_mm_add / bm2_mm_gc_finish give the detail and summary files of the host
emulation (tests/host_emul/gcbias_emul.cpp) on crafted, random and no records at several window sizes, and a window holding a bad record
counts nothing; the reference scan equals numpy on a 20 Mbp reference of many short contigs and holes, and gives the closed-form histogram
of a periodic reference longer than 2^31 bases; `bm2_multiplemetrics --program CollectGcBiasMetrics` writes the files Python computes
(tests/gcbias_util.py) from the BAMs of `bm2_mem --bam` (paired, single-end), `bm2_mem --markdup` and `bm2_applybqsr`, against an index
built by bm2_index from a FASTA with N, n and IUPAC runs; the default files equal those of the explicit programs and of all three; the GC
files do not depend on -t, --window, standard input or record order; the error cases exit 1 and leave no file."""
import json, os, subprocess
import numpy as np
import pytest
import bam_util as bu
import bqsr_util as bq
import gcbias_util as gu
import markdup_util as mdu
import multiplemetrics_util as mu
import test_gcbias_cpu as tc
import test_zz_markdup_gpu as tmg
import test_zz_wgsmetrics_gpu as twg

pytestmark = pytest.mark.gpu

TOOL = mu.TOOL
ROOT = mu.ROOT
MEM = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
INDEX = os.path.join(ROOT, "bwa-mem2_b200", "bm2_index")
APPLY = os.path.join(ROOT, "bwa-mem2_b200", "bm2_applybqsr")
GC = ["--program", "CollectGcBiasMetrics"]
ALL = ["--program", "CollectAlignmentSummaryMetrics", "--program", "CollectInsertSizeMetrics"] + GC
SUFFIXES = (".alignment_summary_metrics", ".insert_size_metrics", ".gc_bias.detail_metrics", ".gc_bias.summary_metrics")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return gu.build_emul(tmp_path_factory)


def _set(ctx, ref):
    hb, hc = mu.hole_arrays(ref)
    ctx.mm_set(ref.off, ref.lens, ref.l_pac, mu.pac_bytes(ref), hb[:2 * len(ref.holes)], hc)


def _bins(d):
    return np.array([d["windows"], d["reads"], d["bases"], d["errors"]], np.int64), np.array([d["total_clusters"], d["aligned_reads"]], np.int64)


def _device(ctx, ref, wins, gc=True):
    _set(ctx, ref)
    if gc:
        ctx.mm_gc_set()
    for w in wins:
        ctx.mm_add(*bq.flatten(w))
    return ctx.mm_finish(), ctx.mm_gc_finish() if gc else None


def test_kernels_equal_emulation(gpu_ctx, emul):
    rng = np.random.default_rng(211)
    ref = tc.REF
    rand = [r for r in mu.random_records(ref, rng, 3000) if gu.reads([r], ref)[1] is None]
    for recs in (tc.crafted(), rand, []):
        for sizes in ([max(len(recs), 1)], [1], [7], [333]):
            wins = mu.windows(recs, sizes)
            want = gu.emul_run(emul, ref, wins, "a")
            mm, d = _device(gpu_ctx, ref, wins)
            bins, totals = _bins(d)
            assert want[4] is None and np.array_equal(bins, want[2]) and np.array_equal(totals, want[3]), sizes
            assert gu.emul_texts(emul, bins, totals, "a") == want[:2]
            assert d["scan_ms"] > 0 and d["add_ms"] >= 0
            # GC bias on leaves the alignment summary and insert size counts as they are
            plain = _device(gpu_ctx, ref, wins, gc=False)[0]
            assert all(np.array_equal(mm[k], plain[k]) for k in ("counts", "len_hist", "mism_hist", "nocall", "insert_hist", "insert_big"))
        assert want[:2] == gu.files(recs, ref, "a")
    # mm_set turns GC bias off again
    _set(gpu_ctx, ref)
    with pytest.raises(Exception, match="bm2_mm_gc_set"):
        gpu_ctx.mm_gc_finish()


def test_bad_window_counts_nothing(gpu_ctx, emul):
    ref = tc.REF
    ok = [mu.rec("ok", 0, 0, 100, [(50, 0)]), mu.rec("ok2", 0x10, 4, 400, [(50, 0), (2, 2), (10, 0)])]
    for bad, msg in ((mu.rec("qc_past", 0x200, 0, 2995, [(10, 0)]), "read qc_past (record 4) does not lie inside a contig"),
                     (mu.rec("qc_cig", 0x200, 0, 200, [(10, 0), (2, 1)], seq="A" * 10), "read qc_cig (record 4) has a CIGAR")):
        wins = [ok, ok[:1] + [ok[1], bad]]
        assert msg in gu.emul_run(emul, ref, wins)[4]
        _set(gpu_ctx, ref)
        gpu_ctx.mm_gc_set()
        gpu_ctx.mm_add(*bq.flatten(wins[0]))
        with pytest.raises(Exception, match=msg.replace("(", r"\(").replace(")", r"\)")):
            gpu_ctx.mm_add(*bq.flatten(wins[1]))
        got = _bins(gpu_ctx.mm_gc_finish())
        want = _bins(_device(gpu_ctx, ref, [wins[0]])[1])
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[1][1] == 2


def test_scan_equals_numpy(gpu_ctx):
    """20+ Mbp: thousands of contigs from 50 bases up, many holes, so that tiles straddle contig ends."""
    rng = np.random.default_rng(212)
    ref = gu.random_ref(rng, 6000, 50, 7000, hole_every=400, extra_lens=(100, 101, 102, 103) * 20 + (3_000_000,))
    assert ref.l_pac > 20_000_000 and len(ref.holes) > 30_000
    _set(gpu_ctx, ref)
    gpu_ctx.mm_gc_set()
    got = gpu_ctx.mm_gc_finish()["windows"]
    want = gu.ref_windows_numpy(ref)
    assert np.array_equal(got, want) and want.sum() > 15_000_000


def test_scan_past_2g(gpu_ctx):
    """A periodic reference of 2.2 G bases (GCCATAT repeated, so a window's GC is 42 plus its first two letters') in two contigs, with holes
    of N, n and S below and above 2^31: the closed-form histogram."""
    pat = "GCCATAT"
    lens = [1_100_000_007, 1_100_000_013]
    off = [0, lens[0]]
    l_pac = sum(lens)
    assert l_pac > 2 ** 31
    code = {"A": 0, "C": 1, "G": 2, "T": 3}
    cyc = [code[pat[i % 7]] for i in range(28)]                      # 28 loci = 7 bytes
    unit = bytes(sum(cyc[4 * j + k] << (2 * (3 - k)) for k in range(4)) for j in range(7))
    n_bytes = (l_pac + 3) // 4
    pac = np.tile(np.frombuffer(unit, np.uint8), n_bytes // 7 + 1)[:n_bytes]
    holes = [(5_000_000, 5, "n"), (2_150_000_000, 3, "N"), (2_160_000_000, 10, "N"), (2_170_000_001, 6, "S")]

    def letter(g):
        for b, n, c in holes:
            if b <= g < b + n:
                return c.upper()
        return pat[g % 7]

    def wbin(g, with_holes):
        s = "".join(letter(g + k) if with_holes else pat[(g + k) % 7] for k in range(100))
        return -1 if s.count("N") > 4 else s.count("G") + s.count("C")

    def ceil7(a):
        return -((-a) // 7)

    want = np.zeros(101, np.int64)
    for o, L in zip(off, lens):
        lo, hi = o + 1, o + L - 100
        for r in range(7):
            want[wbin(r, False)] += ceil7(hi - r) - ceil7(lo - r)
    for b, n, _ in holes:                                            # the windows a hole touches
        o, L = next((o, L) for o, L in zip(off, lens) if o <= b < o + L)
        for g in range(max(b - 99, o + 1), min(b + n, o + L - 100)):
            want[wbin(g, False)] -= 1
            nb = wbin(g, True)
            if nb >= 0:
                want[nb] += 1
    h = np.array([(b, b + n) for b, n, _ in holes], np.int64).reshape(-1)
    gpu_ctx.mm_set(off, lens, l_pac, pac, h, "".join(c for _, _, c in holes).encode())
    gpu_ctx.mm_gc_set()
    d = gpu_ctx.mm_gc_finish()
    assert np.array_equal(d["windows"], want), (d["windows"] - want).nonzero()
    assert want.sum() > 2_199_000_000


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    for t in (TOOL, MEM, INDEX, APPLY):
        if not os.path.exists(t):
            pytest.skip(os.path.basename(t) + " not built")
    d = tmp_path_factory.mktemp("gc_gpu")
    rng = np.random.default_rng(213)
    (d / "ref.fa").write_text(twg._genome(rng))
    subprocess.run([INDEX, str(d / "ref.fa")], check=True, capture_output=True, timeout=900)
    prefix = str(d / "ref.fa")
    ref = mu.Ref.read(prefix)
    assert {c for _, _, c in ref.holes} >= {"N", "n", "R"}
    pairs = mdu.planted_pairs(mdu.load_reference(prefix), rng, n_base=400)
    files, _ = tmg._write_pairs(d, pairs, "p")
    bams = {}
    for name, kind, mode in (("bam_pe", "--bam", "pe"), ("bam_se", "--bam", "se"), ("markdup_pe", "--markdup", "pe")):
        out = str(d / (name + ".bam"))
        r = subprocess.run([MEM, kind, "-R", r"@RG\tID:g1\tSM:s", prefix] + files[mode] + ["-o", out], capture_output=True, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        bams[name] = out
    bref = bq.Ref(prefix)
    (d / "s.vcf").write_text(bq.vcf_text(bref, bq.random_sites(bref, np.random.default_rng(214), every=50)))
    r = subprocess.run([MEM, "--recal-file", str(d / "t.txt"), "--known-sites", str(d / "s.vcf"), "-R", r"@RG\tID:g1\tSM:s", prefix] + files["pe"] +
                       ["-o", str(d / "rc.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([APPLY, "--bqsr-recal-file", str(d / "t.txt"), "-o", str(d / "ap.bam"), str(d / "rc.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    bams["applybqsr"] = str(d / "ap.bam")
    return d, prefix, ref, gu.ref_windows_numpy(ref), bams


def _tool(args, stdin=None):
    r = subprocess.run([TOOL] + args, capture_output=True, timeout=900, stdin=stdin)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1])


def _records(bam):
    raw = bu.inflate(open(bam, "rb").read())
    text, _, used = bu.parse_header(raw)
    return text, [r for _, r in bu.records(raw[used:])]


def _read(out, suffixes):
    return tuple(open(out + s).read() for s in suffixes)


def _body(t):
    return t.split("\n", 2)[2]                                       # all but the line with the arguments


@pytest.mark.parametrize("bam", ["bam_pe", "bam_se", "markdup_pe", "applybqsr"])
def test_tool_equals_python(inputs, bam):
    d, prefix, ref, windows, bams = inputs
    out = str(d / ("g_" + bam))
    args = GC + ["-o", out, prefix, bams[bam]]
    st = _tool(args)
    _, recs = _records(bams[bam])
    want = gu.files(recs, ref, " ".join(args), windows)
    assert _read(out, SUFFIXES[2:]) == want
    assert not any(os.path.exists(out + s) for s in SUFFIXES[:2])
    assert st["gc_windows"] == int(windows.sum()) and st["gc_read_starts"] == sum(int(r["READ_STARTS"]) for r in gu.rows(want[0]))
    assert st["gc_read_starts"] > 100 and st["gc_scan_s"] > 0 and st["gc_add_s"] > 0 and st["records"] == len(recs)
    s = gu.rows(want[1])[0]
    assert int(s["ALIGNED_READS"]) > 0 and int(s["TOTAL_CLUSTERS"]) > 0
    assert not [f for f in os.listdir(d) if f.endswith(".tmp")]


def test_default_files_unchanged_by_programs(inputs):
    d, prefix, ref, windows, bams = inputs
    runs = {}
    for name, progs in (("default", []), ("two", ALL[:4]), ("all", ALL), ("rev", ALL[4:] + ALL[2:4] + ALL[:2])):
        out = str(d / ("p_" + name))
        runs[name] = (_tool(progs + ["-o", out, prefix, bams["bam_pe"]]), out)
    base = tuple(_body(t) for t in _read(runs["default"][1], SUFFIXES[:2]))
    for name in ("two", "all", "rev"):
        assert tuple(_body(t) for t in _read(runs[name][1], SUFFIXES[:2])) == base, name
    assert not any(os.path.exists(runs[n][1] + s) for n in ("default", "two") for s in SUFFIXES[2:])
    assert tuple(map(_body, _read(runs["all"][1], SUFFIXES[2:]))) == tuple(map(_body, _read(runs["rev"][1], SUFFIXES[2:])))
    keys = set(runs["default"][0])
    assert set(runs["two"][0]) == keys and not any(k.startswith("gc_") for k in keys)
    assert set(runs["all"][0]) == keys | {"gc_windows", "gc_read_starts", "gc_scan_s", "gc_add_s"}
    assert runs["all"][0]["device_bytes"] > runs["default"][0]["device_bytes"]


def test_gc_bytes_do_not_depend_on_threads_windows_stdin_or_order(inputs):
    d, prefix, ref, windows, bams = inputs
    text, recs = _records(bams["markdup_pe"])
    shuffled = str(d / "shuffled.bam")
    order = np.random.default_rng(215).permutation(len(recs))
    open(shuffled, "wb").write(mu.bam_bytes(ref, [recs[i] for i in order], text=text))
    bodies, stats = [], []
    for k, (extra, bam) in enumerate(((["-t", "1"], bams["markdup_pe"]), (["-t", "16"], bams["markdup_pe"]),
                                      (["-t", "16", "--window", "64K"], bams["markdup_pe"]), (["-t", "3", "--window", "100K"], shuffled))):
        out = str(d / ("o%d" % k))
        stats.append(_tool(GC + extra + ["-o", out, prefix, bam]))
        bodies.append(tuple(map(_body, _read(out, SUFFIXES[2:]))))
    with open(bams["markdup_pe"], "rb") as f:
        stats.append(_tool(GC + ["-o", str(d / "o_stdin"), prefix, "-"], stdin=f))
    bodies.append(tuple(map(_body, _read(str(d / "o_stdin"), SUFFIXES[2:]))))
    assert all(b == bodies[0] for b in bodies)
    assert stats[2]["windows"] > 3 and stats[0]["windows"] == 1
    assert len({(s["gc_windows"], s["gc_read_starts"]) for s in stats}) == 1


def test_errors_leave_no_file(inputs, tmp_path):
    d, prefix, ref, windows, bams = inputs
    text, recs = _records(bams["bam_pe"])
    i = next(k for k, x in enumerate(recs) if not bu.fields(x)["flag"] & 0x904)
    f = bu.fields(recs[i])
    past = bytearray(recs[i]); past[8:12] = (ref.lens[f["rid"]] - 5).to_bytes(4, "little")
    qc = bytearray(past); qc[18:20] = (f["flag"] | 0x200).to_bytes(2, "little")
    (tmp_path / "past.bam").write_bytes(mu.bam_bytes(ref, recs[:i] + [bytes(past)] + recs[i + 1:], text=text))
    (tmp_path / "qc.bam").write_bytes(mu.bam_bytes(ref, recs[:i] + [bytes(qc)] + recs[i + 1:], text=text))
    (tmp_path / "notbam.bam").write_bytes(b"hello")
    golden = os.path.join(ROOT, "tests", "golden", "c0_index", "ref.fa")
    msg_past = "read %s (record %d) does not lie inside a contig" % (f["qname"], i)
    for progs, args, msg in ((ALL, [prefix, str(tmp_path / "past.bam")], msg_past), (GC, [prefix, str(tmp_path / "qc.bam")], msg_past),
                             (ALL, [prefix, str(tmp_path / "qc.bam")], msg_past), (ALL, [prefix, str(tmp_path / "notbam.bam")], ""),
                             (ALL, [golden, bams["bam_pe"]], "in the header, chr1 of length"),
                             (ALL + ["--program", "CollectQualityYieldMetrics"], [prefix, bams["bam_pe"]], "CollectQualityYieldMetrics is not")):
        out = str(tmp_path / "e")
        r = subprocess.run([TOOL] + progs + ["-o", out] + args, capture_output=True, timeout=900)
        assert r.returncode == 1 and msg in r.stderr.decode(), (progs, args, r.stderr[-2000:])
        assert not [x for x in os.listdir(tmp_path) if x.startswith("e.")]
    # a QC-failed record past its contig is an error only when GC bias runs
    _tool(["-o", str(tmp_path / "ok"), prefix, str(tmp_path / "qc.bam")])

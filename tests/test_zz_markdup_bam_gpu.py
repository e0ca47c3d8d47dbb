"""bm2_markdup on the GPU: bm2_markdup_records equals the host emulation (tests/host_emul/markdup_bam_emul.cpp) record for record, counts
included; bm2_markdup_pair joins the halves the emulation and Python join, under forced hash collisions too; bm2_dup_resolve_ex's exact cell
pass keeps read groups apart as the emulation does; the tool writes the emulation's BAM, BAI and metrics bytes on crafted and random lanes and
on a group of 40 copies over two read groups, and the same records' BGZF members and
metrics whatever -t, --window and --sig-mem; and on
`bm2_mem --sort` output of reads with planted duplicates under Illumina names, one input of one library gives bm2_mem --markdup-metrics's
values, two lanes of one library give the same, two libraries give two rows with duplicates found within each, and only flag bytes differ
from the merged inputs.  Errors exit 1 and leave no file."""
import json, os, re, subprocess
import numpy as np
import pytest
import bam_util as bu
import markdup_bam_util as mb
import markdup_metrics_util as mm
import markdup_util as mu
import test_markdup_bam_cpu as tc
import test_zz_bam_gpu as tg
import test_zz_markdup_gpu as tmg
import test_zz_markdup_metrics_gpu as tmm

pytestmark = pytest.mark.gpu

MEM = tg.TOOL


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mb.build_emul(tmp_path_factory)


def _lanes(tmp_path):
    rng = np.random.default_rng(81)
    lanes = [("l1", "a"), ("l2", "a"), ("l3", "b")]
    by = mb.random_lanes(rng, 3000, lanes)
    rgs = ["@RG\tID:%s\tSM:s\tLB:%s" % l for l in lanes]
    ins = [(mb.header(rgs[:2] if k < 2 else rgs)[0], mb.header()[1], mb.sort_recs(by[rg])) for k, (rg, _) in enumerate(lanes)]
    return tc._write(tmp_path, ins, "r"), rgs, lanes, by


def test_record_kernel_equals_emulation(gpu_ctx, emul, tmp_path):
    paths, rgs, lanes, by = _lanes(tmp_path)
    recs = [r for k in sorted(by) for r in by[k]] + [r for _, _, rs in tc.crafted() for r in rs]
    recs.append(mb.rec(0, 10, 0x41, "other", rg="zz"))                                  # an RG:Z value that is no @RG ID
    ids, libs = ["l1", "l2", "l3"], [1, 1, 2]
    for part in (recs[:1], recs[:777], recs):
        gpu_ctx.markdup_set(ids, libs, 3, 0)
        data = b"".join(part)
        starts = np.cumsum([0] + [len(r) for r in part[:-1]])
        got = gpu_ctx.markdup_records(data, starts)
        want, cnt = mb.emul_records(emul, part, ids, libs, 3, 0)
        assert got.tobytes() == want.tobytes()
        assert np.array_equal(gpu_ctx.markdup_counts(3).reshape(-1), cnt)
        for k, r in enumerate(part[:300]):                                              # and Python's restatement
            assert tuple(got[k].tolist()) == mb.record_info(r, ids, libs, 0)[0]
    assert min(gpu_ctx.markdup_stats()) >= 0


def test_pairing_equals_emulation(gpu_ctx, emul, tmp_path):
    rng = np.random.default_rng(97)
    _, _, _, by = _lanes(tmp_path)
    recs = mb.sort_recs([r for k in sorted(by) for r in by[k]])
    gpu_ctx.markdup_set(["l1", "l2", "l3"], [1, 1, 2], 3, 0)
    got = gpu_ctx.markdup_records(b"".join(recs), np.cumsum([0] + [len(r) for r in recs[:-1]]))
    real = [(int(g["hash"]), int(g["rg"]), mb.bu.fields(r)["qname"].encode()) for g, r in zip(got, recs) if g["kind"] in (mb.HALF, mb.UNMAPPED_HALF)]
    for halves in ([], [(7, 0, b"a"), (7, 0, b"b"), (7, 0, b"a")], tc.collision_halves(rng), tc.collision_halves(rng, 20000), real):
        a, names = mb.halves_array(halves)
        part = gpu_ctx.markdup_pair(a, names)
        assert part == mb.emul_pair(emul, halves) == mb.pair_halves(halves, None)
    assert sum(p >= 0 for p in part) > len(real) // 2
    assert gpu_ctx.markdup_stats()[1] >= 0


def test_exact_optical_pass_keeps_read_groups_apart(gpu_ctx, emul):
    rng = np.random.default_rng(99)
    for d in (0, 100, 2500):
        for n in (3000, 40000):
            e = tc.rg_groups(rng, n, d)
            got, opt, _ = gpu_ctx.dup_resolve_ex(e, d)
            want, wopt = mb.emul_resolve_ex(emul, e, d)
            assert np.array_equal(got, want) and opt == wopt, (n, d)
    dense = mm.located_entries(rng, 6000, 5, 100)                                       # one spot, three read groups
    dense["k1"][:5000], dense["k2"][:5000] = dense["k1"][0], dense["k2"][0]
    dense["tile"][:5000], dense["x"][:5000], dense["y"][:5000] = 2202, 1000 + np.arange(5000) % 7, 2000 + np.arange(5000) % 11
    dense["loc"][:5000] = mm.HAS | (np.arange(5000) % 3) << 2
    got, opt, _ = gpu_ctx.dup_resolve_ex(dense, 100)
    want, wopt = mb.emul_resolve_ex(emul, dense, 100)
    assert np.array_equal(got, want) and opt == wopt and opt >= 5000 - 3


def _tool(argv, w):
    r = subprocess.run([mb.TOOL] + argv, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1])


def _same_as_emulation(emul, w, paths, extra, tag, **kw):
    out, met = str(w / (tag + ".bam")), str(w / (tag + ".txt"))
    argv = extra + ["--write-index", "-M", met, "-o", out] + paths
    st = _tool(argv, w)
    eo, em = str(w / (tag + "_e.bam")), str(w / (tag + "_e.txt"))
    rc, msg, est = mb.emul_run(emul, paths, eo, em, eo + ".bai", args=" ".join(argv), cl=mb.TOOL + " " + " ".join(argv), **kw)
    assert rc == 0, msg
    (gt, _, gr), (et, _, er) = mb.read_bam(out), mb.read_bam(eo)
    assert gt == et and gr == er
    assert open(out, "rb").read() == open(eo, "rb").read() and open(out + ".bai", "rb").read() == open(eo + ".bai", "rb").read()
    assert open(met).read() == open(em).read()
    for k in ("records", "pairs", "fragments", "dup_pair_templates", "dup_fragment_templates", "dup_records", "dup_optical_pairs", "libraries"):
        assert st[k] == est[k], k
    return st, tg._records_part(open(out, "rb").read()), mb.read_bam(out)[2], open(met).read().split("\n", 2)[2]


def test_tool_equals_emulation(emul, tmp_path):
    if not os.path.exists(mb.TOOL):
        pytest.skip("bm2_markdup not built")
    paths, *_ = _lanes(tmp_path)
    cpaths = tc._write(tmp_path, tc.crafted(), "c")
    gpaths = tc._write(tmp_path, tc.big_group(), "g")                                  # a group for the exact cell pass, two read groups
    for ps, tag in ((paths, "r"), (cpaths, "c"), (gpaths, "g")):
        base = None
        for k, (extra, kw) in enumerate([([], {}), (["-t", "4"], dict(threads=4)), (["--window", "64K"], dict(window=64 << 10)),
                                         (["--sig-mem", "64K", "--window", "100K"], dict(sig_bytes=64 << 10, window=100 << 10))]):
            st, part, recs, met = _same_as_emulation(emul, tmp_path, ps, extra, "out_%s%d" % (tag, k), **kw)
            if base is None:
                base = (part, recs, met, st)
            # the records' members, the records and the metrics rows do not depend on the options (the header's @PG CL does, and with it
            # the BAI's virtual offsets, which each run checks against the emulation)
            assert part == base[0] and recs == base[1] and met == base[2]
            if "--sig-mem" in extra and tag == "r":
                assert st["dup_sig_runs"] >= 2
        assert base[3]["dup_pair_templates"] > 0 and st["windows"] >= 1
        if tag == "g":
            assert st["dup_optical_pairs"] == 38


def _sorted_lane(prefix, d, pairs, name, rg):
    files, _ = tmg._write_pairs(d, pairs, name)
    out = str(d / (name + ".bam"))
    r = subprocess.run([MEM, "--sort", "-R", rg, "-K", "20000", prefix] + files["pe"] + ["-o", out], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return out, files


@pytest.fixture(scope="module")
def lanes(golden_dir, tmp_path_factory):
    if not os.path.exists(MEM) or not os.path.exists(mb.TOOL):
        pytest.skip("bm2_mem or bm2_markdup not built")
    d = tmp_path_factory.mktemp("markdup_bam_gpu")
    prefix = os.path.join(golden_dir, "c0_index", "ref.fa")
    ref = mu.load_reference(prefix)
    rng = np.random.default_rng(83)
    plain = sorted(mu.planted_pairs(ref, rng, n_base=120), key=lambda p: (len(p[0]), p[0]))
    named = tmm._name_pairs(plain, rng)                                                # in plain's order
    lane = [int(re.match(r"b(\d+)", p[0]).group(1)) % 2 for p in plain]                 # each copy in its original's lane
    return d, prefix, named, lane


def _metrics_rows(text):
    lines = text.split("\n")
    k = lines.index("\t".join(mm.COLUMNS))
    rows = []
    for l in lines[k + 1:]:
        if not l:
            break
        rows.append(dict(zip(mm.COLUMNS, l.split("\t"))))
    return rows


def test_one_input_equals_bm2_mem_metrics(lanes):
    d, prefix, named, _ = lanes
    w = d / "one"; w.mkdir()
    rg = r"@RG\tID:l1\tSM:s\tLB:a"
    srt, files = _sorted_lane(prefix, w, named, "all", rg)
    met_mem = str(w / "mem.txt")
    r = subprocess.run([MEM, "--markdup-metrics", met_mem, "-R", rg, "-K", "20000", prefix] + files["pe"] + ["-o", str(w / "mem.bam")],
                       capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    st = _tool(["-M", str(w / "md.txt"), "-o", str(w / "md.bam"), srt], w)
    a, b = open(met_mem).read(), open(w / "md.txt").read()
    assert a.split("\n", 2)[2] == b.split("\n", 2)[2] and b.startswith("## htsjdk.samtools.metrics.StringHeader\n# bm2_markdup -M ")
    assert st["dup_optical_pairs"] > 0 and st["libraries"] == 1 and "CoverageMult" in b
    # the primary flags equal Python's, and only flag bytes differ from the input
    text, want, mtext, _ = mb.markdup_files([srt], cl="x", args=" ".join(["-M", str(w / "md.txt"), "-o", str(w / "md.bam"), srt]))
    _, _, got = mb.read_bam(str(w / "md.bam"))
    _, _, inp = mb.read_bam(srt)
    assert got == want and mtext == b and len(got) == len(inp)
    assert all(g[:18] == i[:18] and g[20:] == i[20:] for g, i in zip(got, inp))
    assert sum(1 for g in got if bu.fields(g)["flag"] & 0x400) == st["dup_records"] > 0


def test_two_lanes(lanes):
    """The records of one bm2_mem run split by lane (so that both runs hold the same alignments) and relabelled l1 / l2."""
    d, prefix, named, lane = lanes
    w = d / "two"; w.mkdir()
    one, _ = _sorted_lane(prefix, w, named, "all", r"@RG\tID:l1\tSM:s\tLB:a")
    _tool(["-M", str(w / "single.txt"), "-o", str(w / "single.bam"), one], w)
    single = _metrics_rows(open(w / "single.txt").read())
    text, refs, recs = mb.read_bam(one)
    lane_of = {p[0]: l for p, l in zip(named, lane)}
    for libs in (("a", "a"), ("a", "b")):
        ins = []
        for k in range(2):
            h = text.replace("@RG\tID:l1\tSM:s\tLB:a", "@RG\tID:l%d\tSM:s\tLB:%s" % (k + 1, libs[k]))
            rs = [r.replace(b"RGZl1\0", b"RGZl%d\0" % (k + 1)) for r in recs if lane_of[bu.fields(r)["qname"]] == k]
            ins.append(str(w / ("l%d%s.bam" % (k + 1, "".join(libs)))))
            mb.write_bam(ins[-1], h, refs, rs)
        tag = "".join(libs)
        argv = ["-M", str(w / (tag + ".txt")), "-o", str(w / (tag + ".bam")), "--write-index"] + ins
        st = _tool(argv, w)
        rows = _metrics_rows(open(w / (tag + ".txt")).read())
        _, want, mtext, _ = mb.markdup_files(ins, args=" ".join(argv))
        _, _, got = mb.read_bam(str(w / (tag + ".bam")))
        assert got == want and open(w / (tag + ".txt")).read() == mtext
        merged = sorted([(mb.key(r), i, k, r) for i, p in enumerate(ins) for k, r in enumerate(mb.read_bam(p)[2])], key=lambda t: t[:3])
        assert all(g[:18] == m[3][:18] and g[20:] == m[3][20:] for g, m in zip(got, merged)) and len(got) == len(merged)
        if libs == ("a", "a"):
            assert len(rows) == 1 and {k: v for k, v in rows[0].items() if k != "LIBRARY"} == {k: v for k, v in single[0].items() if k != "LIBRARY"}
        else:
            assert [r["LIBRARY"] for r in rows] == ["a", "b"] and st["libraries"] == 2
            assert sum(int(r["READ_PAIRS_EXAMINED"]) for r in rows) == int(single[0]["READ_PAIRS_EXAMINED"])
            assert sum(int(r["READ_PAIR_DUPLICATES"]) for r in rows) <= int(single[0]["READ_PAIR_DUPLICATES"])
    assert sorted(f for f in os.listdir(w) if ".tmp" in f) == []


@pytest.mark.parametrize("case", [c[0] for c in tc._errors()])
def test_errors_exit_1_and_leave_no_file(tmp_path, case):
    if not os.path.exists(mb.TOOL):
        pytest.skip("bm2_markdup not built")
    _, ins, text = next(c for c in tc._errors() if c[0] == case)
    paths = tc._write(tmp_path, ins)
    r = subprocess.run([mb.TOOL, "-M", str(tmp_path / "m.txt"), "-o", str(tmp_path / "o.bam"), "--write-index"] + paths, capture_output=True,
                       timeout=300)
    assert r.returncode == 1 and text in r.stderr.decode(), r.stderr
    assert sorted(os.listdir(tmp_path)) == sorted(os.path.basename(p) for p in paths)

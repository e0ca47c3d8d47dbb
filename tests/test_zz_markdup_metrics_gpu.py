"""Duplication metrics and optical duplicates on the GPU: bm2_dup_signatures_ex and bm2_dup_resolve_ex equal the host emulation
(tests/host_emul/markdup_metrics_emul.cpp) byte for byte, counters and optical counts included, and give bm2_dup_signatures's entries and
bm2_dup_resolve's duplicates; `bm2_mem --markdup-metrics` on reads with planted duplicates under Illumina-style names (copies near their
original on the same tile, further away, on another tile, and in the other orientation class) writes the metrics Python computes from the
output BAM's records and names - paired, single-end, smart pairing and -R with and without LB - while its BAM members equal --markdup's; the
file is the same at -p 1, -p 3 and --sort-mem 100K, and --optical-distance changes only what it should."""
import json, os, re, subprocess
import numpy as np
import pytest
import bam_util as bu
import markdup_util as mu
import markdup_metrics_util as mm
import test_markdup_cpu as tmc
import test_markdup_metrics_cpu as tmm
import test_zz_bam_gpu as tg
import test_zz_markdup_gpu as tmg

pytestmark = pytest.mark.gpu

TOOL = tg.TOOL


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mm.build_emul(tmp_path_factory)


def test_kernels_equal_emulation(gpu_ctx, emul):
    rng = np.random.default_rng(41)
    cases = [tmc.crafted_templates(), tmm.located_templates(rng, 3000), tmm.located_templates(rng, 3000, paired=False), []]
    for t in cases:
        data, first, ids = mu.flatten(t)
        starts = np.array([a for a, _ in bu.records(data)], np.int64)
        gp, gf, counts, ms = gpu_ctx.dup_signatures_ex(data, starts, first, ids)
        ep, ef, ec = mm.emul_signatures_ex(emul, data, first, ids)
        assert gp.tobytes() == ep.tobytes() and gf.tobytes() == ef.tobytes() and counts == ec and ms >= 0
        pp, pf, _ = gpu_ctx.dup_signatures(data, starts, first, ids)                # the plain call's entries
        assert gp[list(mu.DUP_ENTRY_DT.names)].tolist() == pp.tolist() and gf.tobytes() == pf.tobytes()
    groups = []
    for n in (1, 2, 31, 33, 1000, 20_000, 200_000):
        for d in (0, 100, 2500):
            groups.append((mm.located_entries(rng, n, max(n // 40, 1), d), d))
    dense = mm.located_entries(rng, 60_000, 5, 100)                                 # a dense group of 50 000 at one spot
    dense["k1"][:50_000], dense["k2"][:50_000] = dense["k1"][0], dense["k2"][0]
    dense["tile"][:50_000], dense["loc"][:50_000] = 2202, mm.HAS | mm.REV * (np.arange(50_000) % 2)
    dense["x"][:50_000], dense["y"][:50_000] = 1000 + np.arange(50_000) % 7, 2000 + np.arange(50_000) % 11
    groups.append((dense, 100))
    for e, d in groups:
        got, opt, ms = gpu_ctx.dup_resolve_ex(e, d)
        want, wopt = mm.emul_resolve_ex(emul, e, d)
        assert np.array_equal(got, want) and opt == wopt, (len(e), d)
        plain, _ = gpu_ctx.dup_resolve(np.array(e[list(mu.DUP_ENTRY_DT.names)].tolist(), mu.DUP_ENTRY_DT))
        assert np.array_equal(got, plain)
        srt, _ = gpu_ctx.dup_resolve_ex(e, d, False)
        assert srt.tobytes() == mm.emul_resolve_ex(emul, e, d, False).tobytes()
    assert mm.emul_resolve_ex(emul, dense, 100)[1] >= 50_000 - 2


def _name_pairs(pairs, rng):
    """Illumina names: an original at a random spot; its copies within 100 pixels on its tile, 300 to 3000 pixels away, or on another tile."""
    spot, names, out = {}, set(), []
    for n, *rest in sorted(pairs, key=lambda p: (len(p[0]), p[0])):
        base = re.match(r"b\d+", n).group(0)
        if n == base:
            t, x, y = 1101 + int(rng.integers(0, 3)), int(rng.integers(3000, 30000)), int(rng.integers(3000, 30000))
            spot[base] = (t, x, y)
        else:
            t, x, y = spot[base]
            k = int(rng.integers(0, 4))
            if k < 2:
                x, y = x + int(rng.integers(-100, 101)), y + int(rng.integers(-100, 101))
            elif k == 2:
                x, y = x + int(rng.integers(300, 3000)), y - int(rng.integers(0, 3000))
            else:
                t = t + 10
        while (t, x, y) in names:
            x += 1
        names.add((t, x, y))
        out.append((mm.illumina_name(t, x, y), *rest))
    return out


@pytest.fixture(scope="module")
def planted(golden_dir, tmp_path_factory):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    d = tmp_path_factory.mktemp("markdup_metrics_gpu")
    prefix = os.path.join(golden_dir, "c0_index", "ref.fa")
    ref = mu.load_reference(prefix)
    rng = np.random.default_rng(43)
    plain = mu.planted_pairs(ref, rng, n_base=120)
    named = _name_pairs(plain, rng)
    order = rng.permutation(len(named))
    files, tids = tmg._write_pairs(d, [named[i] for i in order], "p")
    plain_files, plain_tids = tmg._write_pairs(d, plain, "q")
    return d, prefix, files, tids, plain_files, plain_tids


def _run(args, w, tag):
    out, met = str(w / (tag + ".bam")), str(w / (tag + ".txt"))
    argv = ["--markdup-metrics", met] + args + ["-o", out]
    r = subprocess.run([TOOL] + argv, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1]), open(met).read(), " ".join(argv), out


def _want(out, tid_of_name, d):
    by = {}
    for r in tmg._records(out):
        f = bu.fields(r)
        by.setdefault(f["qname"], []).append(f)
    return mm.metrics_of([(tid_of_name[q], fs) for q, fs in by.items()], d)


@pytest.mark.parametrize("mode,args", [("pe", []), ("se", []), ("smart", ["-p"]), ("pe", ["-R", r"@RG\tID:g1\tSM:s\tLB:lib7"]),
                                       ("pe", ["-R", r"@RG\tID:g1\tSM:s"])])
def test_metrics_equal_python(planted, mode, args):
    d, prefix, files, tids, _, _ = planted
    w = d / ("m_%s_%d" % (mode, len(args[-1]) if args else 0)); w.mkdir()
    common = args + ["-K", "100000000" if mode == "smart" else "20000", prefix] + files[mode]
    st, text, argv, out = _run(common, w, "md")
    r = subprocess.run([TOOL, "--markdup"] + common + ["-o", str(w / "plain.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    plain = json.loads(r.stderr.decode().strip().split("\n")[-1])
    assert sorted(os.listdir(w)) == ["md.bam", "md.txt", "plain.bam"]                 # no temporary file
    assert tg._records_part(open(out, "rb").read()) == tg._records_part(open(w / "plain.bam", "rb").read())
    assert "dup_optical_pairs" not in plain and plain["dup_pair_templates"] == st["dup_pair_templates"]
    want = _want(out, tids[mode], 100)
    lib = "lib7" if "LB:lib7" in "".join(args) else "Unknown Library"
    assert text == mm.metrics_text(want, argv, lib)
    row, hist = mm.parse_metrics(text)
    assert int(row["READ_PAIR_DUPLICATES"]) == st["dup_pair_templates"] and int(row["UNPAIRED_READ_DUPLICATES"]) == st["dup_fragment_templates"]
    assert int(row["READ_PAIR_OPTICAL_DUPLICATES"]) == st["dup_optical_pairs"]
    if mode == "se":
        assert want["pairs"] == 0 and want["unpaired"] > 0 and not hist and st["dup_optical_pairs"] == 0
    else:
        assert st["dup_optical_pairs"] > 0 and want["pair_dups"] > st["dup_optical_pairs"] and len(hist) == 100


def test_distance_and_names_without_location(planted):
    d, prefix, files, tids, plain_files, plain_tids = planted
    w = d / "dist"; w.mkdir()
    common = ["-K", "20000", prefix] + files["pe"]
    s1, t1, _, out1 = _run(common, w, "a")
    s2, t2, argv2, out2 = _run(["--optical-distance", "2500"] + common, w, "b")
    assert tg._records_part(open(out1, "rb").read()) == tg._records_part(open(out2, "rb").read())
    r1, h1 = mm.parse_metrics(t1)
    r2, h2 = mm.parse_metrics(t2)
    changed = {k for k in mm.COLUMNS if r1[k] != r2[k]}
    assert changed == {"READ_PAIR_OPTICAL_DUPLICATES", "ESTIMATED_LIBRARY_SIZE"} and h1 != h2
    assert int(r2["READ_PAIR_OPTICAL_DUPLICATES"]) > int(r1["READ_PAIR_OPTICAL_DUPLICATES"]) and s2["dup_optical_pairs"] > s1["dup_optical_pairs"]
    assert t2 == mm.metrics_text(_want(out2, tids["pe"], 2500), argv2)
    s3, t3, argv3, out3 = _run(["-K", "20000", prefix] + plain_files["pe"], w, "c")
    want = _want(out3, plain_tids["pe"], 100)
    assert s3["dup_optical_pairs"] == 0 and want["optical"] == 0 and want["pair_dups"] > 0 and t3 == mm.metrics_text(want, argv3)


def test_metrics_do_not_depend_on_workers_or_budgets(planted):
    d, prefix, files, tids, _, _ = planted
    w = d / "budgets"; w.mkdir()
    common = ["-K", "20000", prefix] + files["pe"]
    texts, parts, stats = [], [], []
    for k, extra in enumerate((["-p", "1"], ["-p", "3"], ["-p", "2", "--sort-mem", "100K"])):
        st, text, _, out = _run(extra + common, w, "m%d" % k)
        stats.append(st); parts.append(tg._records_part(open(out, "rb").read()))
        texts.append(text.split("\n", 2)[2])                                           # all but the command line
    assert sorted(os.listdir(w)) == ["m0.bam", "m0.txt", "m1.bam", "m1.txt", "m2.bam", "m2.txt"]
    assert texts[0] == texts[1] == texts[2] and parts[0] == parts[1] == parts[2]
    assert stats[2]["dup_sig_runs"] >= 3 and stats[2]["sort_runs"] >= 3 and stats[0]["dup_sig_runs"] == 0
    assert stats[0]["dup_optical_pairs"] == stats[1]["dup_optical_pairs"] == stats[2]["dup_optical_pairs"] > 0

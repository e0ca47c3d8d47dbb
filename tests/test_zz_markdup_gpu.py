"""Duplicate marking on the GPU: bm2_dup_signatures, bm2_dup_resolve and bm2_bam_sort_compress_ex equal the host emulation
(tests/host_emul/markdup_emul.cpp, bam_sort_emul.cpp) byte for byte, and `bm2_mem --markdup` on reads with planted duplicates drawn from the
golden index's reference is, decoded, `--sort`'s records from the same options with the flags of the rule restated in Python
(tests/markdup_util.py) - paired, single-end, smart pairing, FASTA (every score 0: input order decides) and -a -M - with the stderr counts
equal to Python's.  The records' BGZF members are the same at -p 1 and 3 and with a --sort-mem small enough for several signature and
record runs and a pile of duplicates larger than a signature window; no temporary file is left; the .bai reaches exactly the overlapping
records; and on input without duplicates the members equal --sort's."""
import json, os, re, subprocess
import numpy as np
import pytest
import bam_util as bu
import bam_sort_util as bs
import markdup_util as mu
import test_bam_sort_cpu as tsc
import test_markdup_cpu as tmc
import test_zz_bam_gpu as tg

pytestmark = pytest.mark.gpu

TOOL = tg.TOOL


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mu.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def sort_emul(tmp_path_factory):
    return bs.build_emul(tmp_path_factory)


def test_kernels_equal_emulation(gpu_ctx, emul, sort_emul):
    rng = np.random.default_rng(21)
    for t in (tmc.crafted_templates(), mu.random_templates(rng, 3000), mu.random_templates(rng, 3000, paired=False), []):
        data, first, ids = mu.flatten(t)
        starts = np.array([a for a, _ in bu.records(data)], np.int64)
        gp, gf, ms = gpu_ctx.dup_signatures(data, starts, first, ids)
        ep, ef = mu.emul_signatures(emul, data, first, ids)
        assert gp.tobytes() == ep.tobytes() and gf.tobytes() == ef.tobytes()
        assert ms >= 0
    for space in (mu.PAIR, mu.FRAG):
        for n in (1, 1000, 200_000):
            e = mu.entries_array(mu.random_entries(rng, n, space))
            got, ms = gpu_ctx.dup_resolve(e)
            assert np.array_equal(got, mu.emul_resolve(emul, e)), (space, n)
            srt, _ = gpu_ctx.dup_resolve(e, False)
            assert srt.tobytes() == mu.emul_resolve(emul, e, False).tobytes()
    # marking in the coordinate sort: the records of duplicate templates, unless unmapped, get 0x400; the ids come back in output order
    t = mu.random_templates(rng, 4000, piles=30)
    data, first, ids = mu.flatten(t)
    tids = np.repeat(ids, np.diff(first))
    starts = np.array([a for a, _ in bu.records(data)], np.int64)
    pd, fd, _ = mu.duplicates([(tid, [bu.fields(r) for r in recs]) for tid, recs in t])
    dups = set(pd) | set(fd)
    plain = gpu_ctx.bam_sort_compress(data, starts)
    gpu_ctx.dup_set(sorted(dups), int(ids.max()) + 2)
    try:
        got = gpu_ctx.bam_sort_compress_ex(data, starts, tids)
        recs = [r for _, r in bu.records(data)]
        marked = b"".join(mu.set_flag(r, bu.fields(r)["flag"] | 0x400) if int(k) in dups and not bu.fields(r)["flag"] & 4 else r
                          for r, k in zip(recs, tids))
        want = bs.emul_once(sort_emul, marked, starts)
        assert got["z"] == want["z"] and np.array_equal(got["recs"]["flag"], want["recs"]["flag"])
        assert np.array_equal(got["recs"]["block"], want["recs"]["block"]) and np.array_equal(got["recs"]["offset"], want["recs"]["offset"])
        keys = [bs.key(bu.fields(r)) for r in recs]
        order = sorted(range(len(recs)), key=lambda i: keys[i])
        assert np.array_equal(got["tids"], tids[order]) and (got["recs"]["flag"] & 0x400).any()
        assert got["z"] != plain["z"]
        assert gpu_ctx.bam_sort_compress(data, starts)["z"] == plain["z"]             # the plain entry never marks
    finally:
        gpu_ctx.dup_set([], 0)
    assert gpu_ctx.bam_sort_compress_ex(data, starts, tids)["z"] == plain["z"]        # no bitset: no mark


def _write_pairs(d, pairs, name):
    r1 = [(n, a, qa) for n, a, qa, _, _ in pairs]
    r2 = [(n, b, qb) for n, _, _, b, qb in pairs]
    f = {}
    (d / (name + "1.fq")).write_bytes(mu.fastq(r1)); (d / (name + "2.fq")).write_bytes(mu.fastq(r2))
    (d / (name + "1.fa")).write_bytes(mu.fasta(r1)); (d / (name + "2.fa")).write_bytes(mu.fasta(r2))
    inter, tid_inter = [], {}
    for k, (n, a, qa, b, qb) in enumerate(pairs):
        tid_inter[n] = len(inter)
        inter.append((n, a, qa))
        if k % 7 != 3:
            inter.append((n, b, qb))
    (d / (name + "i.fq")).write_bytes(mu.fastq(inter))
    f.update(pe=[str(d / (name + "1.fq")), str(d / (name + "2.fq"))], se=[str(d / (name + "1.fq"))], smart=[str(d / (name + "i.fq"))],
             fasta=[str(d / (name + "1.fa")), str(d / (name + "2.fa"))])
    tid = dict(pe={n: 2 * k for k, (n, *_) in enumerate(pairs)}, se={n: k for k, (n, *_) in enumerate(pairs)}, smart=tid_inter)
    tid["fasta"] = tid["pe"]
    return f, tid


@pytest.fixture(scope="module")
def planted(golden_dir, tmp_path_factory):
    if not os.path.exists(TOOL):
        pytest.skip("bm2_mem not built")
    d = tmp_path_factory.mktemp("markdup_gpu")
    prefix = os.path.join(golden_dir, "c0_index", "ref.fa")
    ref = mu.load_reference(prefix)
    rng = np.random.default_rng(31)
    pairs = mu.planted_pairs(ref, rng, n_base=120)
    files, tids = _write_pairs(d, pairs, "p")
    base = [p for p in pairs if re.fullmatch(r"b\d+", p[0])]                      # the drawn pairs alone: no duplicates
    nd_files, nd_tids = _write_pairs(d, base, "n")
    c = [p for p in pairs if p[0] == "b0"][0]                                     # a pile larger than a signature window
    deep = pairs + [("deep%d" % k, c[1], bytes(int(x) + 33 for x in rng.integers(2, 41, len(c[1]))), c[3],
                     bytes(int(x) + 33 for x in rng.integers(2, 41, len(c[3])))) for k in range(400)]
    order = rng.permutation(len(deep))
    deep_files, deep_tids = _write_pairs(d, [deep[i] for i in order], "d")
    return d, prefix, dict(planted=(files, tids), none=(nd_files, nd_tids), deep=(deep_files, deep_tids))


def _run(args, out):
    r = subprocess.run([TOOL] + args + ["-o", out], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1])


def _records(path):
    raw = bu.inflate(open(path, "rb").read())
    _, _, used = bu.parse_header(raw)
    return [r for _, r in bu.records(raw[used:])]


def _expected(sorted_recs, tid_of_name):
    by = {}
    for r in sorted_recs:
        f = bu.fields(r)
        by.setdefault(f["qname"], []).append(f)
    pd, fd, n = mu.duplicates([(tid_of_name[q], fs) for q, fs in by.items()])
    dups = set(pd) | set(fd)
    want = mu.apply_flags(sorted_recs, lambda r: tid_of_name[bu.fields(r)["qname"]], dups)
    return want, pd, fd, n


@pytest.mark.parametrize("mode,args", [("pe", []), ("se", []), ("smart", ["-p"]), ("fasta", []), ("pe", ["-a", "-M"])])
def test_markdup_equals_python_flags(planted, mode, args):
    d, prefix, sets = planted
    files, tids = sets["planted"]
    w = d / ("m_%s%s" % (mode, "".join(args))); w.mkdir()
    # smart pairing pairs mates within a chunk only (a pair across a chunk boundary is two single-end reads): one chunk, so that a read's
    # name tells its template
    common = args + ["-K", "100000000" if mode == "smart" else "20000", prefix] + files[mode]
    _run(["--sort"] + common, str(w / "sort.bam"))
    st = _run(["--markdup"] + common, str(w / "md.bam"))
    assert sorted(os.listdir(w)) == ["md.bam", "sort.bam"]
    srt, got = _records(w / "sort.bam"), _records(w / "md.bam")
    want, pd, fd, n = _expected(srt, tids[mode])
    assert got == want
    assert (st["dup_pair_templates"], st["dup_fragment_templates"], st["dup_templates"]) == (len(pd), len(fd), n)
    assert st["dup_records"] == sum(bu.fields(r)["flag"] & 0x400 != 0 for r in want) > 0
    assert st["dup_sig_runs"] == 0 and st["dup_sig_bytes"] == 0 and st["markdup_s"] > 0
    if mode != "se":
        assert len(pd) > 20
    if mode == "fasta":
        assert all(bu.fields(r)["qual"][:1] in (b"", b"\xff") for r in srt[:50])
    if mode == "pe" and not args:                                                  # supplementary records are marked with their template
        assert any(bu.fields(r)["flag"] & 0xC00 == 0xC00 for r in got)


def test_members_do_not_depend_on_workers_or_budgets(planted):
    d, prefix, sets = planted
    files, tids = sets["deep"]
    w = d / "budgets"; w.mkdir()
    common = ["-K", "20000", prefix] + files["pe"]
    _run(["--sort"] + common, str(w / "sort.bam"))
    parts, stats = [], []
    for k, extra in enumerate((["-p", "1"], ["-p", "3"], ["-p", "2", "--sort-mem", "100K"])):
        stats.append(_run(["--markdup", "--write-index"] + extra + common, str(w / ("m%d.bam" % k))))
        parts.append(tg._records_part(open(w / ("m%d.bam" % k), "rb").read()))
    assert sorted(os.listdir(w)) == ["m0.bam", "m0.bam.bai", "m1.bam", "m1.bam.bai", "m2.bam", "m2.bam.bai", "sort.bam"]   # no temporary file
    assert parts[0] == parts[1] == parts[2]
    s = stats[2]
    window = (100 << 10) // 8 // 32 // max(s["dup_sig_runs"], 1)
    assert s["dup_sig_runs"] >= 3 and s["dup_sig_bytes"] > 0 and s["sort_runs"] >= 3 and s["spill_bytes"] > 0 and 400 > window
    want, pd, fd, n = _expected(_records(w / "sort.bam"), tids["pe"])
    assert _records(w / "m2.bam") == want and (s["dup_pair_templates"], s["dup_fragment_templates"]) == (len(pd), len(fd))
    assert stats[0]["dup_records"] == s["dup_records"]
    data = open(w / "m2.bam", "rb").read()
    tsc.check_index(str(w / "m2.bam"), str(w / "m2.bam.bai"), len(data) - len(tg._records_part(data)), 4,
                    np.random.default_rng(4))


def test_no_duplicates_equals_sort(planted):
    d, prefix, sets = planted
    files, _ = sets["none"]
    w = d / "nodup"; w.mkdir()
    common = ["-K", "20000", prefix] + files["pe"]
    _run(["--sort"] + common, str(w / "sort.bam"))
    st = _run(["--markdup"] + common, str(w / "md.bam"))
    assert st["dup_records"] == 0 and st["dup_templates"] > 0
    assert tg._records_part(open(w / "md.bam", "rb").read()) == tg._records_part(open(w / "sort.bam", "rb").read())

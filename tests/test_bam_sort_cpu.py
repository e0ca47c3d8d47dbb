"""bm2_mem --sort without a GPU: the coordinate key and reference end of bam_sort_device.cuh against Python's, and bam_sort.h (runs, temporary
files, merge windows, BAI) driven by the host emulation tests/host_emul/bam_sort_emul.cpp, whose bytes the GPU must give.  The decoded output
is Python's stable sort of the input by the key, the bytes do not depend on the run budget, no temporary file survives, and the index reaches
exactly the overlapping records of every region asked.  Plus the option errors of --sort-mem and --write-index, and --dump-opt's fields."""
import json, os, random, subprocess
import numpy as np
import pytest
import bam_util as bu
import bam_inputs
import bam_sort_util as bs
import test_bam_cpu as tb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
IDX = os.path.join(ROOT, "tests", "golden", "c0_index", "ref.fa")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return bs.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def bgzf(tmp_path_factory):
    return tb.build_emul(tmp_path_factory)


def special_records():
    """Unmapped, placed unmapped, reverse strand, CG:B,I, no reference-consuming operation, and a deletion across a 16 kbp window."""
    return b"".join([
        bs.make_rec(-1, -1, 4, name=b"unplaced"),
        bs.make_rec(1, 5000, 4 | 1, name=b"placed_unmapped"),
        bs.make_rec(1, 5000, 16, name=b"reverse"),
        bs.make_rec(0, 70, 0, cigar=((5, 4), (10, 1), (5, 4)), name=b"insertion_only"),
        bs.make_rec(0, 16380, 0, cigar=((10, 0), (100000, 2), (10, 0)), name=b"deletion"),
        bs.make_rec(2, 123, 16, name=b"cg", cg=[(1, 0), (1, 2)] * 40000 + [(1, 0)]),
        bs.make_rec(2, 7, 0, cigar=((20, 0), (300, 3), (20, 7), (5, 8)), name=b"n_eq_x"),
    ])


@pytest.mark.parametrize("which", ["bam_records", "realistic_bam", "special"])
def test_key_and_end_equal_python(emul, which):
    data = {"bam_records": lambda: bam_inputs.bam_records(4000, seed=2)[0], "realistic_bam": lambda: tb.realistic_bam()[0],
            "special": special_records}[which]()
    keys, info = bs.emul_keys(emul, data)
    recs = [r for _, r in bu.records(data)]
    for k, (r, ky, inf) in enumerate(zip(recs, keys, info)):
        f = bu.fields(r)
        assert int(ky) == bs.key(f), k
        assert (inf["rid"], inf["pos"], inf["flag"]) == (f["rid"], f["pos"], f["flag"])
        if f["rid"] >= 0:
            assert inf["end"] == bs.end_pos(f) and inf["bin"] == bu.reg2bin(f["pos"], inf["end"]), k
        else:
            assert inf["bin"] == 4680
    if which == "special":
        by = {bu.fields(r)["qname"]: (int(i["end"]), int(i["pos"])) for r, i in zip(recs, info)}
        assert by["placed_unmapped"] == (5001, 5000) and by["insertion_only"] == (71, 70) and by["deletion"] == (16380 + 100020, 16380)
        assert by["cg"] == (123 + 80001, 123) and by["n_eq_x"] == (7 + 345, 7)


def hostile(name, rng):
    if name == "one_position":
        return b"".join(bs.make_rec(0, 1000, 16, name=b"s%d" % i) for i in range(3000))
    if name == "unmapped_only":
        return b"".join(bs.make_rec(-1, -1, 4 | (16 if i % 3 == 0 else 0), name=b"u%d" % i) for i in range(2500))
    if name == "one_contig":
        return b"".join(bs.make_rec(0, int(rng.integers(0, 3000)), int(rng.choice([0, 16, 4 | 1])), name=b"c%d" % i) for i in range(4000))
    if name == "many_contigs":
        rids = [r for r in range(40) if r % 3 != 1] + [-1]
        out = []
        for i in range(5000):
            rid = int(rng.choice(rids))
            out.append(bs.make_rec(rid, int(rng.integers(0, 200_000)) if rid >= 0 else -1, 4 if rid < 0 else int(rng.choice([0, 16])),
                                   cigar=((int(rng.integers(20, 200)), 0),), name=b"m%d" % i))
        return b"".join(out)
    if name == "big_records":
        out = []
        for i in range(60):
            big = i % 4 == 0
            out.append(bs.make_rec(int(rng.integers(0, 2)), int(rng.integers(0, 50)) * 100, 0, name=b"b%d" % i,
                                   cigar=((70000 if big else 150, 0),), extra=b"XZZ" + bytes(rng.integers(65, 90, 20000 if big else 10, dtype=np.uint8)) + b"\0"))
        return b"".join(out)
    raise KeyError(name)


def decoded_records(path, out_off=0):
    data = open(path, "rb").read()[out_off:]
    return [r for _, r in bu.records(bu.inflate(data))] if data else []


def stable_sorted(data):
    recs = [r for _, r in bu.records(data)]
    return sorted(recs, key=lambda r: bs.key(bu.fields(r)))


@pytest.mark.parametrize("name", ["one_position", "unmapped_only", "one_contig", "many_contigs", "big_records"])
def test_sorted_output_is_the_stable_sort_at_every_budget(emul, tmp_path, name):
    data = hostile(name, np.random.default_rng(sum(name.encode())))
    small = b"".join(r for _, r in bu.records(data)[:150])            # one record per run: a temporary file each
    outs = {}
    for step, budget in enumerate((1 << 40, len(data) // 4 + 1, 1, -1)):  # one run, a few runs, one record per run (and its input in one run)
        d = tmp_path / ("b%d" % step); d.mkdir()
        if budget == 1:
            data, outs = small, {}
            budget = 1
        elif budget == -1:
            budget = 1 << 40
        want = stable_sorted(data)
        out = str(d / "out.bam")
        st = bs.emul_file(emul, data, budget, str(d / "out.bam.tmp."), out, chunk=20000, n_ref=40)
        assert os.listdir(d) == ["out.bam"]                              # no temporary file survives
        assert decoded_records(out) == want
        if budget == 1:
            assert st["runs"] == len(want) and st["windows"] >= 1
        elif budget > len(data):
            assert st["runs"] == 0 and st["spill_bytes"] == 0
        else:
            assert 2 <= st["runs"] <= 6
        outs[len(outs)] = open(out, "rb").read()
        assert len(set(outs.values())) == 1


def test_empty_input(emul, bgzf, tmp_path):
    out = str(tmp_path / "e.bam")
    bs.emul_file(emul, b"", 1000, str(tmp_path / "e.tmp."), out, bai_path=str(tmp_path / "e.bai"), n_ref=2)
    assert open(out, "rb").read() == b""                                 # bm2_mem adds the header before and the EOF block after
    refs, n_no = bs.parse_bai(open(tmp_path / "e.bai", "rb").read())
    assert n_no == 0 and all(not r["bins"] and r["pseudo"] is None and not r["lin"] for r in refs) and len(refs) == 2


def test_carry_gives_the_whole_stream_cut(emul, bgzf):
    """Windows passed one after another with the carry equal the whole sorted stream compressed at once."""
    data, starts = bam_inputs.bam_records(3000, seed=5)
    recs = stable_sorted(data)
    srt = b"".join(recs)
    whole = bs.emul_once(emul, srt, [a for a, _ in bu.records(srt)])
    z, carry, k = b"", b"", 0
    for size in (1, 7, 500, 40, 1000, 2000):                             # consecutive slices of the sorted stream
        part = b"".join(recs[k:k + size])
        k += size
        o = bs.emul_once(emul, part, [a for a, _ in bu.records(part)], carry, last=k >= len(recs))
        z += o["z"]; carry = o["carry"]
    assert carry == b"" and z == whole["z"]
    assert z == tb.emul_stream(bgzf, srt, [a for a, _ in bu.records(srt)])[0]


def check_index(data_file, bai_file, out_off, n_ref, rng, n_regions=200):
    data = open(data_file, "rb").read()
    refs, n_no = bs.parse_bai(open(bai_file, "rb").read())
    assert len(refs) == n_ref
    recs = [r for _, r in bu.records(bu.inflate(data[out_off:]))]
    fs = [bu.fields(r) for r in recs]
    assert n_no == sum(f["rid"] < 0 for f in fs)
    f = bs.BgzfFile(data)
    for rid in range(n_ref):
        mine = [(r, x) for r, x in zip(recs, fs) if x["rid"] == rid]
        p = refs[rid]["pseudo"]
        if not mine:
            assert p is None and not refs[rid]["bins"]
            continue
        assert (p["mapped"], p["unmapped"]) == (sum(not x["flag"] & 4 for _, x in mine), sum(bool(x["flag"] & 4) for _, x in mine))
        assert f.read_records(p["beg"], p["end"]) == [r for r, _ in mine]
        top = max(bs.end_pos(x) for _, x in mine) + 20000
        regions = [(0, 1 << 29)] + [tuple(sorted(rng.integers(0, top, 2))) for _ in range(n_regions)]
        for beg, end in regions:
            end = max(end, beg + 1)
            want = [r for r, x in mine if x["pos"] < end and bs.end_pos(x) > beg]
            assert bs.query(refs, f, rid, int(beg), int(end)) == want, (rid, beg, end)


@pytest.mark.parametrize("budget", [1 << 40, 300_000, 1])
def test_bai_reaches_the_overlapping_records(emul, tmp_path, budget):
    rng = np.random.default_rng(9)
    data = hostile("many_contigs", rng) + special_records() + hostile("big_records", rng)
    if budget == 1:
        data = b"".join(r for _, r in bu.records(data)[::40]) + special_records()
    out, bai = str(tmp_path / "o.bam"), str(tmp_path / "o.bai")
    bs.emul_file(emul, data, budget, str(tmp_path / "o.tmp."), out, bai_path=bai, n_ref=40, chunk=50_000)
    assert sorted(os.listdir(tmp_path)) == ["o.bai", "o.bam"]
    check_index(out, bai, 0, 40, np.random.default_rng(1), n_regions=200 if budget > 1 << 30 else 50)


def _dump(*args):
    return subprocess.run([TOOL, "--dump-opt"] + list(args) + [IDX, "a.fq", "b.fq"], capture_output=True, text=True, timeout=60)


@pytest.mark.skipif(not os.path.exists(TOOL), reason="bm2_mem not built")
def test_options_and_dump_opt():
    plain = _dump()
    assert plain.returncode == 0
    j0 = json.loads(plain.stdout)
    assert "sort" not in j0 and not j0["header"].startswith("@HD")
    j = json.loads(_dump("--sort", "--sort-mem", "300M", "--write-index", "-o", "x.bam").stdout)
    assert j["sort"] is True and j["bam"] is True and j["sort_mem"] == 300 << 20 and j["write_index"] is True
    assert j["header"].split("\n")[0] == "@HD\tVN:1.6\tSO:coordinate" and j["header"].count("@HD") == 1
    assert json.loads(_dump("--sort").stdout)["sort_mem"] == 2 << 30
    for v, n in (("7", 7), ("64k", 64 << 10), ("2G", 2 << 30), ("3m", 3 << 20)):
        assert json.loads(_dump("--sort", "--sort-mem", v).stdout)["sort_mem"] == n
    h = json.loads(_dump("--sort", "-H", "@CO\tfirst", "-H", "@HD\tVN:1.4\tSO:unsorted\tGO:query").stdout)["header"].split("\n")
    assert h[0] == "@HD\tVN:1.4\tSO:coordinate\tGO:query" and "@CO\tfirst" in h and sum(l.startswith("@HD") for l in h) == 1
    for bad in (["--sort-mem", "0"], ["--sort-mem", "12X"], ["--sort-mem", "-5"], ["--sort-mem", "K"], ["--sort-mem"]):
        r = _dump("--sort", *bad) if bad != ["--sort-mem"] else subprocess.run([TOOL, "--sort", "--sort-mem"], capture_output=True, text=True)
        assert r.returncode == 1 and "--sort-mem" in r.stderr, bad
    for bad in (["--write-index", "--sort"], ["--write-index", "-o", "x.bam"], ["--write-index", "--bam", "-o", "x.bam"]):
        r = _dump(*bad)
        assert r.returncode == 1 and "--write-index needs --sort and -o" in r.stderr, bad

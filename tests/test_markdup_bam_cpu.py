"""bm2_markdup on the CPU: the host emulation (tests/host_emul/markdup_bam_emul.cpp, which runs bwa-mem2_b200/csrc/markdup_bam.h unchanged)
writes the BAM records, header and metrics file that the rule restated in Python (tests/markdup_bam_util.py) gives - on crafted records for
each branch of the rule, and on random lanes and libraries at every window size down to one record and with spilled entry runs - and every
error exits 1 and leaves no file."""
import os, subprocess
import numpy as np
import pytest
import markdup_bam_util as mb

RGS = ["@RG\tID:l1\tSM:s\tLB:a", "@RG\tID:l2\tSM:s\tLB:a", "@RG\tID:l3\tSM:s\tLB:b"]


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mb.build_emul(tmp_path_factory)


def _name(lane, t, x, y):
    return "M01:77:FC:%d:%d:%d:%d" % (lane, t, x, y)


def crafted():
    """Two inputs (lanes l1 and l2 of library a, with l3 of library b and records without RG:Z in the second) -> [(header, refs, records)]"""
    r = mb.rec
    one, two = [], []
    # a pair and its copy in the other lane of the same library, optical neighbours by name but in different read groups: a duplicate, not optical
    n1, n2 = _name(1, 1101, 5000, 5000), _name(2, 1101, 5010, 5010)
    one += [r(0, 100, 0x1 | 0x40 | 0x20, n1, mrid=0, mpos=300, rg="l1"), r(0, 300, 0x1 | 0x80 | 0x10, n1, mrid=0, mpos=100, rg="l1")]
    two += [r(0, 100, 0x1 | 0x40 | 0x20, n2, mrid=0, mpos=300, rg="l2", qual=20), r(0, 300, 0x1 | 0x80 | 0x10, n2, mrid=0, mpos=100, rg="l2")]
    # two copies in one read group near each other: optical
    n3, n4 = _name(1, 1102, 700, 700), _name(1, 1102, 750, 720)
    one += [r(0, 1000, 0x1 | 0x40 | 0x20, n3, mrid=0, mpos=1200, rg="l1"), r(0, 1200, 0x1 | 0x80 | 0x10, n3, mrid=0, mpos=1000, rg="l1")]
    one += [r(0, 1000, 0x1 | 0x40 | 0x20, n4, mrid=0, mpos=1200, rg="l1"), r(0, 1200, 0x1 | 0x80 | 0x10, n4, mrid=0, mpos=1000, rg="l1")]
    # the same keys in library b: kept apart (not a duplicate of library a's pair)
    n5 = _name(3, 1101, 9000, 9000)
    two += [r(0, 100, 0x1 | 0x40 | 0x20, n5, mrid=0, mpos=300, rg="l3"), r(0, 300, 0x1 | 0x80 | 0x10, n5, mrid=0, mpos=100, rg="l3")]
    # the same QNAME in two read groups: two pairs, not joined across
    n6 = "same:name"
    one += [r(1, 500, 0x1 | 0x40 | 0x20, n6, mrid=1, mpos=800, rg="l1"), r(1, 800, 0x1 | 0x80 | 0x10, n6, mrid=1, mpos=500, rg="l1")]
    two += [r(1, 500, 0x1 | 0x40 | 0x20, n6, mrid=1, mpos=800, rg="l3"), r(1, 800, 0x1 | 0x80 | 0x10, n6, mrid=1, mpos=500, rg="l3")]
    # fragments with tied scores (the lowest ordinal kept), one with a lower score, and a mapped read with an unmapped mate (stale 0x400)
    one += [r(1, 2000, 0, "f1", rg="l1"), r(1, 2000, 0, "f2", rg="l1"), r(1, 2000, 0x400, "f3", rg="l1", qual=10)]
    one += [r(1, 3000, 0x1 | 0x40 | 0x8, "mu", mrid=1, mpos=3000, rg="l1"), r(1, 3000, 0x1 | 0x80 | 0x4 | 0x400, "mu", (), mrid=1, mpos=3000, rg="l1")]
    # a fragment over the pair-end of a pair: a duplicate
    one += [r(0, 1000, 0, "fp", rg="l1")]
    # secondary and supplementary records with a stale 0x400
    one += [r(0, 1500, 0x1 | 0x40 | 0x100 | 0x400, n3, mrid=0, mpos=1200, rg="l1"), r(0, 1600, 0x1 | 0x80 | 0x800 | 0x400, n3, mrid=0, mpos=1000, rg="l1")]
    # mates on another contig, carried across windows; records without RG:Z
    n7 = _name(2, 1101, 100, 100)
    two += [r(0, 5000, 0x1 | 0x40, n7, mrid=2, mpos=40, rg="l2"), r(2, 40, 0x1 | 0x80 | 0x10, n7, mrid=0, mpos=5000, rg="l2")]
    two += [r(0, 5000, 0x1 | 0x40, "norg", mrid=2, mpos=40), r(2, 40, 0x1 | 0x80 | 0x10, "norg", mrid=0, mpos=5000)]
    # both unmapped, at the end
    two += [r(-1, -1, 0x1 | 0x40 | 0x4 | 0x8, "uu", (), rg="l2"), r(-1, -1, 0x1 | 0x80 | 0x4 | 0x8, "uu", (), rg="l2")]
    pg1 = ["@PG\tID:bm2_mem\tPN:bm2_mem\tCL:bm2_mem lane1"]
    pg2 = ["@PG\tID:bm2_mem\tPN:bm2_mem\tCL:bm2_mem lane2", "@PG\tID:samtools\tPN:samtools\tPP:bm2_mem\tCL:samtools view"]
    h1, refs = mb.header(RGS[:1], pg1, ["@CO\tlane one"])
    h2, _ = mb.header(RGS, pg2, ["@CO\tlane two"])
    return [(h1, refs, mb.sort_recs(one)), (h2, refs, mb.sort_recs(two))]


def _write(d, ins, stem="in"):
    paths = []
    for k, (h, refs, recs) in enumerate(ins):
        p = str(d / ("%s%d.bam" % (stem, k)))
        mb.write_bam(p, h, refs, recs, 97)                  # small members, so that small windows hold few records
        paths.append(p)
    return paths


def _check(emul, wd, paths, tag, **kw):
    out, met, bai = str(wd / (tag + ".bam")), str(wd / (tag + ".txt")), str(wd / (tag + ".bam.bai"))
    rc, msg, st = mb.emul_run(emul, paths, out, met, bai, args="-M x", **kw)
    assert rc == 0, msg
    text, recs, mtext, ws = mb.markdup_files(paths, args="-M x", d=kw.get("d", 100))
    got_text, _, got = mb.read_bam(out)
    assert got_text == text and got == recs and open(met).read() == mtext
    for k in ("records", "pairs", "fragments", "dup_pair_templates", "dup_fragment_templates", "dup_records", "dup_optical_pairs", "libraries"):
        assert st[k] == ws[k], k
    assert not [f for f in os.listdir(wd) if f.endswith(".tmp") or ".tmp." in f]
    return st, open(out, "rb").read(), open(met).read(), open(bai, "rb").read()


def test_crafted_records_equal_python(emul, tmp_path):
    ins = crafted()
    paths = _write(tmp_path, ins)
    st, bam, met, bai = _check(emul, tmp_path, paths, "a")
    text, recs, _, ws = mb.markdup_files(paths, args="-M x")
    assert "@PG\tID:bm2_mem.1\tPN:bm2_mem\tCL:bm2_mem lane2" in text and "@PG\tID:samtools\tPN:samtools\tPP:bm2_mem.1" in text
    assert "\tPP:bm2_mem\tVN:b200-r2" in text and text.count("@RG\tID:l1") == 1 and "@CO\tlane one\n@CO\tlane two\n" in text
    flags = {}
    for r in recs:
        f = mb.bu.fields(r)
        flags.setdefault((f["qname"], mb._rg_value(r)), []).append(f["flag"])
    dup = lambda k: [bool(x & 0x400) for x in flags[k]]
    n1, n2 = _name(1, 1101, 5000, 5000), _name(2, 1101, 5010, 5010)
    assert dup((n1, "l1")) == [False, False] and dup((n2, "l2")) == [True, True]          # the lower score loses, across lanes
    assert dup((_name(3, 1101, 9000, 9000), "l3")) == [False, False]                       # library b kept apart
    assert dup(("same:name", "l1")) == [False, False] and dup(("same:name", "l3")) == [False, False]
    assert dup(("f1", "l1")) == [False] and dup(("f2", "l1")) == [True] and dup(("f3", "l1")) == [True]
    assert dup(("mu", "l1")) == [False, False] and dup(("fp", "l1")) == [True] and dup(("uu", "l2")) == [False, False]
    assert not any(x & 0x400 for x in flags[(_name(1, 1102, 700, 700), "l1")])            # secondary and supplementary cleared
    assert ws["dup_optical_pairs"] == 1 and ws["libraries"] == 3
    rows = [l.split("\t")[0] for l in met.split("\n")[5:] if l]
    assert rows == ["Unknown Library", "a", "b"] and "CoverageMult" not in met
    for w in (1, 200, 4096):                                                                # one record per window and up
        st2, bam2, met2, bai2 = _check(emul, tmp_path, paths, "w%d" % w, window=w)
        assert bam2 == bam and met2 == met and bai2 == bai
        if w == 1:
            assert st2["pending_max"] >= 2 and st2["windows"] >= len(recs) // 4


def test_random_lanes_equal_python(emul, tmp_path):
    rng = np.random.default_rng(71)
    lanes = [("l1", "a"), ("l2", "a"), ("l3", "b")]
    by = mb.random_lanes(rng, 600, lanes)
    rgs = ["@RG\tID:%s\tSM:s\tLB:%s" % l for l in lanes]
    ins = [(mb.header(rgs[:2] if k < 2 else rgs)[0], mb.header()[1], mb.sort_recs(by[rg])) for k, (rg, _) in enumerate(lanes)]
    paths = _write(tmp_path, ins)
    base = None
    for tag, kw in [("big", {}), ("w1", dict(window=1)), ("w3k", dict(window=3000, threads=3)), ("spill", dict(window=2000, sig_bytes=4096)),
                    ("both", dict(window=20000, sig_bytes=2048))]:
        st, bam, met, bai = _check(emul, tmp_path, paths, tag, **kw)
        if base is None:
            base = (bam, met, bai)
            assert st["dup_pair_templates"] > 20 and st["dup_fragment_templates"] > 5 and st["dup_optical_pairs"] > 0
        assert (bam, met, bai) == base, tag
        if tag == "spill":
            assert st["dup_sig_runs"] >= 3
    st, _, met, _ = _check(emul, tmp_path, paths, "d0", d=0)
    assert st["dup_optical_pairs"] < mb.markdup_files(paths, args="-M x")[3]["dup_optical_pairs"]
    # one lane, one library: one row and its histogram
    ins1 = [(mb.header(rgs[:1])[0], mb.header()[1], mb.sort_recs(by["l1"]))]
    p1 = _write(tmp_path, ins1, "one")
    _, _, met1, _ = _check(emul, tmp_path, p1, "one")
    assert "CoverageMult" in met1 and len([l for l in met1.split("\n")[5:] if l and not l[0].isdigit() and not l.startswith(("#", "BIN"))]) == 1


def _errors():
    r = mb.rec
    h, refs = mb.header(RGS[:1])
    pair = [r(0, 100, 0x41 | 0x20, "p", mrid=0, mpos=300, rg="l1"), r(0, 300, 0x81 | 0x10, "p", mrid=0, mpos=100, rg="l1")]
    yield "missing mate", [(h, refs, pair[:1])], "read p"
    yield "third mate", [(h, refs, mb.sort_recs(pair + [r(0, 400, 0x41, "p", mrid=0, mpos=500, rg="l1")]))], "read p"
    yield "mate flag", [(h, refs, [pair[0], r(0, 300, 0x81 | 0x4, "p", (), mrid=0, mpos=100, rg="l1")])], "read p"
    yield "order", [(h, refs, [r(0, 300, 0, "f2", rg="l1"), r(0, 100, 0, "f1", rg="l1")])], "read f1 is out of coordinate order"
    yield "sq", [(h, refs, pair), (mb.header(RGS[:1], sq=(("c0", 100000),))[0], [("c0", 100000)], [])], "@SQ"
    yield "rg", [(h, refs, pair), (mb.header(["@RG\tID:l1\tSM:other"])[0], refs, [])], "read group l1"
    yield "unsorted", [(mb.header(RGS[:1], so="unsorted")[0], refs, pair)], "coordinate"


@pytest.mark.parametrize("case", [c[0] for c in _errors()])
def test_errors_exit_1_and_leave_no_file(emul, tmp_path, case):
    _, ins, text = next(c for c in _errors() if c[0] == case)
    paths = _write(tmp_path, ins)
    for w in (256 << 20, 1):
        out, met = str(tmp_path / "o.bam"), str(tmp_path / "m.txt")
        rc, msg, _ = mb.emul_run(emul, paths, out, met, out + ".bai", window=w)
        assert rc == 1 and text in msg, msg
        with pytest.raises(mb.MarkdupError):
            mb.markdup_files(paths)
        assert sorted(os.listdir(tmp_path)) == sorted(os.path.basename(p) for p in paths)


def test_option_errors(tmp_path):
    if not os.path.exists(mb.TOOL):
        pytest.skip("bm2_markdup not built")
    p = str(tmp_path / "a.bam")
    h, refs = mb.header()
    mb.write_bam(p, h, refs, [])
    for argv, text in [([p], "-M is required"), (["-M", str(tmp_path / "m.txt"), "-"], "standard input"),
                       (["-M", str(tmp_path / "m.txt"), "--write-index", p], "--write-index needs -o"),
                       (["-M", str(tmp_path / "m.txt"), "--window", "0", p], "--window"), (["-M", str(tmp_path / "m.txt")], "no input"),
                       (["-M", str(tmp_path / "m.txt"), "--optical-distance", "-1", p], "--optical-distance")]:
        r = subprocess.run([mb.TOOL] + argv, capture_output=True, timeout=60)
        assert r.returncode == 1 and text in r.stderr.decode(), (argv, r.stderr)
    assert sorted(os.listdir(tmp_path)) == ["a.bam"]


def collision_halves(rng, n=400):
    """Halves in ordinal order with forced hash collisions: names drawn from a few, hashes from fewer, read groups from two, so that runs of
    equal (hash, read group) mix different names, and a name appears once, twice or three times."""
    names = [b"r%d" % k for k in range(n // 3)]
    out = []
    for _ in range(n):
        nm = names[int(rng.integers(0, len(names)))]
        out.append((int(rng.integers(0, 4)), int(rng.integers(0, 2)), nm))            # hash 0..3: every run is a collision
    return out


def test_pairing_joins_names_not_hashes(emul):
    rng = np.random.default_rng(91)
    for halves in ([], [(7, 0, b"a")], [(7, 0, b"a"), (7, 0, b"b"), (7, 0, b"a")], [(7, 0, b"a"), (7, 1, b"a")],
                   [(1, 0, b"x"), (1, 0, b"x"), (1, 0, b"x")], collision_halves(rng)):
        want = mb.pair_halves(halves, None)
        assert mb.emul_pair(emul, halves) == want
    assert mb.emul_pair(emul, [(7, 0, b"a"), (7, 0, b"b"), (7, 0, b"a")]) == [2, -1, 0]     # the collision of a and b joins nothing


def rg_groups(rng, n=3000, d=100):
    """Located pair entries in groups of about 40 members (the exact cell pass), their read groups in loc's bits 2 and up"""
    import markdup_metrics_util as mm
    e = mm.located_entries(rng, n, max(n // 40, 1), d)
    e["loc"] |= rng.integers(0, 3, n).astype(np.int32) << 2
    return e


def test_optical_keeps_read_groups_apart(emul):
    import markdup_metrics_util as mm
    rng = np.random.default_rng(93)
    for d in (0, 100, 2500):
        e = rg_groups(rng, d=d)
        groups = {}
        for x in e:
            groups.setdefault((int(x["k1"]), int(x["k2"])), []).append((int(x["loc"]), int(x["tile"]), int(x["x"]), int(x["y"])))
        assert max(len(g) for g in groups.values()) > 32
        _, opt = mb.emul_resolve_ex(emul, e, d)
        assert opt == sum(mm.optical_count(g, d) for g in groups.values())
        flat = e.copy(); flat["loc"] &= 3
        assert opt < mb.emul_resolve_ex(emul, flat, d)[1]                                # without read groups more members link


def big_group():
    """One pair copied 40 times on one tile within a few pixels, half in lane l1 and half in l2 of library a: a group for the exact cell
    pass whose optical links stay within a read group"""
    r = mb.rec
    one, two = [], []
    for k in range(40):
        lane = k % 2
        n = _name(lane + 1, 1101, 4000 + 3 * k, 4000 + 2 * k)
        rg = "l%d" % (lane + 1)
        recs = [r(0, 2000, 0x1 | 0x40 | 0x20, n, mrid=0, mpos=2300, rg=rg, qual=20 + k % 7),
                r(0, 2300, 0x1 | 0x80 | 0x10, n, mrid=0, mpos=2000, rg=rg)]
        (one if lane == 0 else two).extend(recs)
    return [(mb.header(RGS[:1])[0], mb.header()[1], mb.sort_recs(one)), (mb.header(RGS[:2])[0], mb.header()[1], mb.sort_recs(two))]


def test_big_group_across_read_groups(emul, tmp_path):
    paths = _write(tmp_path, big_group(), "g")
    st, _, met, _ = _check(emul, tmp_path, paths, "g")
    assert st["dup_pair_templates"] == 39 and st["dup_optical_pairs"] == 38                # 20 + 20 members, one component per read group
    for w in (1, 500):
        assert _check(emul, tmp_path, paths, "out%d" % w, window=w)[2] == met


def test_spill_failure_in_the_sorter_thread_is_an_error(emul, tmp_path):
    rng = np.random.default_rng(95)
    by = mb.random_lanes(rng, 300, [("l1", "a")])
    paths = _write(tmp_path, [(mb.header(RGS[:1])[0], mb.header()[1], mb.sort_recs(by["l1"]))], "s")
    out, met = str(tmp_path / "o.bam"), str(tmp_path / "no_such_dir" / "m.txt")                # the spill files cannot be created
    rc, msg, _ = mb.emul_run(emul, paths, out, met, "", window=2000, sig_bytes=2048)
    assert rc == 2 and "cannot create the temporary file" in msg
    assert sorted(os.listdir(tmp_path)) == ["s0.bam"]

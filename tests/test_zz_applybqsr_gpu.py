"""bm2_applybqsr on the GPU: bm2_bqsr_apply equals the host emulation (tests/host_emul/applybqsr_emul.cpp) on crafted and random records,
read errors included, and its members are those bgzf_emul makes of the expected records cut by htslib's rule; `bm2_applybqsr` on the BAM and
table of `bm2_mem --recal-file` (paired, single-end, smart pairing, -R with and without PU) writes the input's records with the QUAL bytes
Python computes, the input's header plus its @PG line, and a BAI that answers region queries; two read groups are recalibrated by their own
tables; the bytes do not depend on -t, --window or standard input; the error cases exit 1 and leave no output."""
import json, os, re, subprocess
import numpy as np
import pytest
import applybqsr_util as aq
import bam_sort_util as bs
import bam_util as bu
import bqsr_util as bq
import test_bam_cpu as tb
import test_zz_bqsr_gpu as tbq

pytestmark = pytest.mark.gpu

TOOL = aq.TOOL
planted = tbq.planted


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return aq.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def bgzf(tmp_path_factory):
    return tb.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def ref(golden_dir):
    return bq.Ref(os.path.join(golden_dir, "c0_index", "ref.fa"))


def test_kernel_equals_emulation(gpu_ctx, emul, bgzf, ref):
    rng = np.random.default_rng(71)
    tabs = aq.dense(aq.gatk_table(rng, ["fc.1", "fc.2", "fc.3"]))
    ids, tab = ["a", "b", "fc.3", "nope"], [0, 1, 2, -1]
    gpu_ctx.bqsr_apply_set(tabs[1], tabs[2], tabs[3], ids, tab)
    for recs in (aq.crafted(ref, rng, ids), aq.random_records(ref, rng, 5000, ids), []):
        want = aq.emul_apply(emul, recs, ids, tab, tabs)
        assert want[1] is None
        data, starts = bq.flatten(recs)
        carry, z, got_recs = b"", b"", []
        cut = len(recs) // 3
        for part, last in ((recs[:cut], False), (recs[cut:], True)):                   # two calls with the carry between them
            d, s = bq.flatten(part)
            o = gpu_ctx.bqsr_apply(d, s, carry, last)
            z += o["z"]; carry = o["carry"]
            got_recs += list(o["recs"])
        raw = bu.inflate(z) if z else b""
        assert raw == b"".join(want[0])
        zz, _ = tb.emul_stream(bgzf, raw, [int(x) for x in starts]) if raw else (b"", None)
        assert z == zz                                                                   # the members of htslib's cut
        assert len(got_recs) == len(recs)
        for r, g in zip(want[0], got_recs):
            f = bu.fields(r)
            assert (g["rid"], g["pos"], g["flag"]) == (f["rid"], f["pos"], f["flag"])
        st = gpu_ctx.bqsr_apply_stats()
        assert (st["recal_records"], st["kept_records"], st["bases_changed"]) == want[2:] and st["err_kind"] == 0
        gpu_ctx.bqsr_apply_set(tabs[1], tabs[2], tabs[3], ids, tab)
    ok = aq.with_tags(bq.make_rec("ok", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50), aq.rg_tag("a"))
    for bad, kind, msg in ((aq.with_tags(bq.make_rec("long", 0, 0, 100, [(501, 0)], ref.seq(0, 100, 501), [30] * 501), aq.rg_tag("b")), 1,
                            "read long is longer than 500 bases"),
                           (aq.with_tags(bq.make_rec("hiq", 16, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [94] * 50), aq.rg_tag("a")), 2,
                            "read hiq has a base quality above 93")):
        recs = [ok, ok, bad, ok]
        assert aq.emul_apply(emul, recs, ids, tab, tabs)[1] == (2, kind)
        gpu_ctx.bqsr_apply_set(tabs[1], tabs[2], tabs[3], ids, tab)
        d, s = bq.flatten(recs)
        with pytest.raises(Exception, match=msg):
            gpu_ctx.bqsr_apply(d, s)
        st = gpu_ctx.bqsr_apply_stats()
        assert (st["err_kind"], st["err_index"], st["err_name"]) == (kind, 2, bu.fields(bad)["qname"])


def _apply(args, timeout=900, stdin=None):
    r = subprocess.run([TOOL] + args, capture_output=True, timeout=timeout, stdin=stdin)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1])


def _header_records(path):
    raw = bu.inflate(open(path, "rb").read())
    text, refs, used = bu.parse_header(raw)
    return text, refs, [r for _, r in bu.records(raw[used:])]


def _check(inp, table, out, args):
    """out equals Python's recalibration of inp by table; its header is inp's plus the @PG line; its BAI answers region queries."""
    text, refs, recs = _header_records(inp)
    tabs = aq.dense(open(table).read())
    ids, tab = aq.header_map(text, tabs[0])
    want, err, recal, kept, changed = aq.apply_all(recs, ids, tab, tabs)
    otext, orefs, got = _header_records(out)
    assert err is None and got == want and orefs == refs
    last_pg = [l for l in text.split("\n") if l.startswith("@PG\t")][-1].split("\t")[1][3:]
    assert otext == text + "@PG\tID:bm2_applybqsr\tPN:bm2_applybqsr\tPP:%s\tVN:b200-r2\tCL:%s %s\n" % (last_pg, TOOL, " ".join(args))
    data = open(out, "rb").read()
    assert data.endswith(bu.EOF_BLOCK)
    bai_refs, _ = bs.parse_bai(open(out + ".bai", "rb").read())
    bg = bs.BgzfFile(data)
    for rid, (name, ln) in enumerate(refs):
        for beg, end in ((0, ln), (ln // 3, ln // 3 + 500), (ln // 2, ln // 2 + 20000)):
            q = bs.query(bai_refs, bg, rid, beg, end)
            w = [r for r in got if bu.fields(r)["rid"] == rid and bu.fields(r)["pos"] < end and bs.end_pos(bu.fields(r)) > beg]
            assert q == w
    return recal, kept, changed


@pytest.mark.parametrize("mode,rg", [("pe", r"@RG\tID:g1\tSM:s"), ("se", r"@RG\tID:g1\tSM:s\tPU:fc.1"), ("smart", r"@RG\tID:g7\tPU:x.2"),
                                     ("pe", r"@RG\tID:g1\tPU:fc.3\tLB:l")])
def test_applybqsr_equals_python(planted, mode, rg):
    d, prefix, files, sites = planted
    w = d / ("a_%s_%d" % (mode, len(rg))); w.mkdir()
    known = ["--known-sites", str(d / "a.vcf"), "--known-sites", str(d / "b.vcf.gz")]
    tbq._run(["--recal-file", str(w / "t.txt")] + known + ["--write-index", "-R", rg, "-K", "100000000" if mode == "smart" else "20000", prefix]
             + files[mode] + (["-p"] if mode == "smart" else []) + ["-o", str(w / "md.bam")])
    args = ["--bqsr-recal-file", str(w / "t.txt"), "--write-index", "-o", str(w / "r.bam"), str(w / "md.bam")]
    st = _apply(args)
    assert sorted(os.listdir(w)) == ["md.bam", "md.bam.bai", "r.bam", "r.bam.bai", "t.txt"]
    recal, kept, changed = _check(str(w / "md.bam"), str(w / "t.txt"), str(w / "r.bam"), args)
    assert (st["recal_records"], st["unrecalibrated_records"], st["recal_bases"]) == (recal, kept, changed)
    assert st["records"] == recal + kept and recal > 0 and changed > 0 and st["windows"] == 1
    assert st["out_bytes"] == os.path.getsize(w / "r.bam") and st["in_bytes"] == os.path.getsize(w / "md.bam")


def test_two_read_groups(planted, tmp_path, ref):
    rng = np.random.default_rng(72)
    text = "@HD\tVN:1.6\tSO:unsorted\n@RG\tID:one\tPU:u.1\n@RG\tID:two\tPU:u.2\n@PG\tID:bm2_applybqsr\tPN:x\n"
    recs = aq.random_records(ref, rng, 4000, ["one", "two"])
    h = b"BAM\x01" + len(text).to_bytes(4, "little") + text.encode() + len(ref.names).to_bytes(4, "little")
    for n, ln in zip(ref.names, ref.lens):
        h += (len(n) + 1).to_bytes(4, "little") + n.encode() + b"\0" + ln.to_bytes(4, "little")
    (tmp_path / "in.bam").write_bytes(bq.bgzf(h + b"".join(recs)))
    (tmp_path / "t.txt").write_text(aq.gatk_table(rng, ["u.2", "u.1"]))
    args = ["--bqsr-recal-file", str(tmp_path / "t.txt"), "-o", str(tmp_path / "o.bam"), str(tmp_path / "in.bam")]
    _apply(args)
    otext, _, got = _header_records(str(tmp_path / "o.bam"))
    tabs = aq.dense(open(tmp_path / "t.txt").read())
    want = aq.apply_all(recs, ["one", "two"], [1, 0], tabs)[0]
    assert got == want and want != aq.apply_all(recs, ["one", "two"], [0, 1], tabs)[0]
    assert otext.endswith("@PG\tID:bm2_applybqsr.1\tPN:bm2_applybqsr\tPP:bm2_applybqsr\tVN:b200-r2\tCL:%s %s\n" % (TOOL, " ".join(args)))


def test_bytes_do_not_depend_on_threads_windows_or_stdin(planted, tmp_path):
    d, prefix, files, sites = planted
    tbq._run(["--recal-file", str(tmp_path / "t.txt"), "--known-sites", str(d / "a.vcf"), "-R", r"@RG\tID:g1\tSM:s", "-K", "20000", prefix]
             + files["pe"] + ["-o", str(tmp_path / "md.bam")])
    outs, stats = [], []
    for k, extra in enumerate((["-t", "1"], ["-t", "8"], ["-t", "8", "--window", "64K"], ["-t", "3", "--window", "1M"])):
        stats.append(_apply(["--bqsr-recal-file", str(tmp_path / "t.txt"), "-o", str(tmp_path / ("o%d.bam" % k))] + extra + [str(tmp_path / "md.bam")]))
        outs.append(open(tmp_path / ("o%d.bam" % k), "rb").read())
    with open(tmp_path / "md.bam", "rb") as f:
        r = subprocess.run([TOOL, "--bqsr-recal-file", str(tmp_path / "t.txt"), "-"], stdin=f, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    hdr_len = lambda b: len(bu.members(b)[0][0])                                     # the @PG command lines differ: compare what follows
    bodies = [o[hdr_len(o):] for o in outs + [r.stdout]]
    assert all(b == bodies[0] for b in bodies) and stats[2]["windows"] >= 2 and stats[0]["windows"] == 1
    assert len({s["recal_bases"] for s in stats}) == 1 and stats[0]["recal_bases"] > 0


def test_errors(planted, tmp_path):
    d, prefix, files, sites = planted
    tbq._run(["--recal-file", str(tmp_path / "t.txt"), "--known-sites", str(d / "a.vcf"), "-R", r"@RG\tID:g1\tSM:s", "-K", "20000", prefix]
             + files["pe"] + ["-o", str(tmp_path / "md.bam")])
    tbq._run(["--bam", "-R", r"@RG\tID:g1\tSM:s", prefix] + files["fasta"] + ["-o", str(tmp_path / "fa.bam")])
    _apply(["--bqsr-recal-file", str(tmp_path / "t.txt"), "-o", str(tmp_path / "fa_out.bam"), str(tmp_path / "fa.bam")])
    assert _header_records(str(tmp_path / "fa_out.bam"))[2] == _header_records(str(tmp_path / "fa.bam"))[2]   # QUAL '*': unchanged
    t = re.sub(r"(\nmaximum_cycle_value +)500\b", r"\g<1>400", open(tmp_path / "t.txt").read())
    (tmp_path / "t400.txt").write_text(t)
    for args, msg in ((["--bqsr-recal-file", str(tmp_path / "t400.txt"), "-o", str(tmp_path / "e1.bam"), str(tmp_path / "md.bam")],
                       "maximum_cycle_value is 400"),
                      (["--bqsr-recal-file", str(tmp_path / "t.txt"), "--write-index", "-o", str(tmp_path / "e2.bam"), str(tmp_path / "fa.bam")],
                       "needs a coordinate-sorted input"),
                      (["--bqsr-recal-file", str(tmp_path / "t.txt"), "--write-index", str(tmp_path / "md.bam")], "--write-index needs -o")):
        r = subprocess.run([TOOL] + args, capture_output=True, timeout=900)
        assert r.returncode == 1 and msg in r.stderr.decode() and not r.stdout, (args, r.stderr[-2000:])
    assert sorted(os.listdir(tmp_path)) == ["fa.bam", "fa_out.bam", "md.bam", "t.txt", "t400.txt"]

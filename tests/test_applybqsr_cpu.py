"""bm2_applybqsr without a GPU: the host emulation (tests/host_emul/applybqsr_emul.cpp: bqsr_report.h's table parser and deltas,
bqsr_device.cuh's apply rule, bam_window.h's window reader) equals the rule restated in Python (tests/applybqsr_util.py) on bm2_mem-shaped
and GATK-shaped tables and a prior grid, on crafted records for each branch and on random ones; each malformed table is an error naming its
line; the window reader gives the same records at every window size and names truncated input, and warns on a missing EOF block."""
import os, struct, subprocess, zlib
import numpy as np
import pytest
import applybqsr_util as aq
import bam_util as bu
import bqsr_util as bq

IDX = os.path.join(aq.ROOT, "tests", "golden", "c0_index", "ref.fa")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return aq.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def ref():
    return bq.Ref(IDX)


def _same_dense(a, b):
    return a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:]))


def test_tables_equal_python(emul, ref):
    rng = np.random.default_rng(61)
    recs = bq.random_records(ref, rng, 800)
    t = bq.count(recs, ref, *bq.sites_bits(ref, bq.random_sites(ref, rng)))
    texts = [bq.report_text(t, "fc.1")]                                                   # as bm2_mem --recal-file writes it
    texts.append(aq.gatk_table(rng, ["g1", "g2.PU", "lane3"]))                            # GATK-shaped: I / D rows, fractional Errors
    texts.append(aq.gatk_table(rng, ["a", "b", "c"], shuffle=True))                       # the columns in another order
    grid = [k + d for k in (12, 20, 27, 30, 37) for d in (-0.5, -1e-4, 0.0, 1e-4, 0.4999, 0.5)]
    for k in range(0, len(grid), 6):                                                      # (int) (Q - prior) on both sides of an integer
        texts.append(aq.gatk_table(rng, ["p%d" % j for j in range(6)], priors=grid[k:k + 6]))
    for text in texts:
        want = aq.dense(text)
        got = aq.emul_dense(emul, text)
        assert _same_dense(got, want)
        assert len(got[0]) >= 1 and np.any(got[2] != 0) and np.any(got[3] != 0)


def test_malformed_tables_name_the_line(emul, tmp_path):
    rng = np.random.default_rng(62)
    good = aq.gatk_table(rng, ["g1", "g2"])
    lines = good.split("\n")

    def at(prefix, pred=lambda l: True):
        return next(k for k, l in enumerate(lines) if l.startswith(prefix) and pred(l))

    def edit(k, new):
        return "\n".join(lines[:k] + [new] + lines[k + 1:])

    t2 = at("#:GATKTable:RecalTable2") + 2                                                # RecalTable2's first row (0-based)
    row = lines[t2].split()
    cyc_row = at("g1", lambda l: " Cycle " in l)
    cases = [
        (aq.gatk_table(rng, ["g"], args={"maximum_cycle_value": "400"}), "argument maximum_cycle_value is 400, not 500", None),
        (aq.gatk_table(rng, ["g"], args={"mismatches_context_size": "3"}), "argument mismatches_context_size is 3", None),
        (aq.gatk_table(rng, ["g"], args={"low_quality_tail": "3"}), "argument low_quality_tail is 3", None),
        (aq.gatk_table(rng, ["g"], args={"covariate": "ReadGroupCovariate,QualityScoreCovariate"}), "argument covariate is", None),
        (edit(t2, lines[t2].replace(" " + row[1] + " ", " 94 ", 1)), "quality 94 is not in 0..93", t2 + 1),
        (edit(t2, lines[t2].replace(" " + row[2] + " ", " AN ", 1) if row[3] == "Context" else lines[t2]), "context AN is not two of ACGT", t2 + 1),
        (edit(cyc_row, lines[cyc_row].replace(" " + lines[cyc_row].split()[2] + " ", " 501 ", 1)), "cycle 501 is not in +-1..500", cyc_row + 1),
        (edit(cyc_row, lines[cyc_row].replace(" " + lines[cyc_row].split()[2] + " ", " 0 ", 1)), "cycle 0 is not in +-1..500", cyc_row + 1),
        (edit(t2, lines[t2].replace(" " + row[-1], " x" + row[-1][1:], 1)), "a number does not parse", t2 + 1),
        (good.replace("#:GATKTable:RecalTable1:", "#:GATKTable:RecalTableX:"), "no table RecalTable1", len(lines)),
        (good.replace("EstimatedQReported", "EstimatedQ"), "has no column EstimatedQReported", at("ReadGroup") + 1),
        (edit(t2, " ".join(row[:-1])), "cells, the header has 8", t2 + 1),
        ("not a report\n", "not a GATKReport v1.1 file", 1),
    ]
    assert row[3] == "Context"
    for text, msg, line in cases:
        with pytest.raises(ValueError) as e:
            aq.emul_dense(emul, text, path="bad.txt")
        s = str(e.value)
        assert msg in s and s.startswith("bad.txt:"), (msg, s)
        if line is not None:
            assert s.startswith("bad.txt:%d: " % line), (msg, s, line)
    # the argument errors name the argument's own line
    t = aq.gatk_table(rng, ["g"], args={"maximum_cycle_value": "400"})
    k = next(i for i, l in enumerate(t.split("\n")) if l.startswith("maximum_cycle_value"))
    with pytest.raises(ValueError, match="^t.txt:%d: " % (k + 1)):
        aq.emul_dense(emul, t)


def _tabs_for(rng, rgs):
    text = aq.gatk_table(rng, rgs)
    return aq.dense(text)


def test_crafted_records_equal_python(emul, ref):
    rng = np.random.default_rng(63)
    tabs = _tabs_for(rng, ["fc.1", "fc.2", "fc.3"])
    header = "@HD\tVN:1.6\n@RG\tID:a\tPU:fc.1\n@RG\tID:b\tPU:fc.2\tSM:s\n@RG\tID:fc.3\n@RG\tID:nope\tPU:other\n"
    ids, tab = aq.header_map(header, tabs[0])
    assert tab == [0, 1, 2, -1]
    recs = aq.crafted(ref, rng, ["a", "b", "fc.3", "nope"])
    want = aq.apply_all(recs, ids, tab, tabs)
    got = aq.emul_apply(emul, recs, ids, tab, tabs)
    assert got == want
    out, err, recal, kept, changed = got
    by = {bu.fields(r)["qname"]: (r, o) for r, o in zip(recs, out)}
    for name in ("no_rg", "unknown_rg", "qual_star", "lseq0", "fwd3", "rev3"):
        assert by[name][0] == by[name][1], name                                          # unchanged, byte for byte
    for name in ("fwd0", "rev1", "second2", "softclip", "flag_4", "flag_400", "flag_100", "len500", "other_tags", "tails"):
        assert by[name][0] != by[name][1], name                                          # recalibrated, whatever the flags
    assert err is None and recal > 20 and kept == 5 + 4 and changed > 1000
    low = bu.fields(by["low_q"][1])["qual"]
    assert all(low[k] == k % 9 for k in range(64) if k % 9 < 6)                             # q < 6 stays
    assert all(q <= 93 for r in out for q in bu.fields(r)["qual"] if q != 0xFF)
    # the same records with the read groups' tables swapped: different qualities
    assert aq.apply_all(recs, ids, [1, 0, 2, -1], tabs)[0] != out


def test_read_errors_are_named(emul, ref):
    rng = np.random.default_rng(64)
    tabs = _tabs_for(rng, ["g"])
    ok = aq.with_tags(bq.make_rec("ok", 0, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 50), aq.rg_tag("g"))
    long_ = aq.with_tags(bq.make_rec("long", 0, 0, 100, [(501, 0)], ref.seq(0, 100, 501), [30] * 501), aq.rg_tag("g"))
    hiq = aq.with_tags(bq.make_rec("hiq", 16, 0, 100, [(50, 0)], ref.seq(0, 100, 50), [30] * 49 + [94]), aq.rg_tag("g"))
    long_norg = bq.make_rec("long_norg", 0, 0, 100, [(501, 0)], ref.seq(0, 100, 501), [30] * 501)
    for recs, want in (([ok, long_, hiq], (1, 1)), ([ok, hiq, ok], (1, 2)), ([long_norg, ok], None)):
        got = aq.emul_apply(emul, recs, ["g"], [0], tabs)
        assert got == aq.apply_all(recs, ["g"], [0], tabs) and got[1] == want


def test_random_records_equal_python(emul, ref):
    rng = np.random.default_rng(65)
    tabs = _tabs_for(rng, ["x.1", "x.2"])
    ids, tab = ["r1", "r2", "r3"], [0, 1, 0]
    recs = aq.random_records(ref, rng, 3000, ids)
    got = aq.emul_apply(emul, recs, ids, tab, tabs)
    assert got == aq.apply_all(recs, ids, tab, tabs)
    assert got[2] > 2000 and got[4] > 50_000


# ---- the window reader ----

def _bgzf(data: bytes, member: int, eof=True) -> bytes:
    out = b""
    for at in range(0, len(data), member):
        chunk = data[at:at + member]
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        body = c.compress(chunk) + c.flush()
        out += b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(body) + 25) + body + \
            struct.pack("<II", zlib.crc32(chunk), len(chunk))
    return out + (bu.EOF_BLOCK if eof else b"")


def _bam_raw(text, recs):
    h = b"BAM\x01" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", 1) + struct.pack("<i", 3) + b"c0\0" + struct.pack("<i", 10**6)
    return h, b"".join(recs)


def test_window_reader(emul, ref, tmp_path):
    rng = np.random.default_rng(66)
    recs = aq.random_records(ref, rng, 600, ["a"])
    text = "@HD\tVN:1.6\tSO:coordinate\n@RG\tID:a\n"
    h, body = _bam_raw(text, recs)
    for member in (777, 65280):
        p = tmp_path / ("m%d.bam" % member)
        p.write_bytes(_bgzf(h + body, member))
        for window, threads in ((1, 1), (1000, 3), (4096, 2), (65536, 4), (1 << 30, 1)):
            t, got, nw, warn = aq.emul_read(emul, str(p), window, threads)
            assert (t, got, warn) == (text, body, "") and nw >= 1
            if window <= 4096 and member == 777:
                assert nw > 10
    full = _bgzf(h + body, 5000)
    (tmp_path / "noeof.bam").write_bytes(full[:-len(bu.EOF_BLOCK)])
    t, got, nw, warn = aq.emul_read(emul, str(tmp_path / "noeof.bam"), 4096)
    assert got == body and "no BGZF EOF block" in warn
    cases = {"trunc_member.bam": (full[:len(full) // 2], "a truncated BGZF member"),
             "trunc_record.bam": (_bgzf(h + body[:-10], 5000), "the input ends inside record 599"),
             "plain_gzip.bam": (zlib.compress(h + body), "not BGZF"),
             "not_bam.bam": (_bgzf(b"SAM\x01" + body, 5000), "not BAM"),
             "bad_crc.bam": (full[:40] + bytes([full[40] ^ 0xFF]) + full[41:], "does not inflate")}
    for name, (data, msg) in cases.items():
        (tmp_path / name).write_bytes(data)
        with pytest.raises(ValueError) as e:
            aq.emul_read(emul, str(tmp_path / name), 4096)
        assert msg in str(e.value) and name in str(e.value), (name, str(e.value))


def _run(args):
    return subprocess.run([aq.TOOL] + args, capture_output=True, timeout=120)


@pytest.mark.skipif(not os.path.exists(aq.TOOL), reason="bm2_applybqsr not built")
def test_option_errors(tmp_path):
    for args, msg in (([], "no input BAM"), (["x.bam"], "--bqsr-recal-file is required"), (["--bqsr-recal-file", "t.txt", "--write-index", "x.bam"],
                                                                                              "--write-index needs -o"),
                      (["--window", "12Q", "x.bam"], "--window takes a size"), (["-t", "0", "x.bam"], "-t takes a number"),
                      (["--bogus", "x.bam"], "unknown option --bogus"), (["--bqsr-recal-file", str(tmp_path / "none.txt"), "x.bam"], "cannot open")):
        r = _run(args)
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr)
    (tmp_path / "t.txt").write_text(aq.gatk_table(np.random.default_rng(1), ["g"], args={"maximum_cycle_value": "400"}))
    r = _run(["--bqsr-recal-file", str(tmp_path / "t.txt"), "-o", str(tmp_path / "o.bam"), "x.bam"])
    assert r.returncode == 1 and "maximum_cycle_value is 400" in r.stderr.decode() and not os.path.exists(tmp_path / "o.bam")

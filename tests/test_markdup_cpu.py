"""bm2_mem --markdup without a GPU: the per-template entries of markdup_device.cuh equal the rule restated in Python (tests/markdup_util.py)
on crafted records, resolve equals Python on random entries with many ties and piles, and bam_sort.h's duplicate path driven by the host
emulation tests/host_emul/markdup_emul.cpp gives the same output at every signature budget and record-run budget: the records of the
unmarked sort with Python's flags, no other byte changed, and no temporary file left.  Plus --markdup's options and --dump-opt field."""
import json, os, subprocess
import numpy as np
import pytest
import bam_util as bu
import bam_sort_util as bs
import markdup_util as mu
import test_bam_sort_cpu as tsc

TOOL = tsc.TOOL
IDX = tsc.IDX


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mu.build_emul(tmp_path_factory)


def crafted_templates():
    """Clips on both strands, a leading clip at position 0, CG:B,I, QUAL '*', secondary and supplementary records, mate unmapped, both
    unmapped, mates on different contigs, and a single-end read."""
    m = bs.make_rec
    return [
        (0, [mu.with_qual(m(0, 100, 0x41, cigar=((5, 4), (40, 0), (3, 5)), name=b"a"), 30),
             mu.with_qual(m(0, 300, 0x91, cigar=((2, 5), (40, 0), (6, 4)), name=b"a"), 14)]),
        (2, [mu.with_qual(m(0, 0, 0x41, cigar=((9, 4), (30, 0)), name=b"b"), 20),
             mu.with_qual(m(1, 70, 0xB1, cigar=((4, 5), (30, 0), (5, 4)), name=b"b"), None)]),
        (4, [mu.with_qual(m(2, 50, 0x49, cigar=((50, 0),), name=b"c"), 15),
             mu.with_qual(m(2, 50, 0x85, name=b"c", l_seq=50), 30)]),
        (6, [mu.with_qual(m(-1, -1, 0x4D, name=b"d", l_seq=30), 30), mu.with_qual(m(-1, -1, 0x8D, name=b"d", l_seq=30), 30)]),
        (8, [mu.with_qual(m(1, 500, 0x61, cg=[(7, 4)] + [(1, 0), (1, 1)] * 40000 + [(5, 5)], name=b"e"), None),
             mu.with_qual(m(1, 900, 0x841, cigar=((20, 5), (30, 0)), name=b"e"), 30),
             mu.with_qual(m(1, 800, 0x91, cigar=((30, 0),), name=b"e"), 40),
             mu.with_qual(m(0, 10, 0x191, cigar=((30, 0),), name=b"e"), 40)]),
        (10, [mu.with_qual(m(0, 5, 0x10, cigar=((3, 4), (20, 0), (2, 5)), name=b"f"), 128)]),
        (11, [mu.with_qual(m(2, 1, 0x51, cg=[(3, 5), (2, 4)] + [(1, 0), (1, 2)] * 33000 + [(4, 4), (1, 5)], name=b"g"), 41),
              mu.with_qual(m(2, 9, 0xA1, cigar=((3, 5), (10, 0), (2, 4)), name=b"g"), 41)]),
    ]


def python_entries(templates):
    pe, fe = [], []
    for tid, recs in templates:
        p, f = mu.template_entries([bu.fields(r) for r in recs], tid)
        pe += p; fe += f
    return mu.entries_array(pe), mu.entries_array(fe)


@pytest.mark.parametrize("which", ["crafted", "random_pe", "random_se"])
def test_entries_equal_python(emul, which):
    rng = np.random.default_rng(11)
    t = {"crafted": crafted_templates, "random_pe": lambda: mu.random_templates(rng, 600), "random_se": lambda: mu.random_templates(rng, 600, paired=False)}[which]()
    data, first, ids = mu.flatten(t)
    got_p, got_f = mu.emul_signatures(emul, data, first, ids)
    want_p, want_f = python_entries(t)
    assert got_p.tobytes() == want_p.tobytes() and got_f.tobytes() == want_f.tobytes()
    if which == "crafted":
        ends = {e["tid"]: e for e in want_p}
        assert ends[0]["score"] == 45 * 30 and mu.end_key((0, 95, 0)) == ends[0]["k1"] and mu.end_key((0, 300 + 40 - 1 + 6, 1)) == ends[0]["k2"]
        fr = {}
        for e in want_f:                                                            # a pair's first pair end
            fr.setdefault((int(e["tid"]), int(e["kind"])), e)
        assert fr[(2, mu.PAIR_END)]["k1"] == mu.end_key((0, -9, 0))                # a position-0 read with a leading clip: a negative coordinate
        assert fr[(4, mu.FRAG)]["score"] == 50 * 15                                 # mate unmapped: a fragment
        assert not any(e["tid"] == 6 for e in want_f)                              # both unmapped: no entry
        assert fr[(8, mu.PAIR_END)]["k1"] == mu.end_key((1, 500 - 7, 0)) and ends[8]["score"] == 30 * 40   # CG:B,I and QUAL '*'
        assert fr[(10, mu.FRAG)]["k1"] == mu.end_key((0, 5 + 20 - 1 + 2, 1))
        assert ends[11]["score"] == 16383 + 12 * 41                               # the read score's cap


def test_resolve_equals_python(emul):
    rng = np.random.default_rng(5)
    for space in (mu.PAIR, mu.FRAG):
        for n in (1, 7, 500, 4000):
            e = mu.random_entries(rng, n, space)
            got = mu.emul_resolve(emul, mu.entries_array(e))
            assert got.tolist() == mu.resolve(e), (space, n)
            srt = mu.emul_resolve(emul, mu.entries_array(e), False)
            assert [tuple(x) for x in srt.tolist()] == sorted(e, key=lambda x: (x[0], x[1], -x[3], x[2]))
    # a pair end meets fragments: every fragment of its group is a duplicate, the pair end is not
    k = mu.end_key((0, 10, 0))
    e = [(k, 0, 5, 9000, mu.FRAG), (k, 0, 3, 10, mu.PAIR_END), (k, 0, 1, 9000, mu.FRAG), (k + 2, 0, 7, 1, mu.FRAG), (k + 2, 0, 6, 1, mu.FRAG)]
    assert sorted(mu.emul_resolve(emul, mu.entries_array(e)).tolist()) == [1, 5, 7] == sorted(mu.resolve(e))


def _decoded(path):
    return [r for _, r in bu.records(bu.inflate(open(path, "rb").read()))]


def _expected(templates):
    tid_of = {}
    for tid, recs in templates:
        for r in recs:
            tid_of[r] = tid
    pd, fd, n = mu.duplicates([(tid, [bu.fields(r) for r in recs]) for tid, recs in templates])
    srt = tsc.stable_sorted(b"".join(r for _, recs in templates for r in recs))
    return srt, mu.apply_flags(srt, lambda r: tid_of[r], set(pd) | set(fd)), pd, fd, n


@pytest.mark.parametrize("paired", [True, False])
def test_driver_flags_at_every_budget(emul, tmp_path, paired):
    rng = np.random.default_rng(3 if paired else 4)
    t = mu.random_templates(rng, 1500, paired=paired, piles=25)
    unmarked, want, pd, fd, n = _expected(t)
    assert len(pd) + len(fd) > 100 and sum(bu.fields(r)["flag"] & 0x400 != 0 for r in want) > 100
    data = b"".join(r for _, recs in t for r in recs)
    outs = set()
    for step, (run_bytes, sig_bytes) in enumerate(((1 << 40, 1 << 40), (1 << 40, 20_000), (len(data) // 5, 3 * 32), (40_000, 1), (len(data) // 3, 64_000))):
        d = tmp_path / ("b%d" % step); d.mkdir()
        out = str(d / "out.bam")
        st = mu.emul_file(emul, t, run_bytes, sig_bytes, str(d / "out.bam.tmp."), out, chunk_tmpl=37)
        assert os.listdir(d) == ["out.bam"]                                   # no temporary file survives
        got = _decoded(out)
        assert got == want, step
        assert all(a[:18] + a[20:] == b[:18] + b[20:] for a, b in zip(got, unmarked))   # only the flag differs
        assert (st["pair_dups"], st["frag_dups"], st["templates"]) == (len(pd), len(fd), n)
        assert st["records"] == sum(bu.fields(r)["flag"] & 0x400 != 0 for r in want)
        if sig_bytes >= 1 << 40:
            assert st["sig_runs"] == 0 and st["sig_bytes"] == 0
        else:
            assert st["sig_runs"] >= 2 and st["sig_bytes"] > 0
        if run_bytes < len(data):
            assert st["runs"] >= 3 and st["spill_bytes"] > 0
        outs.add(open(out, "rb").read())
    assert len(outs) == 1                                                      # the same bytes at every budget


def test_no_duplicates_changes_nothing(emul, tmp_path):
    t = [(2 * k, [bs.make_rec(k % 3, 1000 * k, 0x41 | (0x10 if k % 2 else 0), name=b"u%d" % k),
                  bs.make_rec(k % 3, 1000 * k + 300, 0x81 | (0x10 if k % 2 == 0 else 0), name=b"u%d" % k)]) for k in range(800)]
    out = str(tmp_path / "o.bam")
    st = mu.emul_file(emul, t, 1 << 40, 1 << 40, str(tmp_path / "o.tmp."), out)
    assert st["pair_dups"] == st["frag_dups"] == st["records"] == 0 and st["templates"] == 800
    srt = tsc.stable_sorted(b"".join(r for _, recs in t for r in recs))
    assert _decoded(out) == srt


def _dump(*args):
    return subprocess.run([TOOL, "--dump-opt"] + list(args) + [IDX, "a.fq", "b.fq"], capture_output=True, text=True, timeout=60)


@pytest.mark.skipif(not os.path.exists(TOOL), reason="bm2_mem not built")
def test_markdup_options_and_dump_opt():
    j0 = json.loads(_dump("--sort").stdout)
    assert "markdup" not in j0
    j = json.loads(_dump("--markdup", "--sort-mem", "64M", "--write-index", "-o", "x.bam").stdout)
    assert j["markdup"] is True and j["sort"] is True and j["bam"] is True and j["sort_mem"] == 64 << 20 and j["write_index"] is True
    assert j["header"].split("\n")[0] == "@HD\tVN:1.6\tSO:coordinate"
    assert json.loads(_dump("--markdup", "-p", "-a", "-M", "-5").stdout)["markdup"] is True
    r = subprocess.run([TOOL], capture_output=True, text=True)
    assert "--markdup" in r.stderr

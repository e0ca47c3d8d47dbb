"""bm2_mem --markdup-metrics without a GPU: the QNAME location parser of markdup_device.cuh equals Picard's rapidParseInt restated in Python,
the optical pass of the host emulation (tests/host_emul/markdup_metrics_emul.cpp: the warp path of groups up to 32 and the exact cell pass
of larger ones) equals a breadth-first search over the link relation, the located signatures and resolve equal the rule in Python, and the
library size, histogram and file text of markdup_metrics.h equal Picard's formulas restated in Python.  Plus the options, --dump-opt and the
start-up errors."""
import json, os, struct, subprocess
import numpy as np
import pytest
import bam_util as bu
import markdup_util as mu
import markdup_metrics_util as mm
import test_bam_sort_cpu as tsc

TOOL = tsc.TOOL
IDX = tsc.IDX


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mm.build_emul(tmp_path_factory)


NAMES = [b"a:b:1:2:3", b"inst:1:1101:100:200", b"M01:77:FC:1:1101:15589:1337", b"a:1:2:3", b"a:b:c:1:2:3", b"a:b:c:d:e:1:2:3",
         b"x::1:2:3", b"x:1::2:3", b"x:1:2:3:", b"x:1:-:2:3", b"x:1:-12:-7:-0", b"x:1:123abc:4x:5.5", b"x:1:abc:2:3", b"x:1:1:2:abc",
         b"x:1:2147483647:2147483648:4294967297", b"x:1:99999999999:-2147483649:-99999999999", b"x:1:0012:0:-",
         b"M01:77:FC:1:1101:15589:1337 1:N:0:ATCACG", b"", b":", b"::::", b"::::::", b"a:b:c:d:e:f:g:h:1", b"SRR1.1", b"x:1:+5:6:7",
         b"x:1:1101:2:3\t"]


def test_name_parser_equals_python(emul):
    for n in NAMES:
        assert mm.emul_location(emul, n) == mm.location(n), n
    assert mm.location(b"M01:77:FC:1:1101:15589:1337") == (1101, 15589, 1337)
    assert mm.location(b"inst:1:1101:100:200") == (1101, 100, 200)
    assert mm.location(b"x:1:123abc:4x:5.5") == (123, 4, 5)
    assert mm.location(b"x:1:-12:-7:-0") == (-12, -7, 0)
    assert mm.location(b"x:1:2147483647:2147483648:4294967297") == (2147483647, -2147483648, 1)    # Java int wrap
    for n in (b"a:1:2:3", b"a:b:c:1:2:3", b"a:b:c:d:e:1:2:3", b"x:1:-:2:3", b"x:1:abc:2:3", b"x:1::2:3", b"x:1:2:3:"):
        assert mm.location(n) is None, n
    rng = np.random.default_rng(7)
    alphabet = b"0123456789-:a "
    for _ in range(3000):
        n = bytes(alphabet[int(i)] for i in rng.integers(0, len(alphabet), int(rng.integers(0, 30))))
        assert mm.emul_location(emul, n) == mm.location(n), n


def _spots(rng, n, d, k):
    """n members in k tight clusters far apart on one tile: k components."""
    c = [(int(rng.integers(0, 1000)) * (5 * d + 10), int(rng.integers(0, 1000)) * (5 * d + 10)) for _ in range(k)]
    c = list(dict.fromkeys(c))
    out = []
    for i in range(n):
        x, y = c[i % len(c)]
        out.append((mm.HAS, 1101, x + int(rng.integers(0, d + 1)), y + int(rng.integers(0, d + 1))))
    return out, len(c)


def test_optical_equals_bfs(emul):
    rng = np.random.default_rng(17)
    for d in (0, 1, 100, 2500):
        for n in (2, 3, 5, 17, 31, 32, 33, 40, 100, 500, 2000):
            for _ in range(3 if n <= 100 else 1):
                g = mm.random_group(rng, n, d, spread=int(rng.choice([d + 2, 3 * d + 3, 10 * d + 10])))
                assert mm.emul_optical(emul, g, d) == mm.optical_count(g, d), (d, n)
    for d in (0, 100):                                                  # chains: A~B and B~C but not A~C is one component
        for n in (3, 20, 40, 300):
            g = [(mm.HAS, 7, k * d + (1 if d == 0 else 0) * k, 5 * (k % 2)) for k in range(n)]
            want = n - 1 if d else 0
            assert mm.optical_count(g, d) == want and mm.emul_optical(emul, g, d) == want
            diag = [(mm.HAS, 7, k * (d or 1), k * (d or 1)) for k in range(n)]       # a diagonal chain crosses cells corner to corner
            assert mm.emul_optical(emul, diag, d) == mm.optical_count(diag, d) == (n - 1 if d else 0)
    for n in (10, 64):                                                  # both classes at the same spot are counted apart; no location is alone
        g = [(mm.HAS | (k % 2) * mm.REV, 1, 50, 50) for k in range(n)] + [(0, 0, 0, 0)] * 3
        assert mm.emul_optical(emul, g, 100) == mm.optical_count(g, 100) == n - 2
        g = [(mm.HAS, 1 + k % 3, 50, 50) for k in range(n)]            # tiles apart
        assert mm.emul_optical(emul, g, 100) == n - 3
    g = [(mm.HAS, 1, 10, 10)] * 5 + [(mm.HAS, 1, 11, 10)]              # N = 0: identical coordinates only
    assert mm.emul_optical(emul, g, 0) == mm.optical_count(g, 0) == 4
    assert mm.emul_optical(emul, [(0, 0, 0, 0)] * 40, 100) == 0
    big, k = _spots(rng, 300_000, 100, 500)                             # the largest counted group, and one more member: none
    assert mm.emul_optical(emul, big, 100) == 300_000 - k
    assert mm.emul_optical(emul, big + [(mm.HAS, 1101, 0, 0)], 100) == 0
    dense = [(mm.HAS | mm.REV * (k % 2), 2202, 1000 + k % 7, 2000 + k % 11) for k in range(50_000)]   # a deep pile at one spot
    assert mm.emul_optical(emul, dense, 100) == 50_000 - 2
    sub = dense[:3000]
    assert mm.emul_optical(emul, sub, 3) == mm.optical_count(sub, 3)


def with_name(rec, name):
    """A BAM record with its QNAME replaced."""
    lrn = rec[12]
    body = rec[4:12] + bytes([len(name) + 1]) + rec[13:36] + name + b"\0" + rec[36 + lrn:]
    return struct.pack("<i", len(body)) + body


def located_templates(rng, n, paired=True):
    t = mu.random_templates(rng, n, paired=paired, piles=20)
    out = []
    for tid, recs in t:
        kind = int(rng.integers(0, 4))
        nm = mm.illumina_name(1101 + int(rng.integers(0, 2)), int(rng.integers(0, 400)), int(rng.integers(0, 400))).encode() if kind else \
            (b"noloc%d" % tid)
        out.append((tid, [with_name(r, nm) for r in recs]))
    return out


def test_signatures_and_resolve_equal_python(emul):
    rng = np.random.default_rng(23)
    for paired in (True, False):
        t = located_templates(rng, 1500, paired)
        data, first, ids = mu.flatten(t)
        p, f, counts = mm.emul_signatures_ex(emul, data, first, ids)
        pe, fe = [], []
        for tid, recs in t:
            a, b = mu.template_entries([bu.fields(r) for r in recs], tid)
            pe += a; fe += b
        assert [tuple(x)[:5] for x in p.tolist()] == pe and f.tobytes() == mu.entries_array(fe).tobytes()
        fs = [(tid, [bu.fields(r) for r in recs]) for tid, recs in t]
        assert counts == (sum((x["flag"] & 0x900) != 0 for _, r in fs for x in r),
                          sum((x["flag"] & 0x900) == 0 and (x["flag"] & 4) != 0 for _, r in fs for x in r))
        for d in (0, 100, 2500):
            want = mm.metrics_of(fs, d)
            dups, opt = mm.emul_resolve_ex(emul, p, d)
            assert sorted(dups.tolist()) == sorted(mu.resolve(pe)) and opt == want["optical"]
            assert (len(p), len(mu.resolve(pe))) == (want["pairs"], want["pair_dups"])
            if paired and d >= 100:
                assert want["optical"] > 0 and len(pe) > 0
        srt = mm.emul_resolve_ex(emul, p, 100, False)
        assert [tuple(x)[:5] for x in srt.tolist()] == sorted(pe, key=lambda x: (x[0], x[1], -x[3], x[2]))
    e = mm.located_entries(rng, 20_000, 300, 100)                       # larger groups through the cell pass
    dups, opt = mm.emul_resolve_ex(emul, e, 100)
    groups = {}
    for x in e.tolist():
        groups.setdefault((x[0], x[1]), []).append((x[8], x[5], x[6], x[7]))
    assert opt == sum(mm.optical_count(g, 100) for g in groups.values()) and max(len(g) for g in groups.values()) > 32


def _m(**kw):
    m = dict(unpaired=0, pairs=0, secsup=0, unmapped=0, unpaired_dups=0, pair_dups=0, optical=0)
    m.update(kw)
    return m


def test_metrics_text_equals_python(emul):
    cases = [_m(unpaired=40, pairs=1000, secsup=7, unmapped=3, unpaired_dups=5, pair_dups=120, optical=30),
             _m(pairs=1000, pair_dups=0),                                     # no duplicates: no library size, no histogram
             _m(pairs=500, pair_dups=80, optical=80),                         # all optical: no library size
             _m(unpaired=300, unpaired_dups=40, unmapped=9),                  # single-end only: no pairs, no histogram
             _m(),                                                            # nothing examined: PERCENT_DUPLICATION 0
             _m(pairs=10_000_000, pair_dups=1, optical=0), _m(pairs=7, pair_dups=6), _m(pairs=3_000_000, pair_dups=2_000_000, optical=12345)]
    for k, m in enumerate(cases):
        for lib in ("Unknown Library", "lib-1"):
            args = "--markdup-metrics m.txt -o x.bam idx r1.fq r2.fq"
            assert mm.emul_metrics_text(emul, m, args, lib) == mm.metrics_text(m, args, lib), (k, m)
        L = mm.library_size(m["pairs"] - m["optical"], m["pairs"] - m["pair_dups"])
        assert emul.mm_library_size(m["pairs"] - m["optical"], m["pairs"] - m["pair_dups"]) == (-1 if L is None else L)
        row, hist = mm.parse_metrics(mm.metrics_text(m, ""))
        assert (row["ESTIMATED_LIBRARY_SIZE"] == "") == (L is None) and len(hist) == (0 if L is None else 100)
    row, hist = mm.parse_metrics(mm.metrics_text(cases[0], ""))
    assert row["PERCENT_DUPLICATION"] == mm.fmt((5 + 240) / 2040) and hist[0].startswith("1.0\t") and hist[-1].startswith("100.0\t")
    assert mm.parse_metrics(mm.metrics_text(cases[4], ""))[0]["PERCENT_DUPLICATION"] == "0"
    assert int(row["ESTIMATED_LIBRARY_SIZE"]) > 1000 - 120
    assert mm.fmt(1.0) == "1" and mm.fmt(0.5) == "0.5" and mm.fmt(0.0000004) == "0" and mm.fmt(2.25e-5) == "0.000023"


def _dump(*args):
    return subprocess.run([TOOL, "--dump-opt"] + list(args) + [IDX, "a.fq", "b.fq"], capture_output=True, text=True, timeout=60)


@pytest.mark.skipif(not os.path.exists(TOOL), reason="bm2_mem not built")
def test_options_dump_opt_and_errors():
    j0 = json.loads(_dump("--markdup").stdout)
    assert "markdup_metrics" not in j0 and "optical_distance" not in j0
    j = json.loads(_dump("--markdup-metrics", "m.txt").stdout)
    assert j["markdup_metrics"] == "m.txt" and j["optical_distance"] == 100 and j["markdup"] and j["sort"] and j["bam"]
    j = json.loads(_dump("--markdup-metrics", "m.txt", "--optical-distance", "2500", "-o", "x.bam", "--write-index").stdout)
    assert j["optical_distance"] == 2500 and j["write_index"] is True
    assert json.loads(_dump("--optical-distance", "0", "--markdup-metrics", "q").stdout)["optical_distance"] == 0
    assert json.loads(_dump("--markdup-metrics", "q", "--optical-distance", "2147483647").stdout)["optical_distance"] == 2147483647
    for bad in (["--optical-distance", "100"], ["--markdup", "--optical-distance", "5"], ["--markdup-metrics", "q", "--optical-distance", "-1"],
                ["--markdup-metrics", "q", "--optical-distance", "2147483648"], ["--markdup-metrics", "q", "--optical-distance", "1e3"],
                ["--markdup-metrics", "q", "--optical-distance", ""], ["--markdup-metrics", "q", "--optical-distance"]):
        r = _dump(*bad)
        assert r.returncode == 1 and "[E::bm2_mem]" in r.stderr and not r.stdout, bad
    r = subprocess.run([TOOL], capture_output=True, text=True)
    assert "--markdup-metrics" in r.stderr and "--optical-distance" in r.stderr

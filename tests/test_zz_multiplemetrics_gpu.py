"""bm2_multiplemetrics on the GPU: bm2_mm_set / bm2_mm_add / bm2_mm_finish give the files of the host emulation
(tests/host_emul/multiplemetrics_emul.cpp) on crafted and random records at several window sizes, and a window holding a bad record raises
the named error and counts nothing; `bm2_multiplemetrics` writes the two files Python computes (Picard's loops,
tests/multiplemetrics_util.py) from the unsorted BAM of `bm2_mem --bam` (paired, single-end, smart pairing), from the sorted BAM of
`bm2_mem --markdup` and from the BAM of `bm2_applybqsr`, against an index built by bm2_index from a FASTA with N, n and IUPAC runs; the
bytes do not depend on -t, --window or standard input; the error cases exit 1 and leave neither file."""
import json, os, subprocess
import numpy as np
import pytest
import bam_util as bu
import bqsr_util as bq
import markdup_util as mdu
import multiplemetrics_util as mu
import test_multiplemetrics_cpu as tc
import test_zz_markdup_gpu as tmg
import test_zz_wgsmetrics_gpu as twg

pytestmark = pytest.mark.gpu

TOOL = mu.TOOL
ROOT = mu.ROOT
MEM = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
INDEX = os.path.join(ROOT, "bwa-mem2_b200", "bm2_index")
APPLY = os.path.join(ROOT, "bwa-mem2_b200", "bm2_applybqsr")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return mu.build_emul(tmp_path_factory)


def _set(ctx, ref):
    hb, hc = mu.hole_arrays(ref)
    ctx.mm_set(ref.off, ref.lens, ref.l_pac, mu.pac_bytes(ref), hb[:2 * len(ref.holes)], hc)


def _device(ctx, ref, wins):
    _set(ctx, ref)
    for w in wins:
        ctx.mm_add(*bq.flatten(w))
    d = ctx.mm_finish()
    cats, ins = mu.from_device(d)
    return mu.summary_text(cats, "a"), mu.insert_text(ins, "a"), d


def test_kernels_equal_emulation(gpu_ctx, emul):
    rng = np.random.default_rng(111)
    ref = tc.REF
    for recs in (tc.crafted(), mu.random_records(ref, rng, 2000), []):
        for sizes in ([max(len(recs), 1)], [1], [7], [333]):
            wins = mu.windows(recs, sizes)
            want = mu.emul_run(emul, ref, wins, "a")
            got = _device(gpu_ctx, ref, wins)
            assert want[4] is None and got[:2] == want[:2], sizes
            assert np.array_equal(got[2]["counts"], want[2]) and got[2]["records"] == len(recs)
            assert got[2]["add_ms"] >= 0 and got[2]["finish_ms"] >= 0
        if recs:
            assert got[:2] == mu.files(recs, ref, "a")
    assert len(_device(gpu_ctx, ref, [tc.crafted()])[2]["insert_big"]) == 2
    ok = mu.rec("ok", 0, 0, 100, [(10, 0)])
    for bad, msg in ((mu.rec("lseq0", 0, 0, 200, [(10, 2)], [], seq=""), "read lseq0 (record 3) has l_seq 0 or above 1048576"),
                     (mu.rec("past", 0, 0, 2995, [(10, 0)]), "read past (record 3) does not lie inside a contig"),
                     (mu.rec("badcig", 0, 0, 200, [(10, 0), (2, 1)], seq="A" * 10), "read badcig (record 3) has a CIGAR")):
        wins = [[ok, ok], [ok, bad, ok]]
        assert msg in mu.emul_run(emul, ref, wins)[4]
        _set(gpu_ctx, ref)
        gpu_ctx.mm_add(*bq.flatten(wins[0]))
        with pytest.raises(Exception, match=msg.replace("(", r"\(").replace(")", r"\)")):
            gpu_ctx.mm_add(*bq.flatten(wins[1]))
        got = gpu_ctx.mm_finish()                                                       # nothing of the failed window was counted
        assert got["records"] == 2 and np.array_equal(got["counts"], _device(gpu_ctx, ref, [wins[0]])[2]["counts"])


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    for t in (TOOL, MEM, INDEX, APPLY):
        if not os.path.exists(t):
            pytest.skip(os.path.basename(t) + " not built")
    d = tmp_path_factory.mktemp("mm_gpu")
    rng = np.random.default_rng(112)
    (d / "ref.fa").write_text(twg._genome(rng))
    subprocess.run([INDEX, str(d / "ref.fa")], check=True, capture_output=True, timeout=900)
    prefix = str(d / "ref.fa")
    ref = mu.Ref.read(prefix)
    assert {c for _, _, c in ref.holes} >= {"N", "n", "R"}
    pairs = mdu.planted_pairs(mdu.load_reference(prefix), rng, n_base=400)
    files, _ = tmg._write_pairs(d, pairs, "p")
    bams = {}
    for mode in ("pe", "se", "smart"):
        for kind in ("--bam", "--markdup"):
            out = str(d / ("%s_%s.bam" % (kind[2:], mode)))
            r = subprocess.run([MEM, kind, "-R", r"@RG\tID:g1\tSM:s", prefix] + files[mode] + (["-p"] if mode == "smart" else []) + ["-o", out],
                               capture_output=True, timeout=900)
            assert r.returncode == 0, r.stderr[-2000:]
            bams[kind[2:] + "_" + mode] = out
    return d, prefix, ref, files, bams


def _tool(args, stdin=None):
    r = subprocess.run([TOOL] + args, capture_output=True, timeout=900, stdin=stdin)
    assert r.returncode == 0, r.stderr[-3000:]
    return r, json.loads(r.stderr.decode().strip().split("\n")[-1])


def _want(bam, ref, args):
    raw = bu.inflate(open(bam, "rb").read())
    _, _, used = bu.parse_header(raw)
    recs = [r for _, r in bu.records(raw[used:])]
    return mu.files(recs, ref, " ".join(args)), len(recs)


def _read(out):
    return open(out + ".alignment_summary_metrics").read(), open(out + ".insert_size_metrics").read()


@pytest.mark.parametrize("bam", ["bam_pe", "bam_se", "bam_smart", "markdup_pe"])
def test_tool_equals_python(inputs, bam):
    d, prefix, ref, files, bams = inputs
    out = str(d / ("m_" + bam))
    args = ["-o", out, prefix, bams[bam]]
    _, st = _tool(args)
    want, n = _want(bams[bam], ref, args)
    assert _read(out) == want and st["records"] == n and st["windows"] == 1
    rows = tc._rows(want[0])
    cats = [r["CATEGORY"] for r in rows]
    pairs_rows = ["FIRST_OF_PAIR", "SECOND_OF_PAIR", "PAIR"]
    assert cats == {"bam_se": ["UNPAIRED"], "bam_smart": pairs_rows + ["UNPAIRED"]}.get(bam, pairs_rows)   # smart pairing keeps lone reads
    assert all(float(r["PF_MISMATCH_RATE"]) > 0 and int(r["PF_READS_ALIGNED"]) > 0 for r in rows if r["CATEGORY"] != "UNPAIRED" or bam == "bam_se")
    assert (st["pairs"] > 0) == (bam != "bam_se") and ("## HISTOGRAM" in want[1]) == (bam != "bam_se")
    assert not [f for f in os.listdir(d) if f.endswith(".tmp")]


def test_applybqsr_bam(inputs):
    d, prefix, ref, files, bams = inputs
    bref = bq.Ref(prefix)
    (d / "s.vcf").write_text(bq.vcf_text(bref, bq.random_sites(bref, np.random.default_rng(113), every=50)))
    r = subprocess.run([MEM, "--recal-file", str(d / "t.txt"), "--known-sites", str(d / "s.vcf"), "-R", r"@RG\tID:g1\tSM:s", prefix] + files["pe"] +
                       ["-o", str(d / "rc.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([APPLY, "--bqsr-recal-file", str(d / "t.txt"), "-o", str(d / "ap.bam"), str(d / "rc.bam")], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    args = ["-o", str(d / "ap"), prefix, str(d / "ap.bam")]
    _tool(args)
    assert _read(str(d / "ap")) == _want(str(d / "ap.bam"), ref, args)[0]


@pytest.mark.parametrize("bam", ["bam_pe", "markdup_pe"])
def test_bytes_do_not_depend_on_threads_windows_or_stdin(inputs, bam):
    d, prefix, ref, files, bams = inputs
    bodies, stats = [], []
    for k, extra in enumerate((["-t", "1"], ["-t", "16"], ["-t", "16", "--window", "64K"], ["-t", "3", "--window", "100K"])):
        out = str(d / ("b%d_%s" % (k, bam)))
        stats.append(_tool(extra + ["-o", out, prefix, bams[bam]])[1])
        bodies.append(tuple(t.split("\n", 2)[2] for t in _read(out)))
    with open(bams[bam], "rb") as f:
        _, st = _tool(["-o", str(d / ("stdin_" + bam)), prefix, "-"], stdin=f)
    bodies.append(tuple(t.split("\n", 2)[2] for t in _read(str(d / ("stdin_" + bam)))))
    assert all(b == bodies[0] for b in bodies)
    assert stats[2]["windows"] > 3 and stats[0]["windows"] == 1
    assert len({(s["records"], s["aligned_bases"]) for s in stats + [st]}) == 1


def test_errors(inputs, tmp_path):
    d, prefix, ref, files, bams = inputs
    raw = bu.inflate(open(bams["bam_pe"], "rb").read())
    text, refs, used = bu.parse_header(raw)
    recs = [x for _, x in bu.records(raw[used:])]
    mapped = next(i for i, x in enumerate(recs) if not bu.fields(x)["flag"] & 0x904)
    f = bu.fields(recs[mapped])
    bad = bytearray(recs[mapped]); bad[8:12] = (ref.lens[f["rid"]] - 5).to_bytes(4, "little")
    (tmp_path / "past.bam").write_bytes(mu.bam_bytes(ref, recs[:mapped] + [bytes(bad)] + recs[mapped + 1:], text=text))
    (tmp_path / "notbam.bam").write_bytes(b"hello")
    golden = os.path.join(ROOT, "tests", "golden", "c0_index", "ref.fa")
    for args, msg in (([prefix, str(tmp_path / "past.bam")], "read %s (record %d) does not lie inside a contig" % (f["qname"], mapped)),
                      ([prefix, str(tmp_path / "notbam.bam")], ""),
                      ([golden, bams["bam_pe"]], "in the header, chr1 of length")):
        out = str(tmp_path / "e")
        r = subprocess.run([TOOL, "-o", out] + args, capture_output=True, timeout=900)
        assert r.returncode == 1 and msg in r.stderr.decode(), (args, r.stderr[-2000:])
        assert not [x for x in os.listdir(tmp_path) if x.startswith("e.")]

"""Coordinate-sorted BAM on the GPU: `bm2_mem --sort`, decoded, is the stable sort by samtools' coordinate key of `bm2_mem --bam`'s records
from the same options, and its bytes and its .bai are what the host emulation (tests/host_emul/bam_sort_emul.cpp) makes of that --bam
output - paired, single-end, smart pairing, FASTA input, -R -C -V -M -a -5, an ALT index and -x ont2d.  The same bytes at 1 and 3 chunks in
flight and with runs small enough for many temporary files and merge windows, none of which is left behind; @HD first with SO:coordinate; the
index reaches exactly the overlapping records of every region asked; and bm2_bam_sort_compress alone equals the emulation."""
import json, os, subprocess
import numpy as np
import pytest
import bam_util as bu
import bam_inputs
import bam_sort_util as bs
import test_bam_cpu as tb
import test_bam_sort_cpu as tsc
import test_zz_bam_gpu as tg

pytestmark = pytest.mark.gpu

TOOL = tg.TOOL
RG = tg.RG
inputs = tg.inputs


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return bs.build_emul(tmp_path_factory)


@pytest.fixture(scope="module")
def bgzf(tmp_path_factory):
    return tb.build_emul(tmp_path_factory)


def _run(args, out=None, env=None):
    r = subprocess.run([TOOL] + args + (["-o", out] if out else []), capture_output=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _stats(r):
    return json.loads(r.stderr.decode().strip().split("\n")[-1])


def _header_and_records(data):
    raw = bu.inflate(data)
    _, refs, used = bu.parse_header(raw)
    return raw[:used], raw[used:], len(refs)


def _emulated(emul, bgzf, tmp, sorted_data, bam_data, bai=True):
    """The sorted file and its index as the emulation makes them from the --bam file's records and the sorted file's header."""
    hdr, _, n_ref = _header_and_records(sorted_data)
    _, recs, _ = _header_and_records(bam_data)
    hz = tb.emul_stream(bgzf, hdr, [])[0]
    out, idx = str(tmp / "emul.part"), str(tmp / "emul.bai")
    bs.emul_file(emul, recs, 1 << 40, str(tmp / "emul.tmp."), out, bai_path=idx if bai else None, out_off=len(hz), n_ref=n_ref)
    return hz + open(out, "rb").read() + bu.EOF_BLOCK, (open(idx, "rb").read() if bai else None), recs


@pytest.mark.parametrize("name,args,files,idx", [
    ("pe", [], ["r1.fq", "r2.fq"], "idx"),
    ("se", [], ["r1.fq"], "idx"),
    ("smart", ["-p"], ["inter"], "idx"),
    ("fasta", [], ["a1.fa", "a2.fa"], "idx"),
    ("R_C_V_M_a_5", ["-R", RG, "-C", "-V", "-M", "-a", "-5"], ["t1.fq", "t2.fq"], "anno"),
    ("alt", [], ["r1.fq", "r2.fq"], "alt"),
    ("ont2d", ["-x", "ont2d"], ["long"], "long"),
])
def test_sort_equals_emulation_of_bam(inputs, emul, bgzf, name, args, files, idx):
    d, f = inputs
    w = d / ("sort_" + name); w.mkdir()
    prefix = str(d / "long" / "ref.fa") if idx == "long" else str(d / idx / "ref.fa")
    common = args + ["-K", "40000", prefix] + [f[x] for x in files]
    _run(["--bam"] + common, str(w / "plain.bam"))
    r = _run(["--sort", "--write-index"] + common, str(w / "out.bam"))
    assert sorted(os.listdir(w)) == ["out.bam", "out.bam.bai", "plain.bam"]           # no temporary file left
    got, bam = open(w / "out.bam", "rb").read(), open(w / "plain.bam", "rb").read()
    text, _, lines, _ = bu.read_bam_file(got)
    assert text.split("\n")[0] == "@HD\tVN:1.6\tSO:coordinate" and got.endswith(bu.EOF_BLOCK)
    want_z, want_bai, recs = _emulated(emul, bgzf, w, got, bam)
    _, srt, _ = _header_and_records(got)
    assert [r for _, r in bu.records(srt)] == tsc.stable_sorted(recs)
    assert got == want_z and open(w / "out.bam.bai", "rb").read() == want_bai
    st = _stats(r)
    assert st["sort_runs"] == 1 and st["spill_bytes"] == 0 and st["sort_s"] > 0 and "index_s" in st and "merge_windows" in st


def test_sort_bytes_do_not_depend_on_workers_or_runs(inputs, emul, bgzf):
    d, f = inputs
    w = d / "runs"; w.mkdir()
    big = d / "big"; big.mkdir()                                          # six copies of the pairs: enough BGZF blocks per run for many windows
    for m in (1, 2):
        (big / ("r%d.fq" % m)).write_bytes(open(f["r%d.fq" % m], "rb").read() * 6)
    common = ["-K", "300000", str(d / "idx" / "ref.fa"), str(big / "r1.fq"), str(big / "r2.fq")]
    _run(["--bam"] + common, str(w / "plain.bam"))
    parts, stats = [], []
    for k, extra in enumerate((["-p", "1"], ["-p", "3"], ["-p", "2", "--sort-mem", "350K"])):
        r = _run(["--sort", "--write-index"] + extra + common, str(w / ("s%d.bam" % k)))
        stats.append(_stats(r))
        data = open(w / ("s%d.bam" % k), "rb").read()
        parts.append((tg._records_part(data), open(w / ("s%d.bam.bai" % k), "rb").read()))
    assert sorted(os.listdir(w)) == ["plain.bam"] + sorted("s%d.bam%s" % (k, x) for k in range(3) for x in ("", ".bai"))   # no temporary file left
    assert parts[0][0] == parts[1][0] == parts[2][0]                     # the records' members (the @PG line differs, and so the BAI's offsets)
    assert stats[2]["sort_runs"] >= 5 and stats[2]["merge_windows"] >= 5 and stats[2]["spill_bytes"] > 0 and stats[2]["merge_s"] > 0
    for k in range(3):
        got = open(w / ("s%d.bam" % k), "rb").read()
        e = w / ("e%d" % k); e.mkdir()
        want_z, want_bai, _ = _emulated(emul, bgzf, e, got, open(w / "plain.bam", "rb").read())
        assert got == want_z and parts[k][1] == want_bai, k
    tsc.check_index(str(w / "s2.bam"), str(w / "s2.bam.bai"), len(got) - len(tg._records_part(got)), 4, np.random.default_rng(3))


def test_sort_to_stdout_uses_tmpdir_and_keeps_hd_fields(inputs, tmp_path):
    d, f = inputs
    tmp = tmp_path / "tmpdir"; tmp.mkdir()
    env = dict(os.environ, TMPDIR=str(tmp))
    r = _run(["--sort", "--sort-mem", "50K", "-H", "@HD\tVN:1.5\tSO:queryname\tGO:none", "-K", "30000", str(d / "idx" / "ref.fa"), f["r1.fq"],
              f["r2.fq"]], env=env)
    assert os.listdir(tmp) == [] and _stats(r)["sort_runs"] >= 5
    text, _, lines, _ = bu.read_bam_file(r.stdout)
    h = text.split("\n")
    assert h[0] == "@HD\tVN:1.5\tSO:coordinate\tGO:none" and sum(l.startswith("@HD") for l in h) == 1
    keys = [bs.key(bu.fields(rec)) for _, rec in bu.records(_header_and_records(r.stdout)[1])]
    assert keys == sorted(keys) and len(keys) == len(lines)


def test_sort_entry_equals_emulation(gpu_ctx, emul):
    data, starts = bam_inputs.bam_records(60_000, seed=3)
    got = gpu_ctx.bam_sort_compress(data, starts)
    want = bs.emul_once(emul, data, starts)
    assert got["z"] == want["z"] and got["carry"] == b"" and len(got["member_size"]) == want["n_members"]
    for fld in ("rid", "pos", "end", "bin", "flag", "block", "offset"):
        assert np.array_equal(got["recs"][fld], want["recs"][fld]), fld
    assert sum(got["member_size"]) == len(got["z"])
    # a window in the middle of a stream: a carry in, the unfinished block out
    carry = bytes(range(256)) * 100
    part = data[:starts[5000]]
    got = gpu_ctx.bam_sort_compress(part, starts[:5000], carry, last=False)
    want = bs.emul_once(emul, part, starts[:5000], carry, last=False)
    assert got["z"] == want["z"] and got["carry"] == want["carry"] and 0 < len(got["carry"]) < 65280
    assert np.array_equal(got["recs"]["block"], want["recs"]["block"]) and np.array_equal(got["recs"]["offset"], want["recs"]["offset"])
    assert all(v >= 0 for v in got["ms"].values()) and got["ms"]["sort"] > 0

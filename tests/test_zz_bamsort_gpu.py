"""bm2_sort on the GPU: bm2_bam_qname_sort_compress equals the host emulation (tests/host_emul/bamsort_emul.cpp) call by call, with the carry
passed across calls; `bm2_sort --write-index` of `bm2_mem --bam` output (paired, single-end, FASTA) has the records of `bm2_mem --sort` and
the emulation's bytes and index, and bm2_markdup and bm2_wgsmetrics give on it what they give on `bm2_mem --sort`'s output; `bm2_sort -n`
equals Python's name order on those BAMs and on crafted names and flags; sorting a sorted file changes nothing, and coordinate after name order
gives the input's multiset in coordinate order; the bytes do not depend on -t, --window, --sort-mem or standard input and output; and every
malformed, truncated or non-BAM input exits 1 and leaves no file."""
import gzip, json, os, struct, subprocess
import numpy as np
import pytest
import bam_util as bu
import bam_sort_util as bs
import bamsort_util as su
import markdup_bam_util as mb
import markdup_util as mu
import test_bam_sort_cpu as tsc
import test_bamsort_cpu as tc
import test_zz_bam_gpu as tg
import test_zz_markdup_gpu as tmg

pytestmark = pytest.mark.gpu

MEM = os.path.join(su.ROOT, "bwa-mem2_b200", "bm2_mem")
MARKDUP = os.path.join(su.ROOT, "bwa-mem2_b200", "bm2_markdup")
WGS = os.path.join(su.ROOT, "bwa-mem2_b200", "bm2_wgsmetrics")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return su.build_emul(tmp_path_factory)


def _flat(recs):
    return b"".join(recs), np.cumsum([0] + [len(r) for r in recs[:-1]]).astype(np.int64)


def _same(got, want):
    assert got["z"] == want["z"] and got["carry"] == want["carry"] and len(got["member_size"]) == want["n_members"]
    for f in ("rid", "pos", "end", "bin", "flag", "block", "offset"):
        assert np.array_equal(got["recs"][f], want["recs"][f]), f


def test_qname_sort_entry_equals_emulation(gpu_ctx, emul):
    rng = np.random.default_rng(41)
    recs = tc.records(rng, 20000)
    data, starts = _flat(recs)
    got = gpu_ctx.bam_qname_sort_compress(data, starts)
    _same(got, su.emul_once(emul, data, starts))
    assert got["ms"]["keys"] > 0 and got["ms"]["sort"] > 0 and got["ms"]["bgzf"] > 0
    srt = [r for _, r in bu.records(bu.inflate(got["z"]))]
    assert srt == su.name_order(recs)
    for window in ([recs[7]], [bs.make_rec(0, 5, f, name=b"same") for f in (0xc1, 0x81, 0x41, 0x1, 0x81, 0x41)] * 300):
        d, s = _flat(window)
        _same(gpu_ctx.bam_qname_sort_compress(d, s), su.emul_once(emul, d, s))
    carry, k = b"", 0                                                                     # windows one after another, the carry passed on
    for size in (1, 700, 3000, 40, 6000):
        part = recs[k:k + size]; k += size
        d, s = _flat(part)
        last = k >= 9741
        g = gpu_ctx.bam_qname_sort_compress(d, s, carry, last=last)
        _same(g, su.emul_once(emul, d, s, carry, last=last))
        carry = g["carry"]
    need, free = gpu_ctx.bam_qname_sort_memory(2 << 30)
    assert 0 < need < free


@pytest.fixture(scope="module")
def aligned(golden_dir, tmp_path_factory):
    if not os.path.exists(MEM):
        pytest.skip("bm2_mem not built")
    d = tmp_path_factory.mktemp("bamsort_gpu")
    prefix = os.path.join(golden_dir, "c0_index", "ref.fa")
    pairs = mu.planted_pairs(mu.load_reference(prefix), np.random.default_rng(43), n_base=150)
    files, _ = tmg._write_pairs(d, pairs, "p")
    bams = {}
    for tag in ("pe", "se", "fasta"):
        for mode in ("bam", "sort"):
            bams[tag, mode] = str(d / ("%s_%s.bam" % (tag, mode)))
            r = subprocess.run([MEM, "--" + mode, "-K", "20000", prefix] + files[tag] + ["-o", bams[tag, mode]], capture_output=True, timeout=900)
            assert r.returncode == 0, r.stderr[-3000:]
    return d, prefix, bams


def _tool(argv, stdin=None, env=None):
    r = su.run_tool(argv, stdin=stdin, env=env)
    return json.loads(r.stderr.decode().strip().split("\n")[-1]), r.stdout


def _check_file(emul, tmp, out, in_bam, by_name, argv, bai=None):
    """out: the header of su.out_header, then the emulation's members of the input's records, then the EOF block; bai: the emulation's index."""
    data = open(out, "rb").read()
    text, refs, recs = mb.read_bam(in_bam)
    got_text, got_refs, got_recs = mb.read_bam(out)
    assert got_text == su.out_header(text, by_name, argv) and got_refs == refs
    assert got_recs == su.expected_records(recs, by_name)
    part = tg._records_part(data)
    e, eb = str(tmp / "emul.part"), str(tmp / "emul.bai")
    su.emul_file(emul, b"".join(recs), 1 << 40, str(tmp / "emul.tmp."), e, by_name=by_name, bai_path=eb if bai else None,
                 out_off=len(data) - len(part), n_ref=len(refs))
    assert part == open(e, "rb").read() + bu.EOF_BLOCK
    if bai:
        assert open(bai, "rb").read() == open(eb, "rb").read()
    os.unlink(e)
    return got_recs


@pytest.mark.parametrize("tag", ["pe", "se", "fasta"])
def test_coordinate_sort_of_bam_equals_bm2_mem_sort(aligned, emul, tmp_path, tag):
    d, _, bams = aligned
    out = str(tmp_path / "x.bam")
    st, _ = _tool(["--write-index", "-o", out, bams[tag, "bam"]])
    assert sorted(os.listdir(tmp_path)) == ["x.bam", "x.bam.bai"]
    got = _check_file(emul, tmp_path, out, bams[tag, "bam"], False, [su.TOOL, "--write-index", "-o", out, bams[tag, "bam"]], bai=out + ".bai")
    assert got == mb.read_bam(bams[tag, "sort"])[2]
    data = open(out, "rb").read()
    tsc.check_index(out, out + ".bai", len(data) - len(tg._records_part(data)), len(mb.read_bam(out)[1]), np.random.default_rng(45))
    assert st["records"] == len(got) and st["sort_runs"] == 1 and st["sort_s"] > 0 and st["device_bytes"] > 0
    for k in ("windows", "in_bytes", "inflate_s", "spill_bytes", "merge_s", "merge_windows", "index_s", "wall_s"):
        assert k in st


def _data_lines(path):
    return [l for l in open(path).read().split("\n") if not l.startswith("#")]


def test_downstream_tools_accept_the_output(aligned, tmp_path):
    d, prefix, bams = aligned
    srt = str(tmp_path / "s.bam")
    _tool(["-o", srt, bams["pe", "bam"]])
    outs = {}
    for k, src in (("ours", srt), ("mem", bams["pe", "sort"])):
        md, mm, wg = str(tmp_path / (k + ".md.bam")), str(tmp_path / (k + ".md.txt")), str(tmp_path / (k + ".wgs.txt"))
        for argv in ([MARKDUP, "-M", mm, "-o", md, src], [WGS, "-o", wg, prefix, src]):
            r = subprocess.run(argv, capture_output=True, timeout=900)
            assert r.returncode == 0, r.stderr[-2000:]
        outs[k] = (mb.read_bam(md)[2], _data_lines(mm), _data_lines(wg))
    assert outs["ours"] == outs["mem"]


def crafted_bam(d):
    rng = np.random.default_rng(47)
    recs = tc.records(rng, 4000)
    recs += [bs.make_rec(k % 3, 10 * k, f, name=n) for k, (n, f) in enumerate(
        [(b"q7", 0xc1), (b"q07", 0x81), (b"q7", 0x41), (b"q7", 0x1), (b"n" + b"9" * 30, 0x41), (b"n" + b"0" * 5 + b"9" * 30, 0x41),
         (bytes([0xc3, 0xa9]) + b"1", 0), (b"x" * 254, 0x81), (b"x" * 254, 0x41)])]
    h, refs = mb.header(so="unsorted", pgs=("@PG\tID:bm2_sort\tPN:bm2_sort",))
    p = str(d / "crafted.bam")
    mb.write_bam(p, h, refs, recs, 97)
    return p


@pytest.mark.parametrize("tag", ["pe", "se", "fasta", "crafted"])
def test_name_sort_equals_python(aligned, emul, tmp_path, tag):
    _, _, bams = aligned
    src = crafted_bam(tmp_path) if tag == "crafted" else bams[tag, "bam"]
    out = str(tmp_path / "n.bam")
    st, _ = _tool(["-n", "-o", out, src])
    _check_file(emul, tmp_path, out, src, True, [su.TOOL, "-n", "-o", out, src])
    assert mb.read_bam(out)[0].split("\n")[0] == "@HD\tVN:1.6\tSO:queryname" and st["sort_s"] > 0
    if tag == "crafted":
        assert "@PG\tID:bm2_sort.1\tPN:bm2_sort\tPP:bm2_sort\t" in mb.read_bam(out)[0]


def test_chained_sorts(aligned, tmp_path):
    _, _, bams = aligned
    src = bams["pe", "bam"]
    recs = mb.read_bam(src)[2]
    c1, c2, n1, n2, nc = (str(tmp_path / x) for x in ("c1.bam", "c2.bam", "n1.bam", "n2.bam", "nc.bam"))
    _tool(["-o", c1, src]); _tool(["-o", c2, c1])
    _tool(["-n", "-o", n1, src]); _tool(["-n", "-o", n2, n1])
    _tool(["-o", nc, n1])
    assert mb.read_bam(c2)[2] == mb.read_bam(c1)[2] and mb.read_bam(n2)[2] == mb.read_bam(n1)[2]
    got = mb.read_bam(nc)[2]
    keys = [bs.key(bu.fields(r)) for r in got]
    assert keys == sorted(keys) and sorted(got) == sorted(recs)


@pytest.mark.parametrize("by_name", [False, True])
def test_bytes_do_not_depend_on_threads_windows_runs_or_stdin(aligned, tmp_path, by_name):
    _, _, bams = aligned
    src = bams["pe", "bam"]
    n = ["-n"] if by_name else []
    tmp = tmp_path / "tmpdir"; tmp.mkdir()
    env = dict(os.environ, TMPDIR=str(tmp))
    parts = []
    for k, (extra, stdin) in enumerate(((["-t", "1"], False), (["-t", "8", "--window", "64K"], False), (["--window", "256M"], True),
                                        (["--sort-mem", "64K", "-t", "3"], False), (["--sort-mem", "64K", "--window", "64K"], True),
                                        (["--sort-mem", "160K"], False), ([], False))):
        if stdin:
            with open(src, "rb") as f:
                st, data = _tool(n + extra + ["-"], stdin=f, env=env)
        else:
            out = str(tmp_path / ("v%d.bam" % k))
            st, _ = _tool(n + extra + ["-o", out, src], env=env)
            data = open(out, "rb").read()
        if "64K" in extra[:2]:                                # many runs (a run of about one BGZF block merges in one window)
            assert st["sort_runs"] >= 4 and st["spill_bytes"] > 0
        if "160K" in extra:                                   # runs larger than a merge window's share: several windows
            assert st["sort_runs"] >= 2 and st["merge_windows"] >= 2
        parts.append(tg._records_part(data))
        assert os.listdir(tmp) == []
    assert all(p == parts[0] for p in parts)
    assert sorted(os.listdir(tmp_path)) == ["tmpdir"] + sorted("v%d.bam" % k for k in (0, 1, 3, 5, 6))


def _malformed():
    r = bs.make_rec(0, 10, 0x41, name=b"bad")

    def patch(at, fmt, v):
        return r[:at] + struct.pack(fmt, v) + r[at + struct.calcsize(fmt):]
    yield "no_nul", patch(36 + 3, "<B", ord("x")), "read name does not end with NUL"
    yield "refid", patch(4, "<i", 3), "(read bad) is malformed: refID 3"
    yield "refid_low", patch(4, "<i", -2), "refID -2"
    yield "next_refid", patch(24, "<i", 7), "next refID 7"
    yield "pos", patch(8, "<i", -5), "pos -5"
    yield "overrun", patch(20, "<i", 5000), "malformed"
    yield "l_seq", patch(20, "<i", -3), "malformed"
    yield "lrn", patch(12, "<B", 0), "malformed"
    yield "block_size", (20).to_bytes(4, "little") + r[4:24], "malformed"


@pytest.mark.parametrize("case", [c[0] for c in _malformed()])
def test_malformed_input_exits_1_and_leaves_no_file(tmp_path, case):
    _, bad, text = next(c for c in _malformed() if c[0] == case)
    good = [bs.make_rec(0, 100, 0x41, name=b"ok%d" % k) for k in range(50)]
    h, refs = mb.header(so="unsorted")
    p = str(tmp_path / "in.bam")
    mb.write_bam(p, h, refs, good + [bad] + good)
    for by_name in (False, True):
        r = su.run_tool((["-n"] if by_name else []) + ["-o", str(tmp_path / "o.bam"), p], check=False)
        assert r.returncode == 1 and text in r.stderr.decode(), r.stderr
        assert os.listdir(tmp_path) == ["in.bam"]


def test_truncated_and_non_bam_inputs_exit_1(tmp_path):
    good = [bs.make_rec(0, 100 * k, 0x41, name=b"ok%d" % k) for k in range(3000)]
    h, refs = mb.header(so="unsorted")
    full = str(tmp_path / "full.bam")
    mb.write_bam(full, h, refs, good)
    data = open(full, "rb").read()
    cases = {"cut_member.bam": (data[:len(data) // 2], "truncated"), "text.bam": (b"@HD\tVN:1.6\n" * 10, "not BGZF"),
             "gzip.bam": (gzip.compress(b"hello" * 100), "not BGZF"),
             "notbam.bam": (mb.bgzf(b"CRAM" + bytes(100)) + bu.EOF_BLOCK, "not BAM"),
             "cut_record.bam": (mb.bgzf(mb.bam_bytes(h, refs, good)[:-10]) + bu.EOF_BLOCK, "ends inside record")}
    for name, (b, text) in cases.items():
        (tmp_path / name).write_bytes(b)
    for name, (_, text) in cases.items():
        r = su.run_tool(["-o", str(tmp_path / "o.bam"), str(tmp_path / name)], check=False)
        assert r.returncode == 1 and text in r.stderr.decode(), (name, r.stderr)
        assert sorted(os.listdir(tmp_path)) == sorted(list(cases) + ["full.bam"])
    r = su.run_tool(["--sort-mem", "1000G", "-o", str(tmp_path / "o.bam"), full], check=False)
    assert r.returncode == 1 and "bytes of device memory" in r.stderr.decode() and not os.path.exists(tmp_path / "o.bam")

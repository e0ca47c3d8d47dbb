"""bm2_bam2fq on the GPU: bm2_bam2fq_records and bm2_bam2fq_format equal the host emulation (tests/host_emul/bam2fq_emul.cpp) window by
window, and a window holding a bad record keeps nothing; the tool writes the emulation's bytes; `bm2_mem --bam` of FASTQ pairs, single-end
FASTQ and FASTA gives back the input files byte for byte; the BAMs of `--sort` and `--markdup` give back the same pairs; the bytes do not
depend on -t, --window or standard input; .gz outputs are bgzip-cut BGZF of the plain text; the interleaved stream of the input-order BAM
aligns as the two files do, and that of the sorted BAM aligns every read as half of a pair; a window whose text passes 2^31 bytes is
formatted and compressed correctly; errors exit with their code and leave no file."""
import gzip, io, json, os, subprocess
import numpy as np
import pytest
import bam2fq_util as bf
import bam_util as bu
import markdup_util as mu
import test_bam2fq_cpu as tc
import test_zz_markdup_gpu as tmg

pytestmark = pytest.mark.gpu

TOOL = bf.TOOL
MEM = os.path.join(bf.ROOT, "bwa-mem2_b200", "bm2_mem")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return bf.build_emul(tmp_path_factory)


def test_kernels_equal_emulation(gpu_ctx, emul):
    rng = np.random.default_rng(401)
    recs = tc.crafted() + tc.random_records(rng, 3000)
    for suffixes in (True, False):
        for a, b in ((0, 1), (0, 777), (777, len(recs))):
            win = recs[a:b]
            data, starts = bf._flat(win)
            got = gpu_ctx.bam2fq_records(b"".join(win), starts, suffixes)
            want, err = bf.emul_records(emul, win, suffixes)
            assert err == -1 and got.tobytes() == want.tobytes()
            extra = [r for r in recs[:40] if bf.kind(bf.fields(r)[1])]                 # the host lists kept records only
            kept = [i for i in range(len(win)) if got["kind"][i]]
            order = [kept[i] for i in rng.permutation(len(kept))] + [~k for k in rng.permutation(len(extra))]
            text = bf.emul_text(emul, win, order, extra, suffixes)
            assert text == b"".join(bf.text(win[i] if i >= 0 else extra[~i], suffixes) for i in order)
            plain, _, n = gpu_ctx.bam2fq_format(order, extra, suffixes)
            assert plain == text and n == len(text)
            carry = b"c" * 65279
            z, tail, _ = gpu_ctx.bam2fq_format(order, extra, suffixes, carry=carry, compress=True, last=False)
            full = carry + text
            cut = len(full) // 65280 * 65280
            assert gzip.decompress(z + bu.EOF_BLOCK) == full[:cut] and tail == full[cut:]
            assert all(len(r) == 65280 for _, r in bu.members(z))
            z2, tail2, _ = gpu_ctx.bam2fq_format(order, extra, suffixes, carry=carry, compress=True, last=True)
            assert gzip.decompress(z2) == full and tail2 == b"" and z2.startswith(z)
    assert min(gpu_ctx.bam2fq_stats()) > 0


def test_bad_window_keeps_nothing(gpu_ctx):
    ok = [bf.rec("a", 0x41, "ACGT", [30] * 4), bf.rec("a", 0x81, "ACGT", [30] * 4)]
    gpu_ctx.bam2fq_records(b"".join(ok), [0, len(ok[0])], True)
    for bad, text in ((bf.rec("q", 0, "AC", [30, 94]), "read q (record 2 of the window) has a quality above 93"),
                      (bf.rec("e", 0x41, "", None), "read e (record 2 of the window) has no bases")):
        w = ok + [bad]
        with pytest.raises(Exception, match=text.replace("(", r"\(").replace(")", r"\)")):
            gpu_ctx.bam2fq_records(b"".join(w), bf._flat(w)[1], True)
        with pytest.raises(Exception, match="names no record of the window"):
            gpu_ctx.bam2fq_format([0], [], True)


def _tool(argv, stdin=None):
    r = subprocess.run([TOOL] + argv, capture_output=True, timeout=900, stdin=stdin)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stderr.decode().strip().split("\n")[-1]), r.stdout


def test_tool_equals_emulation(emul, tmp_path):
    rng = np.random.default_rng(403)
    recs = tc.crafted() + tc.random_records(rng, 4000)
    p = tc._write(tmp_path, recs)
    for split, names in ((False, ["-o"]), (True, ["-1", "-2", "-0", "-s"])):
        for ext in (".fq", ".fq.gz"):
            for w in (200, 256 << 20):
                paths = [str(tmp_path / ("t%d_%d_%d%s" % (split, k, w, ext))) for k in range(len(names))]
                argv = ["--window", str(w), "-t", "3"] + [x for n, q in zip(names, paths) for x in (n, q)] + [p]
                st, _ = _tool(argv)
                epaths = [q + ".e" + ext for q in paths]
                rc, msg, est = bf.emul_run(emul, p, epaths, split=split, window=w)
                assert rc == 0, msg
                for q, e in zip(paths, epaths):
                    assert open(q, "rb").read() == open(e, "rb").read(), q
                for k in ("records", "kept", "pairs", "others", "singletons", "pending_max", "pending_bytes_max", "windows"):
                    assert st[k] == est[k], k
                assert st["record_s"] > 0 and st["pair_s"] >= 0 and st["format_s"] > 0 and (st["bgzf_s"] > 0) == ext.endswith(".gz")


@pytest.fixture(scope="module")
def aligned(golden_dir, tmp_path_factory):
    if not os.path.exists(MEM):
        pytest.skip("bm2_mem not built")
    d = tmp_path_factory.mktemp("bam2fq_gpu")
    prefix = os.path.join(golden_dir, "c0_index", "ref.fa")
    ref = mu.load_reference(prefix)
    pairs = mu.planted_pairs(ref, np.random.default_rng(405), n_base=120)
    files, _ = tmg._write_pairs(d, pairs, "p")
    bams = {}
    for tag, args, fs in (("bam", ["--bam"], files["pe"]), ("se", ["--bam"], files["se"]), ("fasta", ["--bam"], files["fasta"]),
                          ("sort", ["--sort"], files["pe"]), ("markdup", ["--markdup"], files["pe"])):
        bams[tag] = str(d / (tag + ".bam"))
        r = subprocess.run([MEM] + args + ["-K", "20000", prefix] + fs + ["-o", bams[tag]], capture_output=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
    return d, prefix, files, bams


def test_round_trip_is_byte_identical(aligned):
    d, _, files, bams = aligned
    st, _ = _tool(["-1", str(d / "r1.fq"), "-2", str(d / "r2.fq"), bams["bam"]])
    assert open(d / "r1.fq", "rb").read() == open(files["pe"][0], "rb").read()
    assert open(d / "r2.fq", "rb").read() == open(files["pe"][1], "rb").read()
    assert st["pairs"] > 100 and st["singletons"] == 0 and st["others"] == 0 and st["pending_max"] == 0
    _tool(["-o", str(d / "se.fq"), bams["se"]])
    assert open(d / "se.fq", "rb").read() == open(files["se"][0], "rb").read()
    _tool(["-1", str(d / "f1.fa"), "-2", str(d / "f2.fa"), bams["fasta"]])
    assert open(d / "f1.fa", "rb").read() == open(files["fasta"][0], "rb").read()
    assert open(d / "f2.fa", "rb").read() == open(files["fasta"][1], "rb").read()


def _fq_records(data):
    lines = data.split(b"\n")
    return sorted(tuple(lines[i:i + 4]) for i in range(0, len(lines) - 1, 4))


@pytest.mark.parametrize("tag", ["sort", "markdup"])
def test_sorted_bams_give_the_same_pairs(aligned, tag):
    d, _, files, bams = aligned
    o1, o2 = str(d / (tag + "1.fq")), str(d / (tag + "2.fq"))
    st, _ = _tool(["--window", "16K", "-1", o1, "-2", o2, bams[tag]])                # mates carried across windows
    assert st["pending_max"] > 0 and st["windows"] > 3 and st["singletons"] == 0
    a, b = open(o1, "rb").read(), open(o2, "rb").read()
    assert _fq_records(a) == _fq_records(open(files["pe"][0], "rb").read())
    assert _fq_records(b) == _fq_records(open(files["pe"][1], "rb").read())
    assert [x[0] for x in (_split4(a))] == [x[0] for x in _split4(b)]                 # in step: the mates line up


def _split4(data):
    lines = data.split(b"\n")
    return [tuple(lines[i:i + 4]) for i in range(0, len(lines) - 1, 4)]


def test_bytes_do_not_depend_on_threads_windows_or_stdin(aligned):
    d, _, _, bams = aligned
    base = None
    for k, (extra, stdin) in enumerate(((["-t", "1"], False), (["-t", "4", "--window", "10K"], False), (["--window", "1"], True),
                                        (["-t", "16", "--window", "64K"], True))):
        outs = [str(d / ("v%d_%s" % (k, n))) for n in ("i.fq", "i.fq.gz", "1.fq.gz", "2.fq.gz")]
        if stdin:
            with open(bams["sort"], "rb") as f:
                _tool(extra + ["-o", outs[1], "-"], stdin=f)
            with open(bams["sort"], "rb") as f:
                _, so = _tool(extra + ["-"], stdin=f)
            open(outs[0], "wb").write(so)
        else:
            _tool(extra + ["-o", outs[0], bams["sort"]])
            _tool(extra + ["-o", outs[1], bams["sort"]])
        _tool(extra + ["-1", outs[2], "-2", outs[3], bams["sort"]])
        got = [open(o, "rb").read() for o in outs]
        assert gzip.decompress(got[1]) == got[0] and got[1].endswith(bu.EOF_BLOCK)
        sizes = [len(r) for _, r in bu.members(got[1])]
        assert all(s == 65280 for s in sizes[:-2]) and sizes[-1] == 0
        base = base or got
        assert got == base, k


def _sam_records(text):
    return [l for l in text.decode().split("\n") if l and not l.startswith("@")]


def test_interleaved_stream_aligns_as_the_files(aligned):
    d, prefix, files, bams = aligned
    k = ["-K", "100000000"]                                                             # one chunk each: the same insert-size estimate
    fq = subprocess.run([TOOL, bams["bam"]], capture_output=True, timeout=900).stdout
    r = subprocess.run([MEM, "-p"] + k + [prefix, "-"], input=fq, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    r2 = subprocess.run([MEM] + k + [prefix] + files["pe"], capture_output=True, timeout=900)
    assert r2.returncode == 0
    assert _sam_records(r.stdout) == _sam_records(r2.stdout)
    fs = subprocess.run([TOOL, bams["sort"]], capture_output=True, timeout=900).stdout
    r3 = subprocess.run([MEM, "-p"] + k + [prefix, "-"], input=fs, capture_output=True, timeout=900)
    assert r3.returncode == 0
    prim = [l.split("\t") for l in _sam_records(r3.stdout)]
    prim = [f for f in prim if not int(f[1]) & 0x900]
    assert len(prim) == 2 * len(_split4(open(files["pe"][0], "rb").read())) and all(int(f[1]) & 1 for f in prim)


def test_window_text_past_2_31_bytes(gpu_ctx):
    rng = np.random.default_rng(407)
    L, n = 600_000, 2000
    seq = "".join(rng.choice(list("ACGT"), L))
    one = bf.rec("r0000", 0x41 | 0x10, seq, [37] * L)
    recs = [one[:36] + (b"r%04d" % k) + one[41:] for k in range(n)]
    data = b"".join(recs)
    starts = np.arange(n, dtype=np.int64) * len(recs[0])
    info = gpu_ctx.bam2fq_records(data, starts, True)
    assert int(info["text_len"].sum()) > (1 << 31)
    z, tail, tl = gpu_ctx.bam2fq_format(list(range(n)), [], True, compress=True, last=True)
    assert tl == int(info["text_len"].sum()) and tail == b""
    body = bf.text(bf.rec("r0000", 0x41 | 0x10, seq, [37] * L), True)[len(b"@r0000/1"):]
    with gzip.GzipFile(fileobj=io.BytesIO(z)) as g:
        for k in range(n):
            want = b"@r%04d/1" % k + body
            assert g.read(len(want)) == want, k
        assert g.read(1) == b""


def test_errors_exit_with_their_code_and_leave_no_file(tmp_path):
    bad = [bf.rec("a", 0x41, "ACGT", [30] * 4), bf.rec("a", 0x41, "ACGT", [30] * 4)]
    p = tc._write(tmp_path, bad)
    out = str(tmp_path / "o")
    for argv, code, text in ((["-1", out + "1.fq.gz", "-2", out + "2.fq", p], 1, "two READ1"),
                             (["-o", str(tmp_path / "no_dir" / "x.fq"), p], 2, "cannot open"),
                             (["-o", out + ".fq", str(tmp_path / "missing.bam")], 1, "cannot open")):
        r = subprocess.run([TOOL] + argv, capture_output=True, timeout=300)
        assert r.returncode == code and text in r.stderr.decode(), r.stderr
        assert sorted(os.listdir(tmp_path)) == ["in.bam"]
    r = subprocess.run([TOOL, "--window", "1000G", "-o", out + ".fq", p], capture_output=True, timeout=300)
    assert r.returncode == 1 and "bytes of device memory" in r.stderr.decode() and sorted(os.listdir(tmp_path)) == ["in.bam"]

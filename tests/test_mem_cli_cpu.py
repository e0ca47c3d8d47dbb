"""The command line of bwa-mem2_b200/bm2_mem against the reference's own option parser, without a GPU.

`bm2_mem --dump-opt` prints the parsed bm2_mem_opt_t, the -I values, the read group id and the header, and stops before any device call.
The reference side: oracle/_ref/<isa>/ref_driver runs the unmodified `main_mem` (src/fastmap.cpp:616-943), and with BM2_MODE=gpu it hands
its parsed mem_opt_t and the contigs' ALT marks to `bm2_create` of the library named by BM2_LIB.  Here that library is a stand-in compiled by
the test: its bm2_create writes what it was given to a file and ends the process, by which time the reference has printed its header.
The smart-pairing model (bseq_classify, src/bwa.cpp:226-242) is at the end; tests/test_zz_mem_cli_gpu.py checks the GPU split against it."""
import json, os, shutil, subprocess
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")

FAKE_LIB = r"""
#include "bm2_b200.h"
#include <cstdio>
#include <cstdlib>
extern "C" int bm2_create(bm2_ctx **, int, const bm2_index_desc *idx, const bm2_mem_opt_t *opt) {
    FILE *f = fopen(getenv("BM2_FAKE_DUMP"), "wb");
    fwrite(opt, sizeof *opt, 1, f);
    int n = idx ? idx->n_seqs : 0;
    fwrite(&n, 4, 1, f);
    for (int i = 0; i < n; ++i) { int a = idx->ann_is_alt ? idx->ann_is_alt[i] : 0; fwrite(&a, 4, 1, f); }
    fclose(f);
    exit(0);
}
extern "C" void bm2_destroy(bm2_ctx *) {}
extern "C" const char *bm2_last_error(const bm2_ctx *) { return "stand-in"; }
extern "C" int bm2_extend_pairs(bm2_ctx *, bm2_seqpair *, const uint8_t *, const uint8_t *, int32_t, int32_t, int32_t) { return 1; }
extern "C" int bm2_seed_chain_extend(bm2_ctx *, const bm2_read_batch *, bm2_reg_result *) { return 1; }
"""

RG = r"@RG\tID:g1\tSM:s1\tPL:ILLUMINA"

# (name, arguments of both programs, input): "pe" two files, "se" one file, "inter" one interleaved file; hdr / hdrsq: -H files
CASES = [
    ("defaults", [], "pe"),
    ("se", [], "se"),
    ("5SP", ["-5SP"], "pe"),
    ("aMY", ["-aMY"], "pe"),
    ("qCV1v", ["-q", "-C", "-V", "-1", "-v", "1"], "pe"),
    ("attached", ["-k15", "-w60", "-T20", "-d80", "-h3,50"], "pe"),
    ("seeding", ["-c", "20", "-r", "1.0", "-D", "0.3", "-m", "10", "-s", "5", "-G", "500", "-N", "30", "-W", "10", "-y", "5", "-X", "0.3"], "pe"),
    ("Q40_U9", ["-Q", "40", "-U", "9"], "pe"),
    ("Q0", ["-Q", "0"], "pe"),
    ("t3_K5000", ["-t", "3", "-K", "5000"], "pe"),
    ("A2", ["-A", "2"], "pe"),
    ("A2_explicit", ["-A", "2", "-B", "3", "-O", "5", "-E", "2", "-L", "3", "-U", "7", "-T", "25", "-d", "80"], "pe"),
    ("pairs", ["-O", "5,7", "-E", "2,1", "-L", "3,9", "-h", "3,50", "-I", "400,40,700,100"], "pe"),
    ("I400", ["-I", "400"], "pe"),
    ("I400,40", ["-I", "400,40"], "pe"),
    ("x_intractg", ["-x", "intractg"], "pe"),
    ("x_pacbio", ["-x", "pacbio"], "pe"),
    ("x_pbref", ["-x", "pbref"], "pe"),
    ("x_ont2d", ["-x", "ont2d"], "pe"),
    ("x_ont2d_over", ["-x", "ont2d", "-k", "19", "-B", "3", "-L", "2", "-r", "2.5", "-W", "7"], "pe"),
    ("x_intractg_A2", ["-x", "intractg", "-A", "2"], "pe"),        # update_a is not applied with -x
    ("R", ["-R", RG], "pe"),
    ("R_twice", ["-R", r"@RG\tID:first", "-R", r"@RG\tID:second\tSM:x"], "pe"),
    ("H_inline_R", ["-H", r"@CO\tone\\two", "-H", "@CO\tthree", "-R", RG], "pe"),
    ("H_file", ["-H", "{hdr}"], "pe"),
    ("H_file_SQ_R", ["-H", "{hdrsq}", "-R", RG], "pe"),
    ("H_not_header", ["-H", "nothing-here"], "pe"),
    ("o", ["-o", "{out}"], "pe"),
    ("f", ["-f", "{out}"], "pe"),
    ("smart", ["-p"], "inter"),
    ("smart_cluster", ["-aMp"], "inter"),
    ("smart_second_file", ["-p", "-M"], "inter+"),
    ("permuted", ["{idx}", "-M", "{r1}", "-k", "17", "{r2}"], "none"),
    ("alt", [], "pe_alt"),
    ("alt_j", ["-j"], "pe_alt"),
]

ERRORS = [
    ("x_unknown", ["-x", "bogus"]),
    ("R_no_at", ["-R", r"RG\tID:x"]),
    ("R_no_id", ["-R", r"@RG\tSM:x"]),
    ("R_long_id", ["-R", "@RG\\tID:" + "a" * 256]),
    ("unknown_option", ["-Z"]),
    ("missing_argument", ["-k"]),
]


def _driver():
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    drv = os.path.join(ROOT, "oracle", "_ref", isa, "ref_driver")
    if not os.path.exists(TOOL) or not os.path.exists(drv):
        pytest.skip("bm2_mem / oracle/_ref not built")
    return drv


@pytest.fixture(scope="module")
def work(tmp_path_factory, golden_dir):
    import importlib
    drv = _driver()
    d = tmp_path_factory.mktemp("mem_cli")
    fake = str(d / "libfake.so")
    src = d / "fake.cpp"; src.write_text(FAKE_LIB)
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"), str(src), "-o", fake])
    synth = importlib.import_module("bwa_mem2_b200.synth")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"][:16]
    synth.write_fastq(str(d / "r1.fq"), reads[0::2], "p"); synth.write_fastq(str(d / "r2.fq"), reads[1::2], "p")
    with open(d / "inter.fq", "wb") as f:
        for i, r in enumerate(reads):
            s = bytes(b"ACGTN"[c] for c in r)
            f.write(b"@p%d/%d\n%s\n+\n%s\n" % (i // 2, i % 2 + 1, s, b"I" * len(s)))
    (d / "hdr.txt").write_text("@CO\tfrom a file\n@CO\tescaped\\ttab\nnot a header line\n")
    (d / "hdrsq.txt").write_text("@SQ\tSN:chr1\tLN:100\n@CO\tlast\n")
    alt = d / "altidx"; alt.mkdir()
    for f in os.listdir(golden_dir + "/c0_index"):
        shutil.copy(os.path.join(golden_dir, "c0_index", f), alt / f)
    (alt / "ref.fa.alt").write_text("chr3\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\nchr4\t0\tchr1\t1\t60\t100M\t*\t0\t0\t*\t*\n")
    return dict(drv=drv, fake=fake, d=d, idx=golden_dir + "/c0_index/ref.fa", alt=str(alt / "ref.fa"))


def _command(w, args, inp, out):
    d = w["d"]
    sub = {"{hdr}": str(d / "hdr.txt"), "{hdrsq}": str(d / "hdrsq.txt"), "{out}": out, "{idx}": w["idx"], "{r1}": str(d / "r1.fq"), "{r2}": str(d / "r2.fq")}
    args = [sub.get(a, a) for a in args]
    files = {"pe": [w["idx"], str(d / "r1.fq"), str(d / "r2.fq")], "se": [w["idx"], str(d / "r1.fq")], "inter": [w["idx"], str(d / "inter.fq")],
             "inter+": [w["idx"], str(d / "inter.fq"), str(d / "r2.fq")], "pe_alt": [w["alt"], str(d / "r1.fq"), str(d / "r2.fq")], "none": []}[inp]
    return args + files


def _reference(w, argv, tag):
    dump = str(w["d"] / ("ref_%s.bin" % tag))
    if os.path.exists(dump):
        os.remove(dump)
    env = dict(os.environ, BM2_MODE="gpu", BM2_LIB=w["fake"], BM2_FAKE_DUMP=dump)
    r = subprocess.run([w["drv"], "mem"] + argv, env=env, capture_output=True, timeout=300)
    return r, dump


def _field_values(capi, raw):
    o = capi.MemOpt.from_buffer_copy(raw[:C_sizeof(capi.MemOpt)])
    return {name: (list(getattr(o, name)) if name == "mat" else getattr(o, name)) for name, _ in capi.MemOpt._fields_}


def C_sizeof(t):
    import ctypes
    return ctypes.sizeof(t)


@pytest.mark.parametrize("name,args,inp", CASES, ids=[c[0] for c in CASES])
def test_options_and_header_equal_the_reference(pkg, work, name, args, inp):
    capi = pkg.capi
    out_ref, out_ours = str(work["d"] / ("%s.ref.sam" % name)), str(work["d"] / ("%s.ours.sam" % name))
    ref, dump = _reference(work, _command(work, args, inp, out_ref), name)
    assert ref.returncode == 0 and os.path.exists(dump), ref.stderr[-2000:]
    raw = open(dump, "rb").read()
    want = _field_values(capi, raw)
    n = int(np.frombuffer(raw, np.int32, 1, C_sizeof(capi.MemOpt))[0])
    want_alt = np.frombuffer(raw, np.int32, n, C_sizeof(capi.MemOpt) + 4).tolist()
    ours = subprocess.run([TOOL, "--dump-opt"] + _command(work, args, inp, out_ours), capture_output=True, text=True, timeout=120)
    assert ours.returncode == 0, ours.stderr[-2000:]
    got = json.loads(ours.stdout)
    for k, v in want.items():
        if isinstance(v, float):
            assert np.float32(got[k]) == np.float32(v), (k, got[k], v)
        else:
            assert got[k] == v, (k, got[k], v)
    ref_text = open(out_ref).read() if "{out}" in args else ref.stdout.decode()
    ref_hdr = "".join(l + "\n" for l in ref_text.split("\n") if l.startswith("@") and not l.startswith("@PG"))
    assert got["header"] == ref_hdr
    assert [("\tAH:*" in l) for l in got["header"].split("\n") if l.startswith("@SQ")] == [bool(a) for a in want_alt][:got["header"].count("@SQ\tSN")] \
        or "{hdrsq}" in args
    if any(a.startswith("-R") for a in args):
        rg = [a for a in args if a.startswith("@RG")][-1]
        assert got["rg_id"] == rg.replace("\\t", "\t").split("\tID:")[1].split("\t")[0]
    else:
        assert got["rg_id"] is None
    assert got["copy_comment"] == ("-C" in args)
    assert got["smart_pairing"] == bool(want["flag"] & 0x400)
    assert got["files"] == (1 if inp in ("se", "inter", "inter+") else 2)


def test_insert_size_values(work):
    """-I avg[,std[,max[,min]]] (src/fastmap.cpp:760-775)."""
    def parse(v):
        o = subprocess.run([TOOL, "--dump-opt", "-I", v, work["idx"], "a.fq", "b.fq"], capture_output=True, text=True, timeout=60)
        assert o.returncode == 0, o.stderr
        return json.loads(o.stdout)["pes"]
    assert parse("400") == {"low": 240, "high": 560, "avg": 400.0, "std": 40.0}
    assert parse("400,40") == {"low": 240, "high": 560, "avg": 400.0, "std": 40.0}
    assert parse("400,30") == {"low": 280, "high": 520, "avg": 400.0, "std": 30.0}
    assert parse("400,40,700,100") == {"low": 100, "high": 700, "avg": 400.0, "std": 40.0}
    assert parse("20,10") == {"low": 1, "high": 60, "avg": 20.0, "std": 10.0}


def test_worker_count_and_smart_pairing_flag(work):
    """`-p N` as separate arguments with N a positive decimal integer is the number of chunks in flight; any other -p is smart pairing."""
    def run(*args):
        o = subprocess.run([TOOL, "--dump-opt"] + list(args), capture_output=True, text=True, timeout=60)
        assert o.returncode == 0, o.stderr
        return json.loads(o.stdout)
    idx, r1, r2 = work["idx"], str(work["d"] / "r1.fq"), str(work["d"] / "r2.fq")
    j = run("-t", "4", "-K", "40000", "-p", "2", "-o", "/dev/null", idx, r1, r2)
    assert j["workers"] == 2 and not j["smart_pairing"] and j["files"] == 2 and j["flag"] == 0x2 and j["chunk_size"] == 40000
    j = run("-p", "3", "-p", idx, r1)
    assert j["workers"] == 3 and j["smart_pairing"] and j["files"] == 1
    j = run("-p", idx, r1)
    assert j["workers"] == 2 and j["smart_pairing"]
    o = subprocess.run([TOOL, "--dump-opt", "-p", "0", idx, r1], capture_output=True, text=True, timeout=60)
    assert o.returncode != 0 and "index 0" in o.stderr     # not a positive count: smart pairing, and "0" is the index prefix
    j = run("-5SP", "-p", "1", idx, r1, r2)
    assert j["workers"] == 1 and not j["smart_pairing"] and j["flag"] & 0x1800 == 0x1800
    j = run("-k", "-p", idx, r1)                       # "-p" as the argument of -k
    assert j["min_seed_len"] == 0 and j["workers"] == 2 and not j["smart_pairing"]


@pytest.mark.parametrize("name,args", ERRORS, ids=[e[0] for e in ERRORS])
def test_errors_exit_nonzero_in_both(work, name, args):
    ref, dump = _reference(work, _command(work, args, "pe", ""), "err_" + name)
    assert ref.returncode != 0 and not os.path.exists(dump)
    ours = subprocess.run([TOOL, "--dump-opt"] + _command(work, args, "pe", ""), capture_output=True, text=True, timeout=60)
    assert ours.returncode != 0


def test_wrong_argument_count_exits_nonzero(work):
    for files in ([], [work["idx"]], [work["idx"], "a", "b", "c"]):
        assert subprocess.run([TOOL, "--dump-opt"] + files, capture_output=True, timeout=60).returncode != 0
        r, dump = _reference(work, files, "argc")
        assert r.returncode != 0 and not os.path.exists(dump)


# ---- smart pairing: bseq_classify (src/bwa.cpp:226-242) restated --------------------------------------------------------------------

def classify(names):
    """-> (indices of the single-end reads, indices of the paired reads), both in input order."""
    se, pe = [], []
    has_last = True
    for i in range(1, len(names)):
        if has_last:
            if names[i] == names[i - 1]:
                pe += [i - 1, i]; has_last = False
            else:
                se.append(i - 1)
        else:
            has_last = True
    if names and has_last:
        se.append(len(names) - 1)
    return se, pe


def name_patterns():
    """Name lists of the GPU test: runs of 1-7 equal names, alternating runs, all pairs, all singletons, one read."""
    pats = {}
    rng = np.random.default_rng(11)
    runs = [int(x) for x in rng.integers(1, 8, 200)]
    pats["runs_1_7"] = [b"r%d" % k for k, n in enumerate(runs) for _ in range(n)]
    pats["alternating"] = [b"a%d" % k for k in range(120) for _ in range(1 + k % 2)]
    pats["all_pairs"] = [b"q%d" % (i // 2) for i in range(300)]
    pats["all_single"] = [b"s%d" % i for i in range(301)]
    pats["one_read"] = [b"x"]
    pats["prefix_names"] = [b"ab", b"abc", b"abc", b"ab", b"ab", b"ab"]
    return pats


def test_smart_pairing_model():
    assert classify([b"a", b"a", b"a"]) == ([2], [0, 1])
    assert classify([b"a", b"b", b"b", b"c"]) == ([0, 3], [1, 2])
    assert classify([b"a"] * 4) == ([], [0, 1, 2, 3])
    assert classify([b"a"] * 5) == ([4], [0, 1, 2, 3])
    assert classify([b"x"]) == ([0], [])
    assert classify([]) == ([], [])
    for name, names in name_patterns().items():
        se, pe = classify(names)
        assert sorted(se + pe) == list(range(len(names))), name
        assert all(names[pe[2 * k]] == names[pe[2 * k + 1]] and pe[2 * k + 1] == pe[2 * k] + 1 for k in range(len(pe) // 2)), name
        # the rule of the device scan: in a run of equal names starting at s, read i pairs with read i-1 iff i - s is odd
        run, with_prev = 0, []
        for i in range(len(names)):
            if i == 0 or names[i] != names[i - 1]:
                run = i
            with_prev.append((i - run) % 2 == 1)
        pe2 = [i for i in range(len(names)) if with_prev[i] or (i + 1 < len(names) and with_prev[i + 1])]
        assert pe2 == pe, name

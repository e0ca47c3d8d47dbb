"""bm2_index without a GPU.

- bm2_fasta_pack writes .pac / .ann / .amb byte-identical to the unmodified reference's `bwa-mem2 index` (oracle/_ref) on a corpus of small
  FASTA / FASTQ files (tests/index_corpus.py): N runs and IUPAC codes, mixed case, N-only contigs, contigs that start or end with N and N runs
  across contig boundaries, empty records, comments, names ending in /1, wrapped lines, CRLF, junk before the first header, FASTQ records,
  gzip and multi-member gzip, l_pac % 4 in 0..3.
- The tool's usage line and exit codes match `bwa-mem2 index`; malformed and empty inputs are errors with a message.
- tests/host_emul/fmi_emul.cpp (bm2_index_build's passes, rounds and windows over fmi_device.cuh, compiled with g++) gives the suffix array of
  a naive sort and of index_build.suffix_array on hostile texts with a tiny work budget, and index_build.build_fm_arrays' CP_OCC and sampled SA.
"""
import ctypes as C
import os, subprocess
import numpy as np
import pytest
import torch

import index_corpus as ic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bwa-mem2_b200", "csrc")
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_index")
CORPUS = ic.corpus()


def _ref_bin():
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    p = os.path.join(ROOT, "oracle", "_ref", isa, "bwa-mem2")
    if not os.path.exists(p):
        pytest.skip("oracle/_ref not built")
    return p


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_fasta_pack_equals_reference(pkg, tmp_path, name):
    ref = _ref_bin()
    fa = tmp_path / name
    fa.write_bytes(CORPUS[name])
    subprocess.run([ref, "index", "-p", str(tmp_path / "ref"), str(fa)], check=True, capture_output=True, timeout=300)
    st = pkg.capi.fasta_pack(str(fa), str(tmp_path / "ours"))
    for ext in (".pac", ".ann", ".amb"):
        assert (tmp_path / ("ours" + ext)).read_bytes() == (tmp_path / ("ref" + ext)).read_bytes(), ext
    assert st["l_pac"] == int((tmp_path / "ref.ann").read_text().split()[0])


def test_fasta_pack_keeps_drand48_state(pkg, tmp_path):
    # the draws come from a private state: a caller's srand48 sequence goes on as if the pack never ran
    libc = C.CDLL(None)
    libc.lrand48.restype = C.c_long
    libc.srand48(5); want = [libc.lrand48() for _ in range(3)]
    libc.srand48(5); got = [libc.lrand48()]
    (tmp_path / "a.fa").write_bytes(CORPUS["n_runs_iupac.fa"])
    pkg.capi.fasta_pack(str(tmp_path / "a.fa"), str(tmp_path / "a"))
    got += [libc.lrand48() for _ in range(2)]
    assert got == want


def _run(args, **kw):
    return subprocess.run(args, capture_output=True, timeout=300, **kw)


def test_tool_usage_and_exit_codes_match_reference(tmp_path):
    ref = _ref_bin()
    if not os.path.exists(TOOL):
        pytest.skip("bm2_index not built")
    for args in ([], ["-p"], ["-x", "in.fa"], ["-p", "pfx"]):
        a, b = _run([TOOL] + args, cwd=tmp_path), _run([ref, "index"] + args, cwd=tmp_path)
        assert a.returncode == b.returncode == 1, args
        usage_a = [l for l in a.stderr.decode().splitlines() if l.startswith("Usage")]
        usage_b = [l.replace("bwa-mem2 index", "bm2_index") for l in b.stderr.decode().splitlines() if l.startswith("Usage")]
        assert usage_a == usage_b, args


def test_default_prefix_is_the_input(pkg, tmp_path):
    # -p absent: the files go next to the input, named after it (the pack step runs without a GPU; the build step needs one)
    if not os.path.exists(TOOL):
        pytest.skip("bm2_index not built")
    (tmp_path / "g.fa").write_bytes(CORPUS["edges.fa"])
    r = _run([TOOL, str(tmp_path / "g.fa")])
    assert (tmp_path / "g.fa.pac").exists() and (tmp_path / "g.fa.ann").exists() and (tmp_path / "g.fa.amb").exists()
    if r.returncode:
        assert b"bm2_index_build" in r.stderr


@pytest.mark.parametrize("data,what", [
    (b"@r1\nACGT\n+\nII\n", b"malformed record 1"),
    (b">a\nACGT\n@r2\nAC\n+\n", b"malformed record 2"),
    (b"", b"no sequence"),
    (b">only_empty\n>another\n", b"no sequence"),
    (b"no header at all\n", b"no sequence"),
])
def test_bad_inputs_are_errors(pkg, tmp_path, data, what):
    (tmp_path / "x.fa").write_bytes(data)
    with pytest.raises(pkg.capi.Bm2Error) as e:
        pkg.capi.fasta_pack(str(tmp_path / "x.fa"), str(tmp_path / "x"))
    assert what.decode() in str(e.value)
    if os.path.exists(TOOL):
        r = _run([TOOL, str(tmp_path / "x.fa")])
        assert r.returncode == 1 and what in r.stderr


# ---- the builder's structure on the host ----

@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fmi_emul") / "libfmiemul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC,
                           os.path.join(ROOT, "tests", "host_emul", "fmi_emul.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.fmi_emul.restype = C.c_int
    lib.fmi_emul.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64] + [C.c_void_p] * 5

    def run(t, cap, win):
        t = np.ascontiguousarray(t, np.uint8); n = len(t); N = n + 1
        sa = np.zeros(n, np.int64); cp = np.zeros(((N >> 6) + 1, 8), np.int64)
        ms = np.zeros((N >> 3) + 1, np.int8); ls = np.zeros((N >> 3) + 1, np.uint32); info = np.zeros(6, np.int64)
        rc = lib.fmi_emul(t.ctypes.data, n, cap, win, sa.ctypes.data, cp.ctypes.data, ms.ctypes.data, ls.ctypes.data, info.ctypes.data)
        assert rc == 0
        return sa, cp, ms, ls, dict(zip(("groups", "pieces", "rounds", "windows", "sentinel", "cap"), info.tolist()))
    return run


def _naive(t):
    s = bytes(np.asarray(t, np.uint8) + 1)
    return np.array(sorted(range(len(t)), key=lambda i: s[i:]), np.int64)


def _texts():
    rng = np.random.default_rng(11)
    unit = rng.integers(0, 4, 50, dtype=np.uint8)
    out = {
        # test_index_build.test_suffix_array_against_naive's text
        "index_build_naive": np.concatenate([np.tile(unit, 40), rng.integers(0, 2, 500, dtype=np.uint8), np.zeros(70, np.uint8), np.tile(unit, 7),
                                             np.zeros(40, np.uint8)]),
        "tandem": np.concatenate([np.tile(np.array([0, 1, 2], np.uint8), 400), np.tile(np.array([3, 0], np.uint8), 300), rng.integers(0, 4, 200, dtype=np.uint8)]),
        "poly_a": np.concatenate([rng.integers(0, 4, 300, dtype=np.uint8), np.zeros(900, np.uint8), rng.integers(0, 4, 300, dtype=np.uint8), np.zeros(200, np.uint8)]),
        "random_end_ties": np.repeat(rng.integers(0, 2, 125, dtype=np.uint8), 20),
    }
    c = rng.integers(0, 4, 700, dtype=np.uint8)
    out["two_identical_contigs"] = np.concatenate([c, c])
    # every text as bm2_index sees it: forward then reverse complement
    return {k: np.concatenate([v, (3 - v)[::-1]]).astype(np.uint8) for k, v in out.items()}


TEXTS = _texts()


@pytest.mark.parametrize("name", sorted(TEXTS))
def test_emul_suffix_array_equals_naive_and_index_build(emul, name):
    import importlib
    ib = importlib.import_module("bwa_mem2_b200.index_build")
    t = TEXTS[name]
    sa, cp, ms, ls, info = emul(t, 64, 128)
    assert np.array_equal(sa, _naive(t))
    assert np.array_equal(sa, ib.suffix_array(torch.from_numpy(t), max_bucket=256).numpy())
    assert info["groups"] > 1 and info["windows"] > 1 and info["rounds"] >= 1 and info["pieces"] > info["rounds"], info


@pytest.mark.parametrize("name", sorted(TEXTS))
def test_emul_fm_arrays_equal_index_build(emul, name):
    import importlib
    ib = importlib.import_module("bwa_mem2_b200.index_build")
    t = TEXTS[name]
    sa, cp, ms, ls, info = emul(t, 96, 192)
    fm = ib.build_fm_arrays(torch.from_numpy(t), torch.from_numpy(sa))
    assert np.array_equal(cp, fm["cp_occ"].numpy())
    assert np.array_equal(ms, fm["sa_ms"].numpy()) and np.array_equal(ls.astype(np.int64), fm["sa_ls"].numpy())
    assert info["sentinel"] == fm["sentinel"]


def test_emul_random_genome_with_wide_budget(emul):
    # one group, one window: the same answer as the many-group run
    rng = np.random.default_rng(5)
    v = rng.integers(0, 4, 3000, dtype=np.uint8)
    t = np.concatenate([v, (3 - v)[::-1]]).astype(np.uint8)
    a = emul(t, 64, 64)[0]
    b = emul(t, 1 << 20, 1 << 16)
    assert b[4]["groups"] == 1 and b[4]["windows"] == 1
    assert np.array_equal(a, b[0]) and np.array_equal(a, _naive(t))

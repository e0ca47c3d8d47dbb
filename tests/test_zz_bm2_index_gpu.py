"""bm2_index on the GPU against the unmodified reference's `bwa-mem2 index` (oracle/_ref) and index_build.py.

- The corpus of tests/index_corpus.py, a 100 Mbp genome with N runs and IUPAC codes wrapped at 60, and a 20 Mbp low-entropy genome (long identical
  copies, (AT)n, poly-A, two identical contigs: many rounds, tie groups that span pieces): all five files byte-identical to the reference's, built
  by the tool at the default budget and through the C ABI with a work budget small enough for several groups, pieces and windows.
- 1 Gbp (index_build.make_big_reference as FASTA): .bwt.2bit.64, .0123 and .pac byte-identical to index_build.write_index's.
- bm2_mem on the bm2_index-built 100 Mbp index writes the SAM it writes on the reference-built one.
"""
import os, shutil, subprocess
import numpy as np
import pytest

import index_corpus as ic

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_index")
MEM = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
FILES = (".pac", ".ann", ".amb", ".0123", ".bwt.2bit.64")


def _ref_bin():
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    p = os.path.join(ROOT, "oracle", "_ref", isa, "bwa-mem2")
    if not os.path.exists(p):
        pytest.skip("oracle/_ref not built")
    return p


def _same(a, b, files=FILES):
    for ext in files:
        x = np.fromfile(a + ext, np.uint8); y = np.fromfile(b + ext, np.uint8)
        assert x.shape == y.shape and np.array_equal(x, y), ext


def _build_three_ways(pkg, d, fa, work_bytes):
    """reference, tool (default budget), C ABI with work_bytes; returns the C ABI build's stats."""
    subprocess.run([_ref_bin(), "index", "-p", d + "/ref", fa], check=True, capture_output=True, timeout=1800)
    r = subprocess.run([TOOL, "-p", d + "/tool", fa], capture_output=True, timeout=1800)
    assert r.returncode == 0, r.stderr.decode()
    pkg.capi.fasta_pack(fa, d + "/small")
    st = pkg.capi.index_build(d + "/small", 0, work_bytes)
    _same(d + "/tool", d + "/ref")
    _same(d + "/small", d + "/ref")
    return st


def test_corpus_equals_reference(pkg, tmp_path):
    for name, data in sorted(ic.corpus().items()):
        d = str(tmp_path / name.replace(".", "_")); os.makedirs(d)
        fa = d + "/" + name
        open(fa, "wb").write(data)
        st = _build_three_ways(pkg, d, fa, 4096)
        if st["n"] > 1000:
            assert st["groups"] > 1 and st["windows"] > 1, (name, st)


def test_100mbp_with_ambiguous_bases_equals_reference(pkg, tmp_path):
    d = str(tmp_path); fa = d + "/g.fa"
    open(fa, "wb").write(ic.synthetic_fasta(100_000_000, seed=21))
    st = _build_three_ways(pkg, d, fa, 128 << 20)
    assert st["groups"] > 1 and st["windows"] > 1 and st["pieces"] > st["rounds"] >= 1, st
    # the tool's output loads: bm2_mem gives the same SAM (but the @PG line's paths) on both indexes
    import importlib
    synth = importlib.import_module("bwa_mem2_b200.synth")
    fwd = np.fromfile(d + "/ref.0123", np.uint8)[:int(open(d + "/ref.ann").read().split()[0])]
    rng = np.random.default_rng(4)
    starts = rng.integers(0, len(fwd) - 200, 4000)
    reads = np.stack([fwd[s:s + 151] for s in starts])
    reads[rng.random(reads.shape) < 0.01] ^= 1
    synth.write_fastq_fast(d + "/r.fq", reads)
    sams = []
    for pfx in ("ref", "tool"):
        out = subprocess.run([MEM, "-t", "4", d + "/" + pfx, d + "/r.fq"], capture_output=True, timeout=900, check=True).stdout
        sams.append([l for l in out.split(b"\n") if not l.startswith(b"@PG")])
    assert sams[0] == sams[1] and len(sams[0]) > 4000


def test_20mbp_low_entropy_equals_reference(pkg, tmp_path):
    d = str(tmp_path); fa = d + "/low.fa"
    open(fa, "wb").write(ic.low_entropy_fasta(20_000_000, seed=9))
    st = _build_three_ways(pkg, d, fa, 64 << 20)
    assert st["rounds"] >= 4 and st["pieces"] > st["rounds"] and st["groups"] > 1 and st["windows"] > 1, st


def test_1gbp_equals_index_build(pkg, tmp_path):
    import importlib, torch
    ib = importlib.import_module("bwa_mem2_b200.index_build")
    d = str(tmp_path)
    contigs = ib.make_big_reference(1_000_000_000, seed=3, device="cuda")
    acgt = np.frombuffer(b"ACGT", np.uint8)
    with open(d + "/big.fa", "wb") as f:
        for name, c in contigs:
            f.write(b">" + name.encode() + b"\n")
            f.write(ic.fasta_lines(acgt[c.cpu().numpy()], 60))
    r = subprocess.run([TOOL, "-p", d + "/tool", d + "/big.fa"], capture_output=True, timeout=3000)
    assert r.returncode == 0, r.stderr.decode()
    os.remove(d + "/big.fa")
    ib.write_index(d + "/ib", contigs, device="cuda")
    del contigs
    torch.cuda.empty_cache()
    _same(d + "/tool", d + "/ib", (".bwt.2bit.64", ".0123", ".pac"))
    shutil.rmtree(d, ignore_errors=True)

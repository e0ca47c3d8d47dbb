"""Lazy extension on the GPU: bm2_seed_chain_extend with BM2_EXT_LAZY=0 (every extension job in one wave) and with the default
(waves, purged seeds never extended) must give byte-identical regs, on the golden C0 reads and on the config-1 inputs (10 Mbp synthetic
reference, 10 000 synthetic 2x151 bp pairs), unsplit and as sub-batches in flight."""
import os, subprocess, tempfile
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _both(pkg, idx, codes, offs, monkeypatch, sub_batches=1):
    ctx = pkg.capi.Context(0, index=idx)
    if sub_batches > 1:
        ctx.set_sub_batches(sub_batches, 512)
    out = {}
    for lazy in ("0", "1"):
        monkeypatch.setenv("BM2_EXT_LAZY", lazy)
        regs, ro = ctx.seed_chain_extend(codes, offs)
        out[lazy] = (regs, ro, ctx.counters())
    ctx.close()
    (r0, o0, c0), (r1, o1, c1) = out["0"], out["1"]
    assert len(r0) > 1000
    assert np.array_equal(o0, o1) and r0.tobytes() == r1.tobytes()
    assert c0["jobs_skipped"] == 0 and c1["jobs_skipped"] > 0 and c1["reads_done_wave1"] > 0
    assert c1["cells"] < c0["cells"]
    return c0, c1


def test_lazy_extension_golden(pkg, golden_dir, monkeypatch):
    idx = pkg.capi.Index(golden_dir + "/c0_index/ref.fa")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    codes = reads.reshape(-1); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    _both(pkg, idx, codes, offs, monkeypatch)
    idx.close()


def test_lazy_extension_config1(pkg, monkeypatch):
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    bwa = os.path.join(ROOT, "oracle", "_ref", isa, "bwa-mem2")
    if not os.path.exists(bwa):
        pytest.skip("oracle/_ref not built")
    import importlib
    synth = importlib.import_module("bwa_mem2_b200.synth")
    work = tempfile.mkdtemp(prefix="bm2_lazy_")
    ctg = synth.make_reference(10_000_000, seed=101, n_contigs=5)
    synth.write_fasta(work + "/ref.fa", ctg)
    subprocess.check_call([bwa, "index", work + "/ref.fa"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    r1, r2 = synth.make_pairs_fast(ctg, 10_000, seed=102)
    reads = np.concatenate([r1, r2])
    codes = np.ascontiguousarray(reads.reshape(-1)); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    idx = pkg.capi.Index(work + "/ref.fa")
    _both(pkg, idx, codes, offs, monkeypatch)
    _both(pkg, idx, codes, offs, monkeypatch, sub_batches=4)
    idx.close()

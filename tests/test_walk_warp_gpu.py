"""The post-filter walk of the lazy extension on the GPU walks every read: those with more than BM2_TAIL_HEAVY (24) regs a warp each
(ext_walk_read_warp), the others one per thread.  The regs must be byte-identical with BM2_EXT_LAZY=0 and with the default, and the jobs
skipped and the reads decided after the first wave must equal the host model's (tests/host_emul/lazy_emul.cpp, told to walk every read,
with the per-thread walk), on the golden C0 reads, the tandem-repeat golden reads (over a thousand chains per read) and the config-1 inputs
(10 Mbp synthetic reference, 10 000 synthetic 2x151 bp pairs), unsplit and as sub-batches in flight."""
import os, subprocess, tempfile
import numpy as np
import pytest
import lazy_emul_lib as ll

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(pkg, idx, codes, offs, monkeypatch):
    monkeypatch.setenv("BM2_EXT_WALK_HEAVY", str(1 << 30))      # the host model walks every read, as the kernels do
    _, _, model = ll.seed_chain_extend(idx, pkg.capi.default_opt(), codes, offs)
    assert model["skipped"] > 0 and model["kept_not_extended"] == 0
    for sub_batches in (1, 4):
        ctx = pkg.capi.Context(0, index=idx)
        if sub_batches > 1:
            ctx.set_sub_batches(sub_batches, 512)
        out = {}
        for lazy in ("0", "1"):
            monkeypatch.setenv("BM2_EXT_LAZY", lazy)
            regs, ro = ctx.seed_chain_extend(codes, offs)
            out[lazy] = (regs, ro, ctx.counters())
        ctx.close()
        (r0, o0, _), (r1, o1, c1) = out["0"], out["1"]
        assert len(r0) > 1000
        assert np.array_equal(o0, o1) and r0.tobytes() == r1.tobytes(), sub_batches
        assert (c1["jobs_skipped"], c1["reads_done_wave1"]) == (model["skipped"], model["done_wave1"]), sub_batches
    return model


def test_walk_golden(pkg, golden_dir, monkeypatch):
    idx = pkg.capi.Index(golden_dir + "/c0_index/ref.fa")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    codes = reads.reshape(-1); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    _check(pkg, idx, codes, offs, monkeypatch)
    idx.close()


def test_walk_tandem(pkg, golden_dir, monkeypatch):
    idx = pkg.capi.Index(golden_dir + "/tandem_index/ref.fa")
    rd = np.load(golden_dir + "/tandem_reads.npz")
    model = _check(pkg, idx, rd["codes"], rd["offs"], monkeypatch)
    # the heavy reads matter here: left unwalked, they would run more jobs, so the GPU's counts above came from walking them
    monkeypatch.setenv("BM2_EXT_WALK_HEAVY", "24")
    _, _, light_only = ll.seed_chain_extend(idx, pkg.capi.default_opt(), rd["codes"], rd["offs"])
    assert light_only["skipped"] < model["skipped"]
    idx.close()


def test_walk_config1(pkg, monkeypatch):
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    bwa = os.path.join(ROOT, "oracle", "_ref", isa, "bwa-mem2")
    if not os.path.exists(bwa):
        pytest.skip("oracle/_ref not built")
    import importlib
    synth = importlib.import_module("bwa_mem2_b200.synth")
    work = tempfile.mkdtemp(prefix="bm2_walk_")
    ctg = synth.make_reference(10_000_000, seed=101, n_contigs=5)
    synth.write_fasta(work + "/ref.fa", ctg)
    subprocess.check_call([bwa, "index", work + "/ref.fa"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    r1, r2 = synth.make_pairs_fast(ctg, 10_000, seed=102)
    reads = np.concatenate([r1, r2])
    codes = np.ascontiguousarray(reads.reshape(-1)); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    idx = pkg.capi.Index(work + "/ref.fa")
    _check(pkg, idx, codes, offs, monkeypatch)
    idx.close()

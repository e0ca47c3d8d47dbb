"""Config 1 at its stated size through the GPU path: a 10 Mbp synthetic reference (several contigs, planted repeat families,
N runs) indexed live by the unmodified reference's `bwa-mem2 index`, 10 000 synthetic 2x151 bp pairs, default mem_opt_t.  The pure reference
run and the run whose worker_bwt + worker_aln are replaced by libbm2b200.so through the C ABI (ref_driver BM2_MODE=gpu) must print the same
SAM - SAM diff = 0, as the config asks.  (tests/test_dropin_sam_gpu.py is the same check on the small committed golden set.)"""
import os, subprocess, tempfile
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bin(name):
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    p = os.path.join(ROOT, "oracle", "_ref", isa, name)
    if not os.path.exists(p):
        pytest.skip("oracle/_ref not built")
    return p


def test_config1_sam_diff_is_zero(pkg):
    import importlib
    synth = importlib.import_module("bwa_mem2_b200.synth")
    work = tempfile.mkdtemp(prefix="bm2_cfg1_")
    ctg = synth.make_reference(10_000_000, seed=101, n_contigs=5)
    # a few N runs so that .amb is not trivial (the indexer replaces them by random bases, the reads see what the index holds)
    rng = np.random.default_rng(7)
    for _, c in ctg:
        for _ in range(3):
            p = int(rng.integers(1000, len(c) - 2000)); c[p:p + int(rng.integers(20, 400))] = 4
    synth.write_fasta(work + "/ref.fa", ctg)
    subprocess.check_call([_bin("bwa-mem2"), "index", work + "/ref.fa"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    r1, r2 = synth.make_pairs_fast(ctg, 10_000, seed=102)
    synth.write_fastq_fast(work + "/r1.fq", r1); synth.write_fastq_fast(work + "/r2.fq", r2)
    args = [_bin("ref_driver"), "mem", "-t", "8", "-K", "100000000", work + "/ref.fa", work + "/r1.fq", work + "/r2.fq"]
    outs = {}
    for mode in ("ref", "gpu"):
        env = dict(os.environ, BM2_MODE=mode, BM2_LIB=pkg.capi.LIB_PATH)
        o = subprocess.run(args, env=env, capture_output=True, text=True, timeout=900)
        assert o.returncode == 0, o.stderr[-2000:]
        outs[mode] = [l for l in o.stdout.splitlines() if not l.startswith("@PG")]
    assert len(outs["ref"]) == len(outs["gpu"]) and len(outs["ref"]) >= 20_000
    diff = [i for i, (a, b) in enumerate(zip(outs["ref"], outs["gpu"])) if a != b]
    assert diff == [], (len(diff), outs["ref"][diff[0]], outs["gpu"][diff[0]])

"""bm2_mem's streamed input on the GPU.

- bm2_mem's SAM on BGZF input (files, standard input, smart pairing, BGZF then plain gzip) is byte-identical to its SAM on the same reads as
  plain files, at 1 and 2 chunks in flight, and to the reference's where oracle/_ref is built.
- bm2_mem's peak RSS on standard input does not grow with the input."""
import gzip, json, os, subprocess
import numpy as np
import pytest
import seq_corpus as sc
import test_mem_cli_cpu as cli
from test_input_stream_cpu import bgzf, peak_rss

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def inputs(tmp_path_factory, golden_dir):
    if not os.path.exists(cli.TOOL):
        pytest.skip("bm2_mem not built")
    d = tmp_path_factory.mktemp("input_stream_gpu")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    rng = np.random.default_rng(12)
    L = reads.shape[1]
    seq = [bytes(np.frombuffer(b"ACGTN", np.uint8)[r]) for r in reads]
    qual = [bytes(rng.integers(35, 74, L).astype(np.uint8)) for _ in range(len(reads))]
    mate = [[(b"p%d/%d" % (i // 2, w + 1), seq[i], qual[i]) for i in range(w, len(reads), 2)] for w in (0, 1)]
    inter = [r for pair in zip(mate[0], mate[1]) for r in pair]
    f = {}

    def put(name, data):
        p = d / name; p.write_bytes(data); f[name] = str(p)
    plain = {"1": sc.fastq(mate[0]), "2": sc.fastq(mate[1], 60), "i": sc.fastq(inter)}
    for k, v in plain.items():
        put(k + ".fq", v); put(k + ".bgz", bgzf(v, block=4000))
    v = plain["1"]
    put("1.mix.gz", bgzf(v[:len(v) // 2], block=3000, eof=False) + gzip.compress(v[len(v) // 2:]))
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    drv = os.path.join(ROOT, "oracle", "_ref", isa, "ref_driver")
    return dict(d=d, f=f, idx=golden_dir + "/c0_index/ref.fa", drv=drv if os.path.exists(drv) else None)


def _mem(inputs, args, paths, stdin=None, tag="x"):
    out = str(inputs["d"] / ("%s.sam" % tag))
    o = subprocess.run([cli.TOOL, "-t", "4"] + args + ["-o", out, inputs["idx"]] + paths, input=stdin, capture_output=True, timeout=600)
    assert o.returncode == 0, o.stderr[-2000:]
    return [l for l in open(out, "rb").read().split(b"\n") if not l.startswith(b"@PG")], json.loads(o.stderr.decode().strip().splitlines()[-1])


# (name, smart pairing, BGZF inputs ("-": standard input), standard input, the same reads as plain files)
CASES = [
    ("pe", [], ["1.bgz", "2.bgz"], None, ["1.fq", "2.fq"]),
    ("se", [], ["1.bgz"], None, ["1.fq"]),
    ("smart", ["-p"], ["i.bgz"], None, ["i.fq"]),
    ("stdin_pe", [], ["-", "2.bgz"], "1.bgz", ["1.fq", "2.fq"]),
    ("mixed", [], ["1.mix.gz"], None, ["1.fq"]),
]


@pytest.mark.parametrize("workers", [1, 2])
@pytest.mark.parametrize("name,args,files,stdin,plain", CASES, ids=[c[0] for c in CASES])
def test_bm2_mem_on_bgzf_equals_plain(inputs, name, args, files, stdin, plain, workers):
    f = inputs["f"]
    base = ["-K", "20000", "-p", str(workers)] + args
    data = open(f[stdin], "rb").read() if stdin else None
    got, st = _mem(inputs, base, [p if p == "-" else f[p] for p in files], data, "%s_%d" % (name, workers))
    want, st0 = _mem(inputs, base, [f[p] for p in plain], None, "%s_%d_plain" % (name, workers))
    assert len(got) > 40 and got == want
    assert st["reads"] == st0["reads"] and st["gzip_members"] > 10 and st0["gzip_members"] == 0
    if inputs["drv"] is not None:
        ref = subprocess.run([inputs["drv"], "mem", "-t", "4", "-K", "20000"] + args + [inputs["idx"]] + [f[p] for p in plain],
                             env=dict(os.environ, BM2_MODE="ref"), capture_output=True, timeout=600)
        assert ref.returncode == 0, ref.stderr[-2000:]
        assert [l for l in ref.stdout.split(b"\n") if not l.startswith(b"@PG")] == got


def test_bm2_mem_peak_memory_does_not_grow_with_the_input(inputs):
    """N and 2N reads on standard input, N large enough that the second run's extra input (about 300 MB) is a large share of the
    process's peak RSS (CUDA context, index, buffers): a reader that held its input whole would grow by that much"""
    block = open(inputs["f"]["1.fq"], "rb").read() * 100

    def run(reps):
        def feed(f):
            for _ in range(reps):
                f.write(block)
        rc, _, err, rss = peak_rss([cli.TOOL, "-t", "8", "-K", "10000000", "-o", "/dev/null", inputs["idx"], "-"], feed, inputs["d"] / "rss",
                                   subprocess.DEVNULL)
        assert rc == 0, err[-2000:]
        return rss, json.loads(err.decode().strip().splitlines()[-1])
    reps = 300_000_000 // len(block) + 1
    r1, s1 = run(reps)
    r2, s2 = run(2 * reps)
    assert s2["reads"] == 2 * s1["reads"]
    extra = reps * len(block)
    assert r2 - r1 < 0.1 * r1 and r2 - r1 < 0.2 * extra, (r1, r2, extra)
    assert s2["input_peak_bytes"] < 1.1 * s1["input_peak_bytes"] and s2["input_peak_bytes"] < 0.5 * extra, (s1["input_peak_bytes"], s2["input_peak_bytes"])

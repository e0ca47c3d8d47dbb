"""How fast bm2_mem reads each input shape: the same reads as four-line FASTQ (bm2_fastq_encode), single-line FASTA, FASTA wrapped at 60 and
FASTQ wrapped at 60 (bm2_seq_encode), each aligned by one bm2_mem run.  Prints one JSON line per shape with the parse + encode time
(fastq_encode_s, summed over chunks and workers), the chunk loop time and reads/s, and the card's name and power limit.

    python scripts/seq_input_rate.py [--pairs 500000] [--ref-mbp 50] [--threads 16] [-K 30000000]

The genome, index and reads are those of bench.py's pipeline workload (cached under the temporary directory)."""
import argparse, json, os, subprocess, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def write_shapes(reads, work):
    """the reads (codes 0-4, one row per read) in the four shapes; qualities are one constant byte"""
    L = reads.shape[1]
    seq = np.frombuffer(b"ACGTN", np.uint8)[reads]
    names = [b"r%d" % i for i in range(len(reads))]
    q = b"I" * L
    wrap = lambda s: b"\n".join(s[i:i + 60] for i in range(0, len(s), 60))
    shapes = {"fastq_4line": lambda n, s: b"@" + n + b"\n" + s + b"\n+\n" + q + b"\n",
              "fasta_1line": lambda n, s: b">" + n + b"\n" + s + b"\n",
              "fasta_60": lambda n, s: b">" + n + b"\n" + wrap(s) + b"\n",
              "fastq_60": lambda n, s: b"@" + n + b"\n" + wrap(s) + b"\n+\n" + wrap(q) + b"\n"}
    paths = {}
    for name, fmt in shapes.items():
        p = os.path.join(work, "shape_%s" % name)
        if not os.path.exists(p):
            with open(p, "wb") as f:
                for i in range(len(reads)):
                    f.write(fmt(names[i], seq[i].tobytes()))
        paths[name] = p
    return paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=500_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--workers", type=int, default=2)
    a = ap.parse_args()
    import bench
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    paths = write_shapes(reads, work)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    digests = {}
    for name, p in paths.items():
        out = os.path.join(work, "shape_out.sam")
        r = subprocess.run([tool, "-t", str(a.threads), "-K", str(a.K), "-p", str(a.workers), "-o", out, fa, p], capture_output=True, text=True, check=True)
        st = json.loads(r.stderr.strip().splitlines()[-1])
        # the alignments (columns 1-10 but QUAL) must not depend on the input shape
        import hashlib
        h = hashlib.sha256()
        with open(out, "rb") as f:
            for ln in f:
                if not ln.startswith(b"@"):
                    h.update(b"\t".join(ln.split(b"\t")[:10]))
        digests[name] = h.hexdigest()
        os.remove(out)
        print(json.dumps({"shape": name, "reads": st["reads"], "chunks": st["chunks"], "seq_encode_chunks": st["seq_encode_chunks"],
                          "fastq_encode_s": st["fastq_encode_s"], "loop_s": st["loop_s"], "reads_per_s": st["reads"] / st["loop_s"],
                          "bytes": os.path.getsize(p), "gpu": gpu[0] if gpu else None, "same_alignments": digests[name] == digests["fastq_4line"]}),
              flush=True)


if __name__ == "__main__":
    main()

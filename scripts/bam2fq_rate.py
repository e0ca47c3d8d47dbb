"""What bm2_bam2fq costs: wall time and the stderr JSON's times of `bm2_bam2fq -t 16` on the unsorted (`bm2_mem --bam`, input order) and the
marked (`bm2_mem --markdup`, coordinate order) BAM of bqsr_rate.py's 1.1 M pairs, interleaved plain and BGZF, after a warm-up; the format
kernel alone on one window of about 256 MB of records (CUDA events, bytes read plus written per second); and host zlib at level 6 on the
same FASTQ text, one thread.  Prints JSON lines, with the card's name and power limit.

    python scripts/bam2fq_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--reps 3]"""
import argparse, json, os, subprocess, sys, tempfile, time, zlib
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    # markdup_rate.py's and bqsr_rate.py's reads and qualities, under unique names: their Illumina-like names repeat every 30 000 reads
    # within a tile, which the interleaved input-order BAM tolerates but a sorted one, where such names meet out of order, does not
    p1, p2 = os.path.join(work, "bam2fq_rate_1.fq"), os.path.join(work, "bam2fq_rate_2.fq")
    if not os.path.exists(p2):
        rng = np.random.default_rng(78)
        n = len(reads) // 2
        dup = np.sort(rng.choice(n, int(n * 0.1), replace=False))
        pick = np.concatenate([np.arange(n), dup])
        rd = np.stack([reads[0::2][pick], reads[1::2][pick]], 1).reshape(-1, reads.shape[1])
        quals = bam_inputs.illumina_quals(len(rd), rd.shape[1], np.random.default_rng(77))
        for path, m in ((p1, 0), (p2, 1)):
            with open(path, "wb") as f:
                for i in range(0, len(rd) // 2, 100_000):
                    f.write(b"".join(b"@p%d\n" % k + bytes(b"ACGTN"[c] for c in rd[2 * k + m]) + b"\n+\n" + bytes(quals[2 * k + m]) + b"\n"
                                     for k in range(i, min(len(rd) // 2, i + 100_000))))
    mem = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_bam2fq")
    bams = {"unsorted": os.path.join(work, "bam2fq_rate.unsorted.bam"), "marked": os.path.join(work, "bam2fq_rate.marked.bam")}
    for kind, flags in (("unsorted", ["--bam"]), ("marked", ["--markdup"])):
        subprocess.run([mem] + flags + ["-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o", bams[kind], fa, p1, p2], capture_output=True, check=True)
    print(json.dumps({"progress": "inputs ready", "gpu": gpu, **{k: os.path.getsize(v) for k, v in bams.items()}}), flush=True)
    out = os.path.join(work, "bam2fq_rate.out")
    for rep in range(-1, a.reps):                                       # rep -1: warm-up, not counted
        for kind, path in bams.items():
            for ext in (".fq", ".fq.gz"):
                t0 = time.perf_counter()
                r = subprocess.run([tool, "-t", str(a.threads), "-o", out + ext, path], capture_output=True, text=True)
                if r.returncode:
                    sys.exit(r.stderr[-2000:])
                wall = time.perf_counter() - t0
                st = json.loads(r.stderr.strip().splitlines()[-1])
                if rep >= 0:
                    print(json.dumps({"what": "bm2_bam2fq", "bam": kind, "out": ext, "rep": rep, "gpu": gpu, "wall_s": wall,
                                      **{k: st[k] for k in ("records", "pairs", "pending_max", "pending_bytes_max", "windows", "in_bytes", "out_bytes",
                                                            "inflate_s", "record_s", "pair_s", "format_s", "bgzf_s", "wall_s")}}), flush=True)

    # ---- the format kernel alone on one window of about 256 MB of the unsorted BAM's records, and host zlib on its text
    import bam_util as bu
    from __graft_entry__ import load_package
    capi = load_package().capi
    raw = bu.inflate(open(bams["unsorted"], "rb").read())
    _, _, used = bu.parse_header(raw)
    body = raw[used:]
    starts, last = [], 0
    for st, r in bu.records(body):                                       # the whole records of the first 256 MB
        if st + len(r) > 256 << 20:
            break
        starts.append(st); last = st + len(r)
    n, win = len(starts), body[:last]
    ctx = capi.Context(0)
    info = ctx.bam2fq_records(win, np.array(starts, np.int64), True)
    order = [i for i in range(n) if info["kind"][i]]
    kept_bytes = sum(int.from_bytes(win[starts[i]:starts[i] + 4], "little") + 4 for i in order)
    text = b""
    for rep in range(5):
        f0 = ctx.bam2fq_stats()[1]
        text, _, tl = ctx.bam2fq_format(order, [], True)
        ms = ctx.bam2fq_stats()[1] - f0
        if rep:
            print(json.dumps({"what": "format_kernel", "rep": rep, "gpu": gpu, "records": len(order), "record_bytes": kept_bytes, "text_bytes": tl,
                              "device_ms": ms, "bytes_per_s": (kept_bytes + tl) / (ms / 1e3),
                              "share_of_3.35TB/s": (kept_bytes + tl) / (ms / 1e3) / 3.35e12}), flush=True)
    ctx.close()
    t0 = time.perf_counter()
    c = zlib.compressobj(6, zlib.DEFLATED, 31)
    z = c.compress(text) + c.flush()
    dt = time.perf_counter() - t0
    print(json.dumps({"what": "host_zlib_level6", "gpu": gpu, "text_bytes": len(text), "out_bytes": len(z), "s": dt, "bytes_per_s": len(text) / dt}), flush=True)


if __name__ == "__main__":
    main()

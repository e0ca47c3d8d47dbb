"""What bm2_wgsmetrics costs: three runs at -t 16 after a warm-up on the marked BAM of scripts/bqsr_rate.py's input (wall time, records/s and
the stderr JSON's inflate_s, add_s and finish_s), and bm2_wgs_finish alone over a genome-sized counter array (CUDA events over several calls,
bytes/s of the counters and the no-call bitset).  Prints JSON lines, with the card's name and power limit.

    python scripts/wgsmetrics_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [--reps 3] [--loci 3100000000]

The BAM comes from `bm2_mem --markdup` on bqsr_rate.py's reads (run that script first, or this one makes the same inputs through it).  The
finish pass runs over counters that are all zero, so every locus falls in one bin."""
import argparse, json, os, subprocess, sys, tempfile, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loci", type=int, default=3_100_000_000)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa, vcf = os.path.join(work, "ref.fa"), os.path.join(work, "bqsr_rate_30.vcf")
    p1, p2 = os.path.join(work, "markdup_rate_1.fq"), os.path.join(work, "markdup_rate_2.fq")
    if not all(os.path.exists(p) for p in (vcf, p2)):                   # bqsr_rate.py's inputs, made by its own code (one rep)
        subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bqsr_rate.py"), "--pairs", str(a.pairs), "--ref-mbp", str(a.ref_mbp),
                        "--reps", "1"], check=True, stdout=subprocess.DEVNULL)
    md = os.path.join(work, "wgsmetrics_rate.md.bam")
    mem = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    subprocess.run([mem, "--markdup", "-R", r"@RG\tID:g1\tSM:s", "-t", str(a.threads), "-K", "30000000", "-o", md, fa, p1, p2], check=True,
                   capture_output=True)
    print(json.dumps({"progress": "inputs ready", "bam_bytes": os.path.getsize(md)}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_wgsmetrics")
    out = os.path.join(work, "wgsmetrics_rate.txt")
    for rep in range(-1, a.reps):                                          # rep -1: warm-up, not counted
        t0 = time.perf_counter()
        r = subprocess.run([tool, "-t", str(a.threads), "-o", out, fa, md], capture_output=True, text=True, check=True)
        wall = time.perf_counter() - t0
        st = json.loads(r.stderr.strip().splitlines()[-1])
        if rep < 0:
            continue
        print(json.dumps({"what": "bm2_wgsmetrics", "rep": rep, "gpu": gpu, "threads": a.threads, "wall_s": wall, "records_per_s": st["records"] / wall,
                          **{k: st[k] for k in ("records", "counted_records", "windows", "in_bytes", "inflate_s", "add_s", "finish_s", "carried_max",
                                                "device_bytes")}}), flush=True)

    # ---- bm2_wgs_finish alone over a genome-sized counter array
    from __graft_entry__ import load_package
    capi = load_package().capi
    ctx = capi.Context(0)
    ctx.wgs_set([0], [min(a.loci, 2**31 - 1)], a.loci, [])
    nbytes = a.loci * 4 + a.loci // 8
    for rep in range(6):
        s = ctx.wgs_finish()
        if rep:
            print(json.dumps({"what": "wgs_finish", "rep": rep, "gpu": gpu, "loci": a.loci, "finish_ms": s["finish_ms"], "bytes": nbytes,
                              "bytes_per_s": nbytes / (s["finish_ms"] / 1e3), "datasheet_bytes_per_s": 3.35e12}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

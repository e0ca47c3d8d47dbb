"""What bm2_multiplemetrics costs: three runs at -t 16 after a warm-up on the marked, coordinate-sorted BAM of `bm2_mem --markdup` and on the
unsorted BAM of `bm2_mem --bam`, both over scripts/bqsr_rate.py's reads (wall time, records/s and the stderr JSON's inflate_s, add_s and
finish_s), and bm2_mm_add alone on one window of each (CUDA events over several calls, aligned bases/s).  Prints JSON lines, with the
card's name and power limit.

    python scripts/multiplemetrics_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [--reps 3] [--window-mb 256]

On the unsorted BAM the reference reads of a window are scattered over the whole reference; the two windows measure what that costs the
count kernel."""
import argparse, json, os, subprocess, sys, tempfile, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def window_of(bam, limit):
    """The records of the first `limit` uncompressed bytes after the header: (bytes, starts)."""
    import bam_util as bu
    raw = bu.inflate(open(bam, "rb").read())
    _, _, used = bu.parse_header(raw)
    body = raw[used:]
    starts, at = [], 0
    while at + 4 <= len(body):
        n = int.from_bytes(body[at:at + 4], "little") + 4
        if at + n > limit:
            break
        starts.append(at); at += n
    return body[:at], np.array(starts, np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--window-mb", type=int, default=256)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa, vcf = os.path.join(work, "ref.fa"), os.path.join(work, "bqsr_rate_30.vcf")
    p1, p2 = os.path.join(work, "markdup_rate_1.fq"), os.path.join(work, "markdup_rate_2.fq")
    if not all(os.path.exists(p) for p in (vcf, p2)):                   # bqsr_rate.py's inputs, made by its own code (one rep)
        subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bqsr_rate.py"), "--pairs", str(a.pairs), "--ref-mbp", str(a.ref_mbp),
                        "--reps", "1"], check=True, stdout=subprocess.DEVNULL)
    mem = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    bams = {}
    for kind in ("markdup", "bam"):
        bams[kind] = os.path.join(work, f"multiplemetrics_rate.{kind}.bam")
        subprocess.run([mem, "--" + kind, "-R", r"@RG\tID:g1\tSM:s", "-t", str(a.threads), "-K", "30000000", "-o", bams[kind], fa, p1, p2],
                       check=True, capture_output=True)
    print(json.dumps({"progress": "inputs ready", **{k + "_bytes": os.path.getsize(v) for k, v in bams.items()}}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_multiplemetrics")
    out = os.path.join(work, "multiplemetrics_rate")
    for kind, bam in bams.items():
        for rep in range(-1, a.reps):                                      # rep -1: warm-up, not counted
            t0 = time.perf_counter()
            r = subprocess.run([tool, "-t", str(a.threads), "-o", out, fa, bam], capture_output=True, text=True, check=True)
            wall = time.perf_counter() - t0
            st = json.loads(r.stderr.strip().splitlines()[-1])
            if rep < 0:
                continue
            print(json.dumps({"what": "bm2_multiplemetrics", "input": kind, "rep": rep, "gpu": gpu, "threads": a.threads, "wall_s": wall,
                              "records_per_s": st["records"] / wall,
                              **{k: st[k] for k in ("records", "counted_records", "aligned_bases", "pairs", "windows", "in_bytes", "inflate_s", "add_s",
                                                    "finish_s", "device_bytes")}}), flush=True)

    # ---- bm2_mm_add alone on one window of each input
    from __graft_entry__ import load_package
    import multiplemetrics_util as mu
    capi = load_package().capi
    ref = mu.Ref.read(fa)
    hb, hc = mu.hole_arrays(ref)
    pac = np.fromfile(fa + ".pac", np.uint8)[:(ref.l_pac + 3) // 4]
    ctx = capi.Context(0)
    for kind, bam in bams.items():
        data, starts = window_of(bam, a.window_mb << 20)
        for rep in range(6):
            ctx.mm_set(ref.off, ref.lens, ref.l_pac, pac, hb[:2 * len(ref.holes)], hc)
            ctx.mm_add(data, starts)
            s = ctx.mm_finish()
            bases = int(s["counts"][:, 13].sum())                          # MM_ALIGNED_BASES
            if rep:
                print(json.dumps({"what": "mm_add", "input": kind, "rep": rep, "gpu": gpu, "window_bytes": len(data), "records": len(starts),
                                  "aligned_bases": bases, "add_ms": s["add_ms"], "aligned_bases_per_s": bases / (s["add_ms"] / 1e3)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

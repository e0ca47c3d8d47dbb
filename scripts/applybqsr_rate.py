"""What bm2_applybqsr costs: three runs at -t 16 on the marked BAM and recalibration table of scripts/bqsr_rate.py's input (wall time,
records/s, bases/s and the stderr JSON's inflate_s, apply_s and bgzf_s), and bm2_bqsr_apply alone on one window of those records (CUDA
events, bases/s).  Prints JSON lines, with the card's name and power limit.

    python scripts/applybqsr_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [--reps 3] [--window-mb 256]

The BAM and table come from `bm2_mem --recal-file` on bqsr_rate.py's reads and known sites (run that script first, or this one makes the
same inputs through it)."""
import argparse, json, os, subprocess, sys, tempfile, time
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
    table, md = os.path.join(work, "applybqsr_rate.recal.txt"), os.path.join(work, "applybqsr_rate.md.bam")
    mem = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    subprocess.run([mem, "--recal-file", table, "--known-sites", vcf, "-R", r"@RG\tID:g1\tSM:s\tPU:fc.1", "-t", str(a.threads), "-K", "30000000",
                    "-o", md, fa, p1, p2], check=True, capture_output=True)
    print(json.dumps({"progress": "inputs ready", "bam_bytes": os.path.getsize(md)}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_applybqsr")
    out = os.path.join(work, "applybqsr_rate.out.bam")
    bases = None
    for rep in range(-1, a.reps):                                          # rep -1: warm-up, not counted
        t0 = time.perf_counter()
        r = subprocess.run([tool, "--bqsr-recal-file", table, "-t", str(a.threads), "-o", out, md], capture_output=True, text=True, check=True)
        wall = time.perf_counter() - t0
        st = json.loads(r.stderr.strip().splitlines()[-1])
        if bases is None:
            import bam_util as bu
            raw = bu.inflate(open(md, "rb").read())
            _, _, used = bu.parse_header(raw)
            body = raw[used:]
            recs = bu.records(body)
            bases = sum(int.from_bytes(rc[20:24], "little") for _, rc in recs)
        if rep < 0:
            continue
        print(json.dumps({"what": "bm2_applybqsr", "rep": rep, "gpu": gpu, "threads": a.threads, "records": st["records"], "bases": bases,
                          "wall_s": wall, "records_per_s": st["records"] / wall, "bases_per_s": bases / wall,
                          **{k: st[k] for k in ("inflate_s", "apply_s", "bgzf_s", "windows", "in_bytes", "out_bytes", "recal_bases")}}), flush=True)

    # ---- bm2_bqsr_apply alone on one window (the first --window-mb of records), CUDA events
    from __graft_entry__ import load_package
    import applybqsr_util as aq
    capi = load_package().capi
    limit = a.window_mb << 20
    n = 0
    while n < len(recs) and recs[n][0] + len(recs[n][1]) <= limit:
        n += 1
    win = body[:recs[n - 1][0] + len(recs[n - 1][1])]
    starts = np.array([s for s, _ in recs[:n]], np.int64)
    wbases = sum(int.from_bytes(rc[20:24], "little") for _, rc in recs[:n])
    tabs = aq.dense(open(table).read())
    text = bu.parse_header(raw)[0]
    ids, tab = aq.header_map(text, tabs[0])
    ctx = capi.Context(0)
    for rep in range(4):
        ctx.bqsr_apply_set(tabs[1], tabs[2], tabs[3], ids, tab)
        ctx.bqsr_apply(win, starts)
        s = ctx.bqsr_apply_stats()
        if rep:
            print(json.dumps({"what": "bqsr_apply", "rep": rep, "gpu": gpu, "records": n, "bases": wbases, "apply_ms": s["apply_ms"],
                              "bgzf_ms": s["bgzf_ms"], "apply_bases_per_s": wbases / (s["apply_ms"] / 1e3)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

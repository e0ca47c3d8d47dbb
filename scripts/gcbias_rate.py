"""What GC bias costs bm2_multiplemetrics.  Prints JSON lines, each with the card's name and power limit read in the same call.

    python scripts/gcbias_rate.py [--gbp 3.1] [--n-bp 150e6] [--scans 5] [--pairs 1000000] [--ref-mbp 50] [--threads 16] [--reps 3]
                                  [--baseline PATH]

  scan   the reference scan alone (bm2_mm_gc_set, CUDA events) on an index_build.make_big_reference genome with N runs planted as
         scripts/index_rate.py plants them (runs of 1-100 kbp, about --n-bp in all), given as .amb holes: the device time of each call
         after a warm-up, windows/s, and the fraction of the HBM bound (the packed bases and the hole bitset read once, at 3.35 TB/s).
  tool   bm2_multiplemetrics -t 16 on the sorted BAM of `bm2_mem --markdup` over scripts/bqsr_rate.py's reads, --reps runs after a warm-up,
         alternating: the default programs with --baseline (another build of the tool, e.g. the parent commit's), the default programs,
         and all three programs; wall time, add_s, gc_scan_s and gc_add_s, and whether the default files equal --baseline's."""
import argparse, json, os, subprocess, sys, tempfile, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_name():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def big_reference(gbp, n_bp, seed=1):
    """(contig offsets, lengths, l_pac, packed bases, holes [beg, end) pairs, hole letters) of a make_big_reference genome with N runs."""
    import torch
    from __graft_entry__ import load_package
    load_package()
    from bwa_mem2_b200 import index_build as ib
    total = int(gbp * 1e9)
    contigs = ib.make_big_reference(total, seed=seed, device="cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(seed + 1)
    lens = [len(c) for _, c in contigs]
    off = np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int64)
    runs = []
    for (name, c), o in zip(contigs, off):
        k = max(1, int(n_bp * len(c) / total) // 50000)
        starts = torch.randint(0, len(c), (k,), device="cuda", generator=g).tolist()
        ln = torch.randint(1, 100000, (k,), device="cuda", generator=g).tolist()
        runs += [(int(o) + a, int(o) + min(a + L, len(c))) for a, L in zip(starts, ln)]
    runs.sort()
    holes = []
    for a, b in runs:                                                # merged: sorted and disjoint
        if holes and a <= holes[-1][1]:
            holes[-1][1] = max(holes[-1][1], b)
        else:
            holes.append([a, b])
    l_pac = int(sum(lens))
    flat = torch.cat([c for _, c in contigs])
    del contigs
    flat = torch.cat([flat, torch.zeros((-l_pac) % 4, dtype=torch.uint8, device="cuda")]).view(-1, 4)
    pac = (flat[:, 0] << 6 | flat[:, 1] << 4 | flat[:, 2] << 2 | flat[:, 3]).cpu().numpy()
    del flat
    torch.cuda.empty_cache()
    h = np.array(holes, np.int64).reshape(-1)
    return off, np.array(lens, np.int32), l_pac, pac, h, b"N" * len(holes)


def scan(a, gpu):
    from __graft_entry__ import load_package
    capi = load_package().capi
    off, lens, l_pac, pac, h, hc = big_reference(a.gbp, a.n_bp)
    ctx = capi.Context(0)
    ctx.mm_set(off, lens, l_pac, pac, h, hc)
    hole_bp = int((h[1::2] - h[0::2]).sum())
    bound_bytes = (l_pac + 3) // 4 + ((l_pac + 127) // 128) * 16
    for rep in range(a.scans + 1):                                   # rep 0: warm-up, not printed
        ctx.mm_gc_set()
        d = ctx.mm_gc_finish()
        if rep:
            s = d["scan_ms"] / 1e3
            print(json.dumps({"what": "gc_scan", "rep": rep, "gpu": gpu, "l_pac": l_pac, "contigs": len(lens), "holes": len(hc), "hole_bp": hole_bp,
                              "windows": int(d["windows"].sum()), "scan_ms": d["scan_ms"], "windows_per_s": int(d["windows"].sum()) / s,
                              "hbm_bound_ms": bound_bytes / 3.35e12 * 1e3, "pct_of_hbm_bound": bound_bytes / 3.35e12 / s * 100}), flush=True)
    ctx.close()


def tool(a, gpu):
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa, vcf = os.path.join(work, "ref.fa"), os.path.join(work, "bqsr_rate_30.vcf")
    p1, p2 = os.path.join(work, "markdup_rate_1.fq"), os.path.join(work, "markdup_rate_2.fq")
    if not all(os.path.exists(p) for p in (vcf, p2)):                   # bqsr_rate.py's inputs, made by its own code (one rep)
        subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bqsr_rate.py"), "--pairs", str(a.pairs), "--ref-mbp", str(a.ref_mbp),
                        "--reps", "1"], check=True, stdout=subprocess.DEVNULL)
    bam = os.path.join(work, "gcbias_rate.markdup.bam")
    if not os.path.exists(bam):
        subprocess.run([os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem"), "--markdup", "-R", r"@RG\tID:g1\tSM:s", "-t", str(a.threads), "-K", "30000000",
                        "-o", bam, fa, p1, p2], check=True, capture_output=True)
    here = os.path.join(ROOT, "bwa-mem2_b200", "bm2_multiplemetrics")
    runs = [("baseline", a.baseline, [])] if a.baseline else []
    runs += [("default", here, []), ("all", here, ["--program", "CollectAlignmentSummaryMetrics", "--program", "CollectInsertSizeMetrics",
                                                   "--program", "CollectGcBiasMetrics"])]
    for rep in range(-1, a.reps):                                      # rep -1: warm-up, not printed
        bodies = {}
        for name, exe, progs in runs:
            out = os.path.join(work, "gcbias_rate_" + name)
            t0 = time.perf_counter()
            r = subprocess.run([exe, "-t", str(a.threads)] + progs + ["-o", out, fa, bam], capture_output=True, text=True, check=True)
            wall = time.perf_counter() - t0
            st = json.loads(r.stderr.strip().splitlines()[-1])
            bodies[name] = tuple(open(out + s).read().split("\n", 2)[2] for s in (".alignment_summary_metrics", ".insert_size_metrics"))
            if rep >= 0:
                print(json.dumps({"what": "bm2_multiplemetrics", "run": name, "rep": rep, "gpu": gpu, "threads": a.threads, "wall_s": wall,
                                  **{k: st[k] for k in ("records", "windows", "inflate_s", "add_s", "finish_s", "device_bytes") if k in st},
                                  **{k: st[k] for k in ("gc_windows", "gc_read_starts", "gc_scan_s", "gc_add_s") if k in st}}), flush=True)
        if rep >= 0:
            print(json.dumps({"what": "default_files_equal", "rep": rep, "baseline": bodies.get("baseline") == bodies["default"] if a.baseline else None,
                              "all_programs": bodies["all"] == bodies["default"]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=3.1)
    ap.add_argument("--n-bp", type=float, default=150e6)
    ap.add_argument("--scans", type=int, default=5)
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--baseline", default=None, help="another bm2_multiplemetrics to compare the default run with")
    ap.add_argument("--only", choices=("scan", "tool"), default=None)
    a = ap.parse_args()
    gpu = gpu_name()
    if a.only != "tool":
        scan(a, gpu)
    if a.only != "scan":
        tool(a, gpu)


if __name__ == "__main__":
    main()

"""What duplicate marking costs: bm2_mem's steady-state reads/s and wall time with --sort and with --sort --markdup, and the same pair with
--sort-mem 256M (spilled runs), alternating, in the same call, with the stderr JSON's markdup_s, dup_sig_bytes and duplicate counts; and
bm2_dup_resolve alone on random entries (CUDA events, entries/s).  Prints JSON lines, with the card's name and power limit.

    python scripts/markdup_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--reps 3] [--dup-frac 0.1] [--entries 8000000]

The inputs are scripts/sort_rate.py's (bench.py's pipeline genome and 2x151 bp pairs, Illumina-like qualities), plus a --dup-frac share of the
pairs copied once under new names with new qualities: planted duplicates.  reads/s is bench.py's steady state; the resolve and the merge run
after the last chunk, so the whole-run time (wall_s) is reported too."""
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
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dup-frac", type=float, default=0.1)
    ap.add_argument("--entries", type=int, default=8_000_000)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    from bam_rate import steady, write_fastq
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    p1, p2 = os.path.join(work, "markdup_rate_1.fq"), os.path.join(work, "markdup_rate_2.fq")
    if not os.path.exists(p2):
        rng = np.random.default_rng(78)
        n = len(reads) // 2
        dup = np.sort(rng.choice(n, int(n * a.dup_frac), replace=False))
        pick = np.concatenate([np.arange(n), dup])                     # each planted copy follows the originals, new qualities
        rd = np.stack([reads[0::2][pick], reads[1::2][pick]], 1).reshape(-1, reads.shape[1])
        quals = bam_inputs.illumina_quals(len(rd), rd.shape[1], np.random.default_rng(77))
        write_fastq(p1, rd[0::2], quals[0::2], 1); write_fastq(p2, rd[1::2], quals[1::2], 2)
    print(json.dumps({"progress": "inputs ready", "pairs": len(reads) // 2, "dup_frac": a.dup_frac}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    kinds = {"sort": ["--sort"], "markdup": ["--sort", "--markdup"], "sort_256M": ["--sort", "--sort-mem", "256M"],
             "markdup_256M": ["--sort", "--markdup", "--sort-mem", "256M"]}
    outs = {k: os.path.join(work, f"markdup_rate_{k}.bam") for k in kinds}
    res = {k: [] for k in kinds}
    walls = {k: [] for k in kinds}
    for rep in range(-1, a.reps):                    # rep -1: warm-up, not counted
        for kind, flags in kinds.items():
            t0 = time.perf_counter()
            r = subprocess.run([tool] + flags + ["-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o", outs[kind], fa, p1, p2],
                               capture_output=True, text=True, check=True)
            wall = time.perf_counter() - t0
            st = json.loads(r.stderr.strip().splitlines()[-1])
            if rep < 0:
                continue
            row = {"what": "bm2_mem", "out": kind, "rep": rep, "gpu": gpu, "reads": st["reads"], "steady_reads_per_s": steady(st), "loop_s": st["loop_s"],
                   "wall_s": wall}
            row.update({k: st[k] for k in ("sort_runs", "spill_bytes", "sort_s", "merge_s", "markdup_s", "dup_templates", "dup_pair_templates",
                                           "dup_fragment_templates", "dup_records", "dup_sig_runs", "dup_sig_bytes") if k in st})
            res[kind].append(row["steady_reads_per_s"]); walls[kind].append(wall)
            print(json.dumps(row), flush=True)
    print(json.dumps({"what": "summary", "gpu": gpu, **{k + "_mean": float(np.mean(v)) for k, v in res.items()},
                      **{k + "_wall_mean": float(np.mean(v)) for k, v in walls.items()},
                      "spread": max(max(v) - min(v) for v in res.values())}), flush=True)

    # ---- bm2_dup_resolve alone: entries of one space, piles of a few members, CUDA events
    from __graft_entry__ import load_package
    capi = load_package().capi
    ctx = capi.Context(0)
    rng = np.random.default_rng(5)
    n = a.entries
    e = np.zeros(n, capi.DUP_ENTRY_DT)
    ends = (rng.integers(0, 25, n, dtype=np.uint64) << np.uint64(34)) | ((rng.integers(0, 50_000_000, n // 2 + 1, dtype=np.uint64)[rng.integers(0, n // 2 + 1, n)]
                                                                          + np.uint64(1 << 32)) << np.uint64(1))
    e["k1"] = ends; e["k2"] = ends + np.uint64(600); e["tid"] = rng.permutation(2 * n)[:n]; e["score"] = rng.integers(0, 32767, n); e["kind"] = 0
    ctx.dup_resolve(e[:1000])                                           # warm-up
    for resolve in (True, False):
        ms = [ctx.dup_resolve(e, resolve)[1] for _ in range(3)]
        print(json.dumps({"what": "resolve_entry" if resolve else "sort_entry", "gpu": gpu, "entries": n, "device_ms": ms,
                          "entries_per_s": n / (min(ms) / 1e3)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

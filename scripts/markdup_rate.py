"""What duplicate marking costs: bm2_mem's steady-state reads/s and wall time with --sort and with --sort --markdup, and the same pair with
--sort-mem 256M (spilled runs), alternating, in the same call, with the stderr JSON's markdup_s, dup_sig_bytes and duplicate counts; and
bm2_dup_resolve alone on random entries (CUDA events, entries/s).  Prints JSON lines, with the card's name and power limit.

    python scripts/markdup_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--reps 3] [--dup-frac 0.1] [--entries 8000000]
                                   [--metrics]

--metrics measures the optical pass instead: --markdup against --markdup --markdup-metrics, alternating, on the same pairs under 7-field
Illumina names where half of the planted copies sit within 100 pixels of their original on its tile (optical duplicates) and the others
elsewhere; then bm2_dup_resolve against bm2_dup_resolve_ex on --entries located pair entries, and on a set that also holds a dense group of
50 000 members at one spot.

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
    ap.add_argument("--metrics", action="store_true")
    a = ap.parse_args()
    if a.metrics:
        return metrics_main(a)
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


def write_named_fastq(path, reads, quals, names, mate):
    with open(path, "wb") as f:
        for i in range(0, len(reads), 100_000):
            f.write(b"".join(b"@%s/%d\n" % (names[k], mate) + bytes(b"ACGTN"[c] for c in reads[k]) + b"\n+\n" + bytes(quals[k]) + b"\n"
                             for k in range(i, min(len(reads), i + 100_000))))


def metrics_main(a):
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    from bam_rate import steady
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    p1, p2 = os.path.join(work, "markdup_rate_opt_1.fq"), os.path.join(work, "markdup_rate_opt_2.fq")
    if not os.path.exists(p2):
        rng = np.random.default_rng(78)
        n = len(reads) // 2
        dup = np.sort(rng.choice(n, int(n * a.dup_frac), replace=False))
        pick = np.concatenate([np.arange(n), dup])
        rd = np.stack([reads[0::2][pick], reads[1::2][pick]], 1).reshape(-1, reads.shape[1])
        quals = bam_inputs.illumina_quals(len(rd), rd.shape[1], np.random.default_rng(77))
        tile, x, y = 1101 + rng.integers(0, 24, n), rng.integers(1000, 31000, n), rng.integers(1000, 31000, n)
        near = rng.random(len(dup)) < 0.5                            # half of the copies: optical, within 100 pixels on the original's tile
        ct = np.where(near, tile[dup], 1101 + rng.integers(0, 24, len(dup)))
        cx = np.where(near, x[dup] + rng.integers(-100, 101, len(dup)), rng.integers(1000, 31000, len(dup)))
        cy = np.where(near, y[dup] + rng.integers(-100, 101, len(dup)), rng.integers(1000, 31000, len(dup)))
        T, X, Y = np.concatenate([tile, ct]), np.concatenate([x, cx]), np.concatenate([y, cy])
        names = [b"A00123:8:HXXXXDSXX:1:%d:%d:%d" % (T[k], X[k], Y[k]) for k in range(len(T))]
        seen = {}
        for k, nm in enumerate(names):                                  # unique names: a clash gets the next y
            while nm in seen:
                Y[k] += 1
                nm = b"A00123:8:HXXXXDSXX:1:%d:%d:%d" % (T[k], X[k], Y[k])
            seen[nm] = k; names[k] = nm
        write_named_fastq(p1, rd[0::2], quals[0::2], names, 1); write_named_fastq(p2, rd[1::2], quals[1::2], names, 2)
    print(json.dumps({"progress": "inputs ready", "pairs": len(reads) // 2, "dup_frac": a.dup_frac}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    met = os.path.join(work, "markdup_rate_opt.metrics.txt")
    kinds = {"markdup": ["--markdup"], "markdup_metrics": ["--markdup", "--markdup-metrics", met]}
    out = os.path.join(work, "markdup_rate_opt.bam")
    res, walls, mds = {k: [] for k in kinds}, {k: [] for k in kinds}, {k: [] for k in kinds}
    for rep in range(-1, a.reps):                    # rep -1: warm-up, not counted
        for kind, flags in kinds.items():
            t0 = time.perf_counter()
            r = subprocess.run([tool] + flags + ["-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o", out, fa, p1, p2],
                               capture_output=True, text=True, check=True)
            wall = time.perf_counter() - t0
            st = json.loads(r.stderr.strip().splitlines()[-1])
            if rep < 0:
                continue
            row = {"what": "bm2_mem", "out": kind, "rep": rep, "gpu": gpu, "reads": st["reads"], "steady_reads_per_s": steady(st), "loop_s": st["loop_s"],
                   "wall_s": wall}
            row.update({k: st[k] for k in ("markdup_s", "dup_pair_templates", "dup_fragment_templates", "dup_records", "dup_optical_pairs") if k in st})
            res[kind].append(row["steady_reads_per_s"]); walls[kind].append(wall); mds[kind].append(st["markdup_s"])
            print(json.dumps(row), flush=True)
    print(json.dumps({"what": "summary", "gpu": gpu, **{k + "_mean": float(np.mean(v)) for k, v in res.items()},
                      **{k + "_wall_mean": float(np.mean(v)) for k, v in walls.items()}, **{k + "_markdup_s_mean": float(np.mean(v)) for k, v in mds.items()},
                      "spread": max(max(v) - min(v) for v in res.values())}), flush=True)
    print(json.dumps({"what": "metrics_file", "text": open(met).read().split("\n")[3:6]}), flush=True)

    # ---- bm2_dup_resolve against bm2_dup_resolve_ex: located pair entries, piles of a few members, 10 % of them within 100 pixels
    from __graft_entry__ import load_package
    capi = load_package().capi
    ctx = capi.Context(0)
    rng = np.random.default_rng(5)
    n = a.entries
    e = np.zeros(n, capi.DUP_LOC_ENTRY_DT)
    ends = (rng.integers(0, 25, n, dtype=np.uint64) << np.uint64(34)) | ((rng.integers(0, 50_000_000, n // 2 + 1, dtype=np.uint64)[rng.integers(0, n // 2 + 1, n)]
                                                                          + np.uint64(1 << 32)) << np.uint64(1))
    e["k1"] = ends; e["k2"] = ends + np.uint64(600); e["tid"] = rng.permutation(2 * n)[:n]; e["score"] = rng.integers(0, 32767, n); e["kind"] = 0
    e["tile"] = 1101 + rng.integers(0, 2, n); e["x"] = rng.integers(0, 1000, n); e["y"] = rng.integers(0, 1000, n); e["loc"] = 1 + 2 * rng.integers(0, 2, n)
    dense = e.copy()
    m = 50_000
    dense["k1"][:m] = dense["k1"][0]; dense["k2"][:m] = dense["k2"][0]; dense["tile"][:m] = 2202
    dense["x"][:m] = 5000 + rng.integers(0, 50, m); dense["y"][:m] = 5000 + rng.integers(0, 50, m)
    plain_e = lambda x: np.array(x[list(capi.DUP_ENTRY_DT.names)].tolist(), capi.DUP_ENTRY_DT)
    ctx.dup_resolve(plain_e(e[:1000])); ctx.dup_resolve_ex(e[:1000])     # warm-up
    for name, x in (("located", e), ("dense_group", dense)):
        px = plain_e(x)
        for rep in range(3):
            d0, ms0 = ctx.dup_resolve(px)
            d1, opt, ms1 = ctx.dup_resolve_ex(x, 100)
            assert np.array_equal(d0, d1)
            print(json.dumps({"what": "resolve", "set": name, "rep": rep, "gpu": gpu, "entries": n, "duplicates": len(d0), "optical": int(opt),
                              "resolve_ms": ms0, "resolve_ex_ms": ms1}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

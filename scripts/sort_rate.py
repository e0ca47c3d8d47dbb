"""What a coordinate-sorted BAM costs: bm2_mem's steady-state reads/s with --bam, with --sort (the default --sort-mem: one run) and with
--sort --sort-mem 256M (spilled runs and a real merge), alternating, in the same call, with the stderr JSON's sort_s, merge_s and
spill_bytes; and bm2_bam_sort_compress alone on the same records (CUDA events, GB/s of input).  Prints JSON lines, with the card's name and
power limit.

    python scripts/sort_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--reps 3] [--piece-mb 256]

The inputs are scripts/bam_rate.py's: bench.py's pipeline genome and 2x151 bp pairs, qualities from tests/bam_inputs.py's Illumina-like walk.
reads/s is bench.py's steady state (reads of the chunks after the first over the time between their ends); the merge runs after the last
chunk, so the whole-run time (wall_s) is reported too."""
import argparse, json, os, struct, subprocess, sys, tempfile, time
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
    ap.add_argument("--piece-mb", type=int, default=256)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    import bam_util as bu
    from bam_rate import steady, write_fastq
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    p1, p2 = os.path.join(work, "bam_rate_1.fq"), os.path.join(work, "bam_rate_2.fq")
    if not os.path.exists(p2):
        quals = bam_inputs.illumina_quals(len(reads), reads.shape[1], np.random.default_rng(77))
        write_fastq(p1, reads[0::2], quals[0::2], 1); write_fastq(p2, reads[1::2], quals[1::2], 2)
    print(json.dumps({"progress": "inputs ready", "pairs": len(reads) // 2}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    kinds = {"bam": ["--bam"], "sort": ["--sort"], "sort_256M": ["--sort", "--sort-mem", "256M"]}
    outs = {k: os.path.join(work, f"sort_rate_{k}.bam") for k in kinds}
    res = {k: [] for k in kinds}
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
            row.update({k: st[k] for k in ("sort_runs", "spill_bytes", "sort_s", "merge_s", "merge_windows", "index_s") if k in st})
            res[kind].append(row["steady_reads_per_s"])
            print(json.dumps(row), flush=True)
    print(json.dumps({"what": "summary", "gpu": gpu, **{k + "_mean": float(np.mean(v)) for k, v in res.items()},
                      "spread": max(max(v) - min(v) for v in res.values())}), flush=True)
    def records_part(path):                          # the members after the header's (the @PG line carries the command line)
        ms = bu.members(open(path, "rb").read())
        _, _, used = bu.parse_header(b"".join(r for _, r in ms))
        at, k = 0, 0
        while at < used:
            at += len(ms[k][1]); k += 1
        return b"".join(m for m, _ in ms[k:])
    same = records_part(outs["sort"]) == records_part(outs["sort_256M"])
    print(json.dumps({"what": "one_run_equals_spilled_runs", "same_record_bytes": same}), flush=True)

    # ---- bm2_bam_sort_compress alone, on the --bam run's records, in pieces of piece_mb
    raw = bu.inflate(open(outs["bam"], "rb").read())
    _, _, used = bu.parse_header(raw)
    body = raw[used:]
    starts, at = [], 0
    while at < len(body):
        starts.append(at); at += 4 + struct.unpack_from("<i", body, at)[0]
    sa = np.array(starts, np.int64)
    from __graft_entry__ import load_package
    capi = load_package().capi
    ctx = capi.Context(0)
    piece = a.piece_mb << 20
    pieces = []
    for lo in range(0, len(body), piece):
        i0, i1 = np.searchsorted(sa, lo), np.searchsorted(sa, min(len(body), lo + piece))
        if i1 > i0:
            b0, b1 = int(sa[i0]), int(sa[i1]) if i1 < len(sa) else len(body)
            pieces.append((b0, b1, sa[i0:i1] - b0))
    for b0, b1, st in pieces:                                       # warm-up
        ctx.bam_sort_compress(body[b0:b1], st)
    tot = {"keys": 0.0, "sort": 0.0, "gather": 0.0, "bgzf": 0.0}
    n_in = 0
    for _ in range(2):
        for b0, b1, st in pieces:
            ms = ctx.bam_sort_compress(body[b0:b1], st)["ms"]
            for k in tot:
                tot[k] += ms[k]
            n_in += b1 - b0
    ctx.close()
    dev_s = sum(tot.values()) / 1e3
    print(json.dumps({"what": "sort_entry", "gpu": gpu, "input_bytes": n_in, "piece_bytes": piece, "device_s": dev_s, "GBps": n_in / dev_s / 1e9,
                      "stage_s": {k: v / 1e3 for k, v in tot.items()},
                      "sort_without_bgzf_GBps": n_in / ((tot["keys"] + tot["sort"] + tot["gather"]) / 1e3) / 1e9}), flush=True)


if __name__ == "__main__":
    main()

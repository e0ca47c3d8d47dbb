"""What the recalibration table costs: bm2_mem's steady-state reads/s and wall time with --markdup and with --markdup --recal-file,
alternating, in the same call, with the stderr JSON's bqsr_s, bqsr_bases and known_sites_s; and bm2_bqsr_count alone on one run's records
(CUDA events, bases/s).  Prints JSON lines, with the card's name and power limit.

    python scripts/bqsr_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--reps 3] [--site-every 30]

The reads are scripts/markdup_rate.py's (bench.py's pipeline genome and 2x151 bp pairs, Illumina-like qualities, 10 % planted duplicates);
the known sites are a synthetic VCF of single- and multi-base records about one per --site-every bp, dbSNP's density."""
import argparse, json, os, subprocess, sys, tempfile, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def write_vcf(path, ref, every, rng):
    with open(path, "w") as f:
        f.write("##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n")
        for rid, (name, ln) in enumerate(zip(ref.names, ref.lens)):
            pos = np.unique(rng.integers(1, ln - 5, ln // every))
            n = rng.choice([1, 1, 1, 1, 2, 3], len(pos))
            g = ref.off[rid] + pos - 1
            f.write("".join("%s\t%d\t.\t%s\t%s\t.\tPASS\t.\n" % (name, p, "".join("ACGT"[c] for c in ref.codes[x:x + k]), "ACGT"[(ref.codes[x] + 1) & 3])
                            for p, x, k in zip(pos.tolist(), g.tolist(), n.tolist())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--site-every", type=int, default=30)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    import bqsr_util as bq
    from bam_rate import steady, write_fastq
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    p1, p2 = os.path.join(work, "markdup_rate_1.fq"), os.path.join(work, "markdup_rate_2.fq")
    if not os.path.exists(p2):                                          # markdup_rate.py's inputs
        rng = np.random.default_rng(78)
        n = len(reads) // 2
        dup = np.sort(rng.choice(n, int(n * 0.1), replace=False))
        pick = np.concatenate([np.arange(n), dup])
        rd = np.stack([reads[0::2][pick], reads[1::2][pick]], 1).reshape(-1, reads.shape[1])
        quals = bam_inputs.illumina_quals(len(rd), rd.shape[1], np.random.default_rng(77))
        write_fastq(p1, rd[0::2], quals[0::2], 1); write_fastq(p2, rd[1::2], quals[1::2], 2)
    ref = bq.Ref(fa)
    vcf = os.path.join(work, f"bqsr_rate_{a.site_every}.vcf")
    if not os.path.exists(vcf):
        write_vcf(vcf, ref, a.site_every, np.random.default_rng(79))
    print(json.dumps({"progress": "inputs ready", "pairs": len(reads) // 2, "vcf_bytes": os.path.getsize(vcf)}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    table = os.path.join(work, "bqsr_rate.recal.txt")
    rg = ["-R", r"@RG\tID:g1\tSM:s\tPU:fc.1"]
    kinds = {"markdup": ["--markdup"], "recal": ["--markdup", "--recal-file", table, "--known-sites", vcf]}
    out = os.path.join(work, "bqsr_rate.bam")
    res, walls = {k: [] for k in kinds}, {k: [] for k in kinds}
    for rep in range(-1, a.reps):                    # rep -1: warm-up, not counted
        for kind, flags in kinds.items():
            t0 = time.perf_counter()
            r = subprocess.run([tool] + flags + rg + ["-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o", out, fa, p1, p2],
                               capture_output=True, text=True, check=True)
            wall = time.perf_counter() - t0
            st = json.loads(r.stderr.strip().splitlines()[-1])
            if rep < 0:
                continue
            row = {"what": "bm2_mem", "out": kind, "rep": rep, "gpu": gpu, "reads": st["reads"], "steady_reads_per_s": steady(st), "loop_s": st["loop_s"],
                   "wall_s": wall}
            row.update({k: st[k] for k in ("sort_s", "markdup_s", "bqsr_s", "bqsr_reads", "bqsr_bases", "known_sites", "known_sites_s") if k in st})
            res[kind].append(row["steady_reads_per_s"]); walls[kind].append(wall)
            print(json.dumps(row), flush=True)
    print(json.dumps({"what": "summary", "gpu": gpu, **{k + "_mean": float(np.mean(v)) for k, v in res.items()},
                      **{k + "_min": float(np.min(v)) for k, v in res.items()}, **{k + "_max": float(np.max(v)) for k, v in res.items()},
                      **{k + "_wall_mean": float(np.mean(v)) for k, v in walls.items()}, **{k + "_wall_min": float(np.min(v)) for k, v in walls.items()},
                      **{k + "_wall_max": float(np.max(v)) for k, v in walls.items()}}), flush=True)

    # ---- bm2_bqsr_count alone on the sorted records of one run (the output BAM), CUDA events
    import bam_util as bu
    from __graft_entry__ import load_package
    capi = load_package().capi
    raw = bu.inflate(open(out, "rb").read())
    _, _, used = bu.parse_header(raw)
    body = raw[used:]
    starts = np.array([s for s, _ in bu.records(body)], np.int64)
    idx = capi.Index(fa)
    ctx = capi.Context(0, index=idx)
    cov, jun = np.zeros(ref.l_pac, bool), np.zeros(ref.l_pac, bool)
    for line in open(vcf):
        if line[0] != "#":
            c, p, _, r_ = line.split("\t")[:4]
            g = ref.off[ref.names.index(c)] + int(p) - 1
            cov[g:g + len(r_)] = True; jun[g:g + len(r_) - 1] = True
    for rep in range(4):
        ctx.bqsr_sites(bq.pack_bits(cov), bq.pack_bits(jun), ref.l_pac, ref.holes, "fc.1")
        ctx.bqsr_count(body, starts)
        t = ctx.bqsr_tables()
        if rep:
            print(json.dumps({"what": "bqsr_count", "rep": rep, "gpu": gpu, "records": len(starts), "bases": t["bases"], "device_ms": t["ms"],
                              "bases_per_s": t["bases"] / (t["ms"] / 1e3)}), flush=True)
    ctx.close(); idx.close()


if __name__ == "__main__":
    main()

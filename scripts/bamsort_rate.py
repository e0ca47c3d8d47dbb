"""What bm2_sort costs: wall time and the stderr JSON's device stage times of `bm2_sort` (coordinate) and `bm2_sort -n` (read name) on the
unsorted (`bm2_mem --bam`, input order) BAM of bqsr_rate.py's 1.1 M pairs (bam2fq_rate.py's uniquely named FASTQ) and on a shuffled copy of
it, at the default --sort-mem and at one that forces several runs, after a warm-up.  Then the two device sorts alone on one run of the
shuffled records (CUDA events): the name sort's merge-sort stage against the coordinate radix sort of the same run, with the bytes each moves.
Prints JSON lines, with the card's name and power limit.

    python scripts/bamsort_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--reps 2] [--small-mem 256M]"""
import argparse, json, math, os, struct, subprocess, sys, tempfile, time, zlib
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def bgzf_fast(data: bytes) -> bytes:
    """BGZF members of 65280 bytes at zlib level 1 (the input only; its compression does not matter) and the EOF block."""
    out = []
    for at in range(0, len(data), 65280):
        blk = data[at:at + 65280]
        c = zlib.compressobj(1, zlib.DEFLATED, -15)
        d = c.compress(blk) + c.flush()
        out.append(b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", len(d) + 25) + d + struct.pack("<II", zlib.crc32(blk), len(blk)))
    return b"".join(out) + bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--small-mem", default="256M")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    import bam_util as bu
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    # bam2fq_rate.py's FASTQ: bqsr_rate.py's reads, 10 % of the pairs twice, and qualities, under unique names
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
    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_sort")
    bams = {"unsorted": os.path.join(work, "bamsort_rate.unsorted.bam"), "shuffled": os.path.join(work, "bamsort_rate.shuffled.bam")}
    subprocess.run([mem, "--bam", "-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o", bams["unsorted"], fa, p1, p2], capture_output=True, check=True)
    raw = bu.inflate(open(bams["unsorted"], "rb").read())
    _, _, used = bu.parse_header(raw)
    recs = [r for _, r in bu.records(raw[used:])]
    order = np.random.default_rng(79).permutation(len(recs))
    shuffled = [recs[i] for i in order]
    with open(bams["shuffled"], "wb") as f:
        f.write(bgzf_fast(raw[:used] + b"".join(shuffled)))
    print(json.dumps({"progress": "inputs ready", "gpu": gpu, "records": len(recs), "record_bytes": len(raw) - used,
                      **{k: os.path.getsize(v) for k, v in bams.items()}}), flush=True)
    out = os.path.join(work, "bamsort_rate.out.bam")
    for rep in range(-1, a.reps):                                       # rep -1: warm-up, not counted
        for kind, path in bams.items():
            for by_name in (False, True):
                for sm in (None, a.small_mem):
                    argv = [tool, "-t", str(a.threads)] + (["-n"] if by_name else []) + (["--sort-mem", sm] if sm else []) + ["-o", out, path]
                    t0 = time.perf_counter()
                    r = subprocess.run(argv, capture_output=True, text=True)
                    if r.returncode:
                        sys.exit(r.stderr[-2000:])
                    wall = time.perf_counter() - t0
                    st = json.loads(r.stderr.strip().splitlines()[-1])
                    if rep >= 0:
                        print(json.dumps({"what": "bm2_sort", "bam": kind, "order": "name" if by_name else "coordinate", "sort_mem": sm or "2G",
                                          "rep": rep, "gpu": gpu, "wall_s": wall, **st}), flush=True)

    # ---- the two device sorts alone on one run: the shuffled records, as many as fit in 2 GB
    from __graft_entry__ import load_package
    capi = load_package().capi
    run, total = [], 0
    for rr in shuffled:
        if total + len(rr) > 2 << 30:
            break
        run.append(rr); total += len(rr)
    data = b"".join(run)
    starts = np.cumsum([0] + [len(rr) for rr in run[:-1]]).astype(np.int64)
    n = len(run)
    names = sorted(rr[36:36 + rr[12] - 1] for rr in run)
    common = np.mean([next((i for i, (x, y) in enumerate(zip(names[k], names[k + 1])) if x != y), min(len(names[k]), len(names[k + 1])))
                      for k in range(0, n - 1, max(1, n // 200_000))])
    mean_name = np.mean([len(x) for x in names[::max(1, n // 200_000)]]) + 1
    ctx = capi.Context(0)
    for rep in range(4):
        for which, call in (("coordinate", ctx.bam_sort_compress), ("name", ctx.bam_qname_sort_compress)):
            o = call(data, starts)
            if rep == 0:
                continue
            ms = o["ms"]
            row = {"what": "device_sort", "order": which, "rep": rep, "gpu": gpu, "records": n, "record_bytes": len(data), **{k + "_ms": v for k, v in ms.items()}}
            if which == "name":
                # comparisons of a merge sort: about n log2 n; each loads two 8-byte entries and the names up to their first difference,
                # every load a random 32-byte sector at least
                cmps = n * math.log2(n)
                sectors = cmps * 2 * (1 + math.ceil((common + 1) / 32))
                row.update(comparisons=cmps, mean_name_bytes=mean_name, mean_common_prefix=common, sector_bytes=sectors * 32,
                           sector_bytes_per_s=sectors * 32 / (ms["sort"] / 1e3), share_of_3_35TBps=sectors * 32 / (ms["sort"] / 1e3) / 3.35e12)
            else:
                # LSD radix sort of 8-byte keys and 4-byte ordinals: each pass reads and writes both, over the key's used bits
                row.update(radix_pass_bytes=n * 12 * 2)
            print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

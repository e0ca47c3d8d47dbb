"""What BAM out costs: bm2_mem's steady-state reads/s writing SAM against writing BAM (--bam, BGZF compressed on the GPU), alternating, in
the same call; bm2_bgzf_compress alone in GB/s of input (CUDA events over at least --kernel-gb of the run's uncompressed BAM); and
single-thread host zlib (levels 1 and 6) on the same bytes and the same block cuts, for its rate and its sizes.  Prints JSON lines, with the
card's name and power limit.

    python scripts/bam_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--reps 3] [--kernel-gb 1]

The genome, index and read bases are those of bench.py's pipeline workload (2x151 bp pairs); the qualities come from a seeded Illumina-like
position-dependent Markov walk (tests/bam_inputs.py), since constant qualities would flatter any compressor.  reads/s is bench.py's steady
state (reads of the chunks after the first over the time between their ends)."""
import argparse, json, os, struct, subprocess, sys, tempfile, time, zlib
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def steady(st):
    d, r = st["chunk_done_s"], st["chunk_reads"]
    return sum(r[1:]) / (d[-1] - d[0]) if len(d) > 1 and d[-1] > d[0] else st["reads"] / st["loop_s"]


def write_fastq(path, reads, quals, mate):
    with open(path, "wb") as f:
        for i in range(0, len(reads), 100_000):
            blk = []
            for k in range(i, min(len(reads), i + 100_000)):
                blk.append(b"@A00123:8:HXXXXDSXX:1:%d:%d:%d/%d\n" % (1101 + k // 40000, 1000 + (k * 37) % 30000, 1000 + (k * 91) % 30000, mate) +
                           bytes(b"ACGTN"[c] for c in reads[k]) + b"\n+\n" + bytes(quals[k]) + b"\n")
            f.write(b"".join(blk))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-gb", type=float, default=1.0)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    import bam_util as bu
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    p1, p2 = os.path.join(work, "bam_rate_1.fq"), os.path.join(work, "bam_rate_2.fq")
    if not os.path.exists(p2):
        quals = bam_inputs.illumina_quals(len(reads), reads.shape[1], np.random.default_rng(77))
        write_fastq(p1, reads[0::2], quals[0::2], 1); write_fastq(p2, reads[1::2], quals[1::2], 2)
    print(json.dumps({"progress": "inputs ready", "pairs": len(reads) // 2}), flush=True)

    # ---- bm2_mem: SAM out against --bam, alternating, both to /dev/null so that the file system's speed does not enter; one more --bam run
    # first (not counted) writes the file the kernel and zlib measurements below read
    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    bam_path = os.path.join(work, "out.bam")
    res = {"sam": [], "bam": []}
    for rep in range(-1, a.reps):
        for kind in (("bam",) if rep < 0 else ("sam", "bam")):
            cmd = [tool] + (["--bam"] if kind == "bam" else []) + ["-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o",
                                                                   bam_path if rep < 0 else "/dev/null", fa, p1, p2]
            r = subprocess.run(cmd, capture_output=True, text=True, check=True)
            st = json.loads(r.stderr.strip().splitlines()[-1])
            if rep < 0:
                continue
            row = {"what": "bm2_mem", "out": kind, "rep": rep, "gpu": gpu, "reads": st["reads"], "steady_reads_per_s": steady(st), "loop_s": st["loop_s"],
                   "sam_format_s": st["sam_format_s"], "write_s": st["write_s"], "wait_for_turn_s": st["wait_for_turn_s"]}
            if kind == "bam":
                row.update({k: st[k] for k in ("bam_format_s", "bgzf_s", "bam_bytes", "bgzf_bytes")})
            res[kind].append(row["steady_reads_per_s"])
            print(json.dumps(row), flush=True)
    spread = max(max(v) - min(v) for v in res.values())
    print(json.dumps({"what": "gate", "sam_mean": float(np.mean(res["sam"])), "bam_mean": float(np.mean(res["bam"])), "spread": spread,
                      "bam_not_slower_beyond_spread": float(np.mean(res["sam"]) - np.mean(res["bam"])) <= spread}), flush=True)

    # ---- the run's uncompressed BAM and its record starts
    data = open(bam_path, "rb").read()
    raw = bu.inflate(data)
    _, _, used = bu.parse_header(raw)
    body = raw[used:]
    starts, at = [], 0
    while at < len(body):
        starts.append(at); at += 4 + struct.unpack_from("<i", body, at)[0]
    print(json.dumps({"what": "bam_stream", "uncompressed_bytes": len(body), "records": len(starts), "file_bytes": len(data)}), flush=True)

    # ---- bm2_bgzf_compress alone, in pieces of about one chunk, until kernel_gb of input
    from __graft_entry__ import load_package
    capi = load_package().capi
    ctx = capi.Context(0)
    piece = 32 << 20
    sa = np.array(starts, np.int64)
    pieces = []
    for lo in range(0, len(body), piece):
        i0, i1 = np.searchsorted(sa, lo), np.searchsorted(sa, min(len(body), lo + piece))
        b0, b1 = int(sa[i0]) if i0 < len(sa) else len(body), int(sa[i1]) if i1 < len(sa) else len(body)
        if b1 > b0:
            pieces.append((b0, b1, sa[i0:i1] - b0))
    gpu_size, ms_total, in_total = 0, 0.0, 0
    for b0, b1, cut in pieces:                                          # warm-up and size: every piece once, output checked
        z, ms, _ = ctx.bgzf_compress(body[b0:b1], cut)
        assert bu.inflate(z) == body[b0:b1]
        gpu_size += len(z)
    while in_total < a.kernel_gb * 1e9:
        for b0, b1, cut in pieces:
            _, ms, _ = ctx.bgzf_compress(body[b0:b1], cut)
            ms_total += ms; in_total += b1 - b0
    ctx.close()
    print(json.dumps({"what": "bgzf_kernel", "gpu": gpu, "input_bytes": in_total, "device_s": ms_total / 1e3, "GBps": in_total / (ms_total / 1e3) / 1e9,
                      "output_bytes_once": gpu_size, "ratio": gpu_size / len(body)}), flush=True)

    # ---- host zlib, one thread, the same blocks
    blocks = []
    for b0, b1, cut in pieces:
        s = bu.htslib_cuts(b1 - b0, cut.tolist())
        blocks += [(b0 + x, b0 + y) for x, y in zip(s[:-1], s[1:])]
    for level in (1, 6):
        size, t = 0, 0.0
        for x, y in blocks:
            c = zlib.compressobj(level, zlib.DEFLATED, -15)
            t0 = time.perf_counter(); z = c.compress(body[x:y]) + c.flush(); t += time.perf_counter() - t0
            size += len(z) + 26
        print(json.dumps({"what": "host_zlib_1thread", "level": level, "input_bytes": len(body), "bgzf_bytes": size, "MBps": len(body) / t / 1e6,
                          "gpu_size_over_this": gpu_size / size}), flush=True)


if __name__ == "__main__":
    main()

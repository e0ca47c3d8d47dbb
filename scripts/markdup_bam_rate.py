"""What bm2_markdup costs: scripts/markdup_rate.py's planted pairs (made by scripts/bqsr_rate.py, 1.1 M pairs at its defaults) split into two
lanes of one library, each sorted by `bm2_mem --sort`, then three runs of `bm2_markdup -t 16 l1.bam l2.bam` after a warm-up (wall time,
records/s and the stderr JSON's device times), and bm2_markdup_records plus bm2_markdup_pair alone on one window of the merged records
(CUDA events, each call separately, records/s over their sum).  Prints JSON lines, with the card's name and power limit.

    python scripts/markdup_bam_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [--reps 3] [--window-mb 256]"""
import argparse, json, os, subprocess, sys, tempfile, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def split_fastq(src, dst0, dst1, mate):
    """four-line records, alternately to dst0 and dst1, each renamed A00123:8:HXXXXDSXX:<lane>:<tile>:<x>:<y> from its index k: the
    source's names repeat every 30 000 pairs on a tile, and a coordinate-sorted file needs one pair per name"""
    with open(src, "rb") as f, open(dst0, "wb") as a, open(dst1, "wb") as b:
        k = 0
        while True:
            rec = [f.readline() for _ in range(4)]
            if not rec[0]:
                break
            rec[0] = b"@A00123:8:HXXXXDSXX:%d:%d:%d:%d/%d\n" % (k % 2 + 1, 1101 + k // 900000, 1000 + k % 30000, 1000 + (k // 30000) % 30000, mate)
            (a if k % 2 == 0 else b).write(b"".join(rec))
            k += 1


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
    lanes = []
    for m in (1, 2):                                                     # pair k to lane k % 2 + 1, mate files in step
        split_fastq(os.path.join(work, f"markdup_rate_{m}.fq"), os.path.join(work, f"mdb_l1_{m}.fq"), os.path.join(work, f"mdb_l2_{m}.fq"), m)
    for k in (1, 2):
        out = os.path.join(work, f"markdup_bam_rate.l{k}.bam")
        subprocess.run([mem, "--sort", "-R", rf"@RG\tID:l{k}\tSM:s\tLB:a", "-t", str(a.threads), "-K", "30000000", "-o", out, fa,
                        os.path.join(work, f"mdb_l{k}_1.fq"), os.path.join(work, f"mdb_l{k}_2.fq")], check=True, capture_output=True)
        lanes.append(out)
    print(json.dumps({"progress": "inputs ready", "bytes": [os.path.getsize(p) for p in lanes]}), flush=True)

    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_markdup")
    out, met = os.path.join(work, "markdup_bam_rate.bam"), os.path.join(work, "markdup_bam_rate.txt")
    for rep in range(-1, a.reps):                                          # rep -1: warm-up, not counted
        t0 = time.perf_counter()
        r = subprocess.run([tool, "-t", str(a.threads), "-M", met, "-o", out] + lanes, capture_output=True, text=True, check=True)
        wall = time.perf_counter() - t0
        st = json.loads(r.stderr.strip().splitlines()[-1])
        if rep < 0:
            continue
        print(json.dumps({"what": "bm2_markdup", "rep": rep, "gpu": gpu, "threads": a.threads, "wall_s": wall, "records_per_s": st["records"] / wall,
                          **{k: st[k] for k in ("records", "inputs", "pairs", "fragments", "pending_max", "dup_pair_templates", "dup_fragment_templates",
                                                "dup_optical_pairs", "windows", "in_bytes", "out_bytes", "inflate_s", "sig_s", "pair_s", "resolve_s", "mark_s",
                                                "bgzf_s", "device_bytes", "wall_s")}}), flush=True)

    # ---- bm2_markdup_records and bm2_markdup_pair alone on one window of the merged output's records
    from __graft_entry__ import load_package
    import markdup_bam_util as mb
    capi = load_package().capi
    _, _, recs = mb.read_bam(out)
    data, starts, at = [], [], 0
    for r in recs:
        if at + len(r) > a.window_mb << 20:
            break
        starts.append(at); data.append(r); at += len(r)
    data = b"".join(data)
    ctx = capi.Context(0)
    names = [r[36:36 + r[12] - 1] for r in recs[:len(starts)]]
    for rep in range(6):
        ctx.markdup_set(["l1", "l2"], [1, 1], 2, 0)
        got = ctx.markdup_records(data, np.array(starts, np.int64))
        sel = np.nonzero((got["kind"] == mb.HALF) | (got["kind"] == mb.UNMAPPED_HALF))[0]
        halves, blob = mb.halves_array([(int(got["hash"][i]), int(got["rg"][i]), names[i]) for i in sel])
        part = ctx.markdup_pair(halves, blob)
        rec_ms, pair_ms = ctx.markdup_stats()[:2]
        if rep:
            print(json.dumps({"what": "markdup_records+pair", "rep": rep, "gpu": gpu, "window_bytes": len(data), "records": len(starts),
                              "halves": len(sel), "joined": sum(p >= 0 for p in part), "records_ms": rec_ms, "pair_ms": pair_ms,
                              "records_per_s": len(starts) / ((rec_ms + pair_ms) / 1e3)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()

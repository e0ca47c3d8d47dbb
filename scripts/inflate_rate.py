"""How fast bm2_mem reads compressed input: single-thread host zlib on FASTQ text as BGZF level 6 (the rate one reading thread can inflate),
and bm2_mem's steady-state reads/s on the same pairs as plain files, single-member gzip, BGZF files and BGZF on standard input.  Prints JSON
lines, with the card's name and power limit.

    python scripts/inflate_rate.py [--gb 2] [--pairs 1000000] [--ref-mbp 50] [--threads 16] [-K 30000000] [--baseline DIR [--bench-only]]

--baseline DIR: a built checkout of another commit (the parent); `bench.py --workload fastq2sam` then runs from DIR and from this tree,
alternating, twice each, in the same call (it reads plain files, so the streaming reader must not move it beyond the run-to-run spread).

The genome, index and reads are those of bench.py's pipeline workload; reads/s is bench.py's steady state (reads of the chunks after the
first over the time between their ends, chunk_done_s).  read_s is the time bm2_mem's chunker spent reading and inflating."""
import argparse, gzip, json, os, struct, subprocess, sys, tempfile, time, zlib
from concurrent.futures import ProcessPoolExecutor
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _bgzf_piece(data):
    from test_input_stream_cpu import bgzf
    return bgzf(data, level=6, eof=False)


def bgzf_parallel(data, piece=65280 * 256):
    with ProcessPoolExecutor() as ex:
        return b"".join(ex.map(_bgzf_piece, [data[i:i + piece] for i in range(0, len(data), piece)]))


def steady(st):
    d, r = st["chunk_done_s"], st["chunk_reads"]
    return sum(r[1:]) / (d[-1] - d[0]) if len(d) > 1 and d[-1] > d[0] else st["reads"] / st["loop_s"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--baseline")
    ap.add_argument("--bench-only", action="store_true")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    if a.baseline:
        for rep in range(2):
            for tree in (a.baseline, ROOT):
                r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", "5", "--warmup", "2", "--workload", "fastq2sam"], cwd=tree,
                                   capture_output=True, text=True, check=True)
                v = json.loads(r.stdout.strip().splitlines()[-1])
                print(json.dumps({"what": "bench_fastq2sam", "tree": "baseline" if tree == a.baseline else "this", "rep": rep, "gpu": gpu,
                                  "reads_per_s": v["value"], "sam_identical": v["parity"]["identical"]}), flush=True)
        if a.bench_only:
            return
    import bench
    import scripts.seq_input_rate as sir
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    fq = open(sir.write_shapes(reads, work)["fastq_4line"], "rb").read()

    # ---- host zlib, one thread, member by member (BSIZE)
    text = fq * max(1, int(a.gb * 1e9 / len(fq) + 0.999))
    comp = bgzf_parallel(text)
    host_s, parts, mv, at = 0.0, [], memoryview(comp), 0
    while at < len(comp):
        m = struct.unpack_from("<H", comp, at + 16)[0] + 1
        t0 = time.perf_counter(); parts.append(zlib.decompress(mv[at:at + m], 31)); host_s += time.perf_counter() - t0
        at += m
    print(json.dumps({"what": "host_zlib_1thread", "gpu": gpu, "text_bytes": len(text), "bgzf_bytes": len(comp),
                      "equal": b"".join(parts) == text, "GBps": len(text) / host_s / 1e9}), flush=True)
    del text, comp, parts, mv

    # ---- bm2_mem: the same pairs as plain, gzip, BGZF files and BGZF on standard input
    p1 = os.path.join(work, "ir_1.fq"); p2 = os.path.join(work, "ir_2.fq")
    rec = fq.split(b"\n")
    with open(p1, "wb") as f1, open(p2, "wb") as f2:
        for i in range(0, len(rec) - 1, 8):
            f1.write(b"\n".join(rec[i:i + 4]) + b"\n"); f2.write(b"\n".join(rec[i + 4:i + 8]) + b"\n")
    files = {"plain": (p1, p2)}
    for kind, enc in (("gzip", lambda d: gzip.compress(d, 6, mtime=0)), ("bgzf", bgzf_parallel)):
        files[kind] = tuple(p + "." + kind for p in (p1, p2))
        for src, dst in zip((p1, p2), files[kind]):
            open(dst, "wb").write(enc(open(src, "rb").read()))
    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    base = [tool, "-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o", "/dev/null", fa]
    runs = [("plain", files["plain"], None), ("gzip", files["gzip"], None), ("bgzf", files["bgzf"], None), ("bgzf_stdin", ("-", files["bgzf"][1]), files["bgzf"][0])]
    print(json.dumps({"progress": "files written"}), flush=True)
    for name, paths, stdin in runs:
        r = subprocess.run(base + list(paths), stdin=open(stdin, "rb") if stdin else None, capture_output=True, text=True, check=True)
        st = json.loads(r.stderr.strip().splitlines()[-1])
        print(json.dumps({"what": "bm2_mem", "input": name, "gpu": gpu, "reads": st["reads"], "steady_reads_per_s": steady(st),
                          "loop_s": st["loop_s"], "read_s": st["read_s"], "gzip_members": st["gzip_members"],
                          "input_peak_bytes": st["input_peak_bytes"]}), flush=True)


if __name__ == "__main__":
    main()

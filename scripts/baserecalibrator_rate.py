"""What bm2_baserecalibrator costs: wall, inflate and device time of the tool on bqsr_rate.py's input (1.1 M pairs marked by bm2_mem, a
dbSNP-density VCF) with one read group and with the same records spread over 16 (both sides of the shared/global table threshold),
alternating; bm2_recal_add alone on one 256 MB window (CUDA events, G bases/s) at 1 and 16 covariates; and, with --parent-mem, bm2_mem
--markdup --recal-file of the parent build against this tree's, alternating, to show that the counting kernel's change did not slow bm2_mem.
Prints JSON lines, with the card's name and power limit.

    python scripts/baserecalibrator_rate.py [--pairs 1000000] [--ref-mbp 50] [--threads 16] [--reps 3] [--parent-mem PATH]"""
import argparse, json, os, struct, subprocess, sys, tempfile, time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def read_bam(path):
    """-> (header text, references, records' bytes, their starts)."""
    import bam_util as bu
    raw = bu.inflate(open(path, "rb").read())
    text, refs, used = bu.parse_header(raw)
    body = raw[used:]
    return text, refs, body, np.array([s for s, _ in bu.records(body)], np.int64)


def spread(src, dst, n):
    """src (every record tagged RG:Z:g1 by bm2_mem -R) with record i's value set to g<hex digit of i % n>, the same length, and n @RG lines;
    written as BGZF at zlib level 1."""
    import re, zlib
    import bam_util as bu
    text, refs, body, starts = read_bam(src)
    at = np.array([m.start() for m in re.finditer(re.escape(b"RGZg1\0"), body)], np.int64)
    if len(at) != len(starts) or not np.all(np.searchsorted(starts, at, side="right") - 1 == np.arange(len(starts))):
        raise AssertionError("not one RG:Z:g1 tag per record")
    b = np.frombuffer(body, np.uint8).copy()
    b[at + 4] = np.frombuffer(b"0123456789abcdef", np.uint8)[np.arange(len(at)) % n]
    lines = [l for l in text.split("\n") if l and not l.startswith("@RG")]
    text = "\n".join(lines + ["@RG\tID:g%x\tSM:s\tPU:fc.%02d" % (k, k) for k in range(n)]) + "\n"
    h = b"BAM\1" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for name, ln in refs:
        h += struct.pack("<i", len(name) + 1) + name.encode() + b"\0" + struct.pack("<i", ln)
    data, out = h + b.tobytes(), []
    for o in range(0, len(data), 65280):
        chunk = data[o:o + 65280]
        c = zlib.compressobj(1, zlib.DEFLATED, -15)
        z = c.compress(chunk) + c.flush()
        out.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(z) + 25) + z +
                   struct.pack("<II", zlib.crc32(chunk), len(chunk)))
    with open(dst, "wb") as f:
        f.write(b"".join(out) + bu.EOF_BLOCK)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=1_000_000)
    ap.add_argument("--ref-mbp", type=int, default=50)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("-K", type=int, default=30_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--site-every", type=int, default=30)
    ap.add_argument("--parent-mem", default="")
    a = ap.parse_args()
    t_start = time.perf_counter()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    import bench
    import bam_inputs
    import baserecalibrator_util as br
    import bqsr_util as bq
    from bam_rate import steady, write_fastq
    from bqsr_rate import write_vcf
    work = os.path.join(tempfile.gettempdir(), f"bm2_bench_pipe_{a.ref_mbp}_{a.pairs}")
    fa = bench.prepare_pipeline_inputs(work, a.ref_mbp * 1_000_000, a.pairs, seed=21)
    reads = np.load(os.path.join(work, "reads.npy"))
    p1, p2 = os.path.join(work, "markdup_rate_1.fq"), os.path.join(work, "markdup_rate_2.fq")
    if not os.path.exists(p2):                                          # bqsr_rate.py's inputs
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
    mem = os.path.join(ROOT, "bwa-mem2_b200", "bm2_mem")
    rg = ["-R", r"@RG\tID:g1\tSM:s\tPU:fc.1"]
    marked, table = os.path.join(work, "brc_rate.bam"), os.path.join(work, "brc_rate.mem.txt")
    run = lambda tool, t: subprocess.run([tool, "--markdup", "--recal-file", t, "--known-sites", vcf] + rg +
                                         ["-t", str(a.threads), "-K", str(a.K), "-p", "2", "-o", marked, fa, p1, p2], capture_output=True, text=True, check=True)
    run(mem, table)
    print(json.dumps({"progress": "marked", "s": time.perf_counter() - t_start}), flush=True)
    sixteen = os.path.join(work, "brc_rate16.bam")
    spread(marked, sixteen, 16)
    print(json.dumps({"progress": "spread", "s": time.perf_counter() - t_start}), flush=True)
    print(json.dumps({"progress": "inputs ready", "s": time.perf_counter() - t_start, "pairs": len(reads) // 2, "bam_bytes": os.path.getsize(marked), "vcf_bytes": os.path.getsize(vcf)}),
          flush=True)

    # ---- the tool, one read group and 16, alternating
    tool = os.path.join(ROOT, "bwa-mem2_b200", "bm2_baserecalibrator")
    out = os.path.join(work, "brc_rate.txt")
    for rep in range(-1, a.reps):                    # rep -1: warm-up, not counted
        for n_rg, bam in ((1, marked), (16, sixteen)):
            r = subprocess.run([tool, "-t", str(a.threads), "--known-sites", vcf, "-o", out, fa, bam], capture_output=True, text=True, check=True)
            st = json.loads(r.stderr.strip().splitlines()[-1])
            if n_rg == 1 and open(out).read() != open(table).read():
                raise AssertionError("the one-read-group table differs from bm2_mem --recal-file's")
            if rep >= 0:
                print(json.dumps({"what": "bm2_baserecalibrator", "read_groups": n_rg, "rep": rep, "gpu": gpu,
                                  **{k: st[k] for k in ("records", "counted_bases", "windows", "wall_s", "inflate_s", "recal_s")}}), flush=True)

    # ---- bm2_recal_add alone on one window of about 256 MB, CUDA events
    from __graft_entry__ import load_package
    capi = load_package().capi
    cov, jun = np.zeros(ref.l_pac, bool), np.zeros(ref.l_pac, bool)
    for line in open(vcf):
        if line[0] != "#":
            c, p, _, r_ = line.split("\t")[:4]
            g = ref.off[ref.names.index(c)] + int(p) - 1
            cov[g:g + len(r_)] = True; jun[g:g + len(r_) - 1] = True
    ctx, pac = capi.Context(0), br.pac_of(ref)
    for n_rg, bam in ((1, marked), (16, sixteen)):
        text, _, body, starts = read_bam(bam)
        ids, id_cov, covs = br.read_groups([text])
        k = int(np.searchsorted(np.append(starts[1:], len(body)), 256 << 20, side="right"))
        starts, body = starts[:k], body[:int(np.append(starts[1:], len(body))[k - 1])]
        for rep in range(4):
            ctx.recal_set(ref.off, ref.lens, ref.l_pac, pac, ref.holes, bq.pack_bits(cov), bq.pack_bits(jun), ids, id_cov, len(covs))
            ctx.recal_add(body, np.array(starts, np.int64))
            ts = [ctx.recal_tables(c) for c in range(len(covs))]
            bases, ms = sum(t["bases"] for t in ts), ts[0]["ms"]
            if rep:
                print(json.dumps({"what": "recal_add", "read_groups": n_rg, "rep": rep, "gpu": gpu, "records": len(starts), "window_bytes": len(body),
                                  "bases": bases, "device_ms": ms, "gbases_per_s": bases / (ms / 1e3) / 1e9}), flush=True)
    ctx.close()

    # ---- bm2_mem --markdup --recal-file: the parent's build against this tree's, alternating
    if a.parent_mem:
        for rep in range(-1, a.reps):
            for kind, tool_ in (("parent", a.parent_mem), ("this", mem)):
                t = os.path.join(work, "brc_rate.%s.txt" % kind)
                t0 = time.perf_counter()
                r = run(tool_, t)
                wall = time.perf_counter() - t0
                st = json.loads(r.stderr.strip().splitlines()[-1])
                if rep >= 0:
                    print(json.dumps({"what": "bm2_mem --recal-file", "build": kind, "rep": rep, "gpu": gpu, "steady_reads_per_s": steady(st),
                                      "bqsr_s": st["bqsr_s"], "bqsr_bases": st["bqsr_bases"], "wall_s": wall}), flush=True)
            if open(os.path.join(work, "brc_rate.parent.txt")).read() != open(os.path.join(work, "brc_rate.this.txt")).read():
                raise AssertionError("bm2_mem --recal-file's table differs from the parent's")


if __name__ == "__main__":
    main()

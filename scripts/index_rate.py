"""bm2_index at human size: a 3.1 Gbp index_build.make_big_reference genome with ~150 Mbp of planted N runs, written as FASTA and indexed by
the tool; prints one JSON line with the stage times, the peak device bytes (the target is at most 48 GiB, so that the card can be shared),
the refinement rounds and the card with its power limit read in the same call, and checks the index without the reference (which would need
1-2 h and ~87 GB of RAM at this size):
  - at every sampled row the BWT character (from the CP_OCC one-hot words) equals .0123[SA - 1];
  - the running counts of consecutive CP_OCC entries differ by the popcounts of the one-hot words;
  - adjacent sampled rows are in suffix order by 31-mer keys; equal keys are compared on the host, the first 1000 of each 64 M-sample chunk;
  - exact 100 bp reads from the forward strand, those that overlap no N run, have a region at their origin through bm2_seed_chain_extend.
For comparison it indexes a 100 Mbp genome with the tool and with the reference binary (oracle/_ref), when present.

    python scripts/index_rate.py [--gbp 3.1] [--reads 100000] [--out results/index_rate.json]
Needs about 25 GB of free disk in the temporary directory; skips with a message otherwise.
"""
from __future__ import annotations
import argparse, json, os, shutil, subprocess, sys, tempfile, time
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_index")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def run_tool(fa, prefix):
    t = time.time()
    r = subprocess.run([TOOL, "-p", prefix, fa], capture_output=True, text=True)
    if r.returncode:
        raise SystemExit("bm2_index failed: " + r.stderr)
    return time.time() - t, json.loads(r.stderr.strip().splitlines()[-1])


def write_genome(path, total_bp, n_bp, seed):
    import index_corpus as ic
    from __graft_entry__ import load_package
    load_package()
    from bwa_mem2_b200 import index_build as ib
    contigs = ib.make_big_reference(total_bp, seed=seed, device="cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(seed + 1)
    acgt = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device="cuda")
    with open(path, "wb") as f:
        for name, c in contigs:
            s = acgt[c.long()]
            k = max(1, int(n_bp * len(c) / total_bp) // 50000)            # runs of 1-100 kbp, ~n_bp in all
            starts = torch.randint(0, len(c), (k,), device="cuda", generator=g)
            lens = torch.randint(1, 100000, (k,), device="cuda", generator=g)
            for a, L in zip(starts.tolist(), lens.tolist()):
                s[a:a + L] = ord("N")
            f.write(b">" + name.encode() + b" synthetic\n" + ic.fasta_lines(s.cpu().numpy(), 60))
    return contigs


def check(prefix, n_reads, seed):
    from __graft_entry__ import load_package
    capi = load_package().capi
    raw = np.memmap(prefix + ".bwt.2bit.64", np.uint8, "r")
    N = int(raw[:8].view(np.int64)[0]); n = N - 1
    n_occ, n_sa = (N >> 6) + 1, (N >> 3) + 1
    cp = raw[48:48 + n_occ * 64].view(np.int64).reshape(n_occ, 8)
    ms = raw[48 + n_occ * 64:48 + n_occ * 64 + n_sa].view(np.int8)
    ls = raw[48 + n_occ * 64 + n_sa:48 + n_occ * 64 + n_sa * 5].view(np.uint32)
    text = torch.from_numpy(np.fromfile(prefix + ".0123", np.uint8)).cuda()
    bad_char = bad_cnt = bad_order = ties = 0
    step = 1 << 26
    prev_last = None
    for i0 in range(0, n_sa, step):
        i1 = min(n_sa, i0 + step)
        sa = (torch.from_numpy(ms[i0:i1].astype(np.int64)).cuda() & 0xff) << 32 | torch.from_numpy(ls[i0:i1].astype(np.int64)).cuda()
        rows = torch.arange(i0, i1, device="cuda", dtype=torch.int64) * 8
        e = torch.from_numpy(np.ascontiguousarray(cp[(rows >> 6).cpu().numpy()])).cuda()
        bit = 63 - (rows & 63)
        onehot = torch.stack([((e[:, 4 + k] >> bit) & 1) for k in range(4)], 1)
        c = torch.where(onehot.sum(1) == 1, onehot.argmax(1), torch.full_like(rows, 4))
        want = torch.where(sa == 0, torch.full_like(sa, 4), text[(sa - 1).clamp(min=0)].long())
        bad_char += int((c != want).sum())
        # 31-mer keys (bases past the end as A) of adjacent samples must not decrease; equal keys are compared on the host
        key = torch.zeros_like(sa)
        for t in range(31):
            idx = sa + t
            key = key * 4 + torch.where(idx < n, text[idx.clamp(max=n - 1)].long(), torch.zeros_like(idx))
        if prev_last is not None:
            key = torch.cat([prev_last[0:1], key]); sa = torch.cat([prev_last[1:2], sa])
        bad_order += int((key[1:] < key[:-1]).sum())
        eq = torch.nonzero(key[1:] == key[:-1]).squeeze(1).cpu().numpy()
        if len(eq):
            ties += len(eq)
            t_np = None
            for j in eq[:1000]:
                a, b = int(sa[j]), int(sa[j + 1])
                if t_np is None:
                    t_np = np.memmap(prefix + ".0123", np.uint8, "r")
                L = 1 << 12
                while True:
                    x, y = bytes(t_np[a:a + L]), bytes(t_np[b:b + L])
                    if x != y or a + L >= n or b + L >= n:
                        bad_order += int(not x < y)
                        break
                    L *= 4
        prev_last = torch.stack([key[-1], sa[-1]])
    for r0 in range(0, n_occ - 1, step):
        r1 = min(n_occ - 1, r0 + step)
        e = torch.from_numpy(np.ascontiguousarray(cp[r0:r1 + 1])).cuda()
        pc = torch.stack([torch.from_numpy(np.unpackbits(e[:-1, 4 + k].cpu().numpy().view(np.uint8)).reshape(-1, 64).sum(1).astype(np.int64)).cuda()
                          for k in range(4)], 1)
        bad_cnt += int((e[1:, :4] - e[:-1, :4] != pc).sum())
    # exact reads from the forward strand (away from N runs, which the pack replaced) must have a region at their origin
    idx = capi.Index(prefix)
    ctx = capi.Context(0, index=idx)
    l_pac = n // 2
    rng = np.random.default_rng(seed)
    starts = np.sort(rng.integers(0, l_pac - 200, n_reads))
    amb = open(prefix + ".amb").read().split("\n")[1:]
    holes = np.array([[int(x) for x in l.split()[:2]] for l in amb if l], np.int64).reshape(-1, 2)
    if len(holes):
        k = np.searchsorted(holes[:, 0], starts + 100, side="left") - 1
        keep = (k < 0) | (holes[np.maximum(k, 0), 0] + holes[np.maximum(k, 0), 1] <= starts)
        keep &= np.searchsorted(holes[:, 0], starts) == np.searchsorted(holes[:, 0], starts + 100)
        starts = starts[keep]
    t_np = np.memmap(prefix + ".0123", np.uint8, "r")
    codes = np.concatenate([np.asarray(t_np[s:s + 100]) for s in starts])
    offs = np.arange(len(starts) + 1, dtype=np.int64) * 100
    regs, ro = ctx.seed_chain_extend(codes, offs)
    hit = np.zeros(len(starts), bool)
    read_of = np.repeat(np.arange(len(starts)), np.diff(ro))
    at = (regs["rb"] == starts[read_of]) & (regs["score"] == 100)
    hit[read_of[at]] = True
    ctx.close(); idx.close()
    return dict(bad_bwt_char=bad_char, bad_counts=bad_cnt, bad_order=bad_order, key_ties=ties, reads=int(len(starts)), reads_at_origin=int(hit.sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=3.1)
    ap.add_argument("--n-bp", type=float, default=150e6)
    ap.add_argument("--reads", type=int, default=100000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    total = int(a.gbp * 1e9)
    tmp = tempfile.mkdtemp(prefix="bm2_index_rate_")
    try:
        free = shutil.disk_usage(tmp).free
        if free < int(8 * total):
            print(json.dumps({"skipped": f"needs ~{8 * total / 1e9:.0f} GB of disk in {tmp}, {free / 1e9:.0f} GB free"}))
            return
        res = {"card": card(), "gbp": a.gbp}
        fa = tmp + "/big.fa"
        t = time.time(); contigs = write_genome(fa, total, int(a.n_bp), 7); res["fasta_write_s"] = time.time() - t
        del contigs; torch.cuda.empty_cache()
        res["wall_s"], res["stats"] = run_tool(fa, tmp + "/big")
        res["peak_device_gib"] = res["stats"]["peak_device_bytes"] / 2 ** 30
        os.remove(fa)
        res["checks"] = check(tmp + "/big", a.reads, 5)
        for ext in (".pac", ".ann", ".amb", ".0123", ".bwt.2bit.64"):
            os.remove(tmp + "/big" + ext)
        # 100 Mbp: the tool against the reference binary, in the same call
        import index_corpus as ic
        open(tmp + "/m.fa", "wb").write(ic.synthetic_fasta(100_000_000, seed=21))
        res["tool_100mbp_s"] = run_tool(tmp + "/m.fa", tmp + "/m_tool")[0]
        isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
        ref = os.path.join(ROOT, "oracle", "_ref", isa, "bwa-mem2")
        if os.path.exists(ref):
            t = time.time()
            subprocess.run([ref, "index", "-p", tmp + "/m_ref", tmp + "/m.fa"], check=True, capture_output=True)
            res["reference_100mbp_s"] = time.time() - t
        else:
            res["reference_100mbp_s"] = "not measured"
        res["card_after"] = card()
        line = json.dumps(res)
        print(line)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            open(a.out, "w").write(line + "\n")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()

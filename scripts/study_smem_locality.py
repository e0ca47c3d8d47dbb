#!/usr/bin/env python
"""Offline study (CPU only): how many 64-byte index lines per read the SMEM stage pulls from DRAM, and what alternatives would save.
Replays the accesses of the kernels' own search logic (fm_device.cuh compiled for the host, three passes) of N reads through an LRU cache
that is scaled to the index (50 MB of H100 L2 against the 6 GB Occ table of a 3 Gbp genome = 0.8 % of the table), for
  0  the current layout (64-byte checkpoint per 64 BWT rows),
  1  a half-size table (64-byte line per 128 rows: 2-bit packed BWT + counts),
  2  a k-mer table that answers the first k-1 extensions of every forward search with one fetch (k scaled with the genome),
  3  unique-interval stretches of the pass-1 forward searches verified against the reference text (8 accesses per stretch).
Usage: study_smem_locality.py <index prefix> <reads.npy> [n_reads]"""
import ctypes as C, os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from __graft_entry__ import load_package


def main():
    capi = load_package().capi
    prefix, reads_path = sys.argv[1], sys.argv[2]
    n = int(sys.argv[3]) if len(sys.argv) > 3 else 20000
    src = os.path.join(ROOT, "tests", "host_emul", "smem_study.cpp")
    so = "/tmp/libsmemstudy.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "bwa-mem2_b200", "csrc"), "-I" + os.path.join(ROOT, "include"), src, "-o", so])
    L = C.CDLL(so)
    idx = capi.Index(prefix)
    reads = np.load(reads_path)[:n]
    codes = np.ascontiguousarray(reads.reshape(-1)); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    table_bytes = (idx.desc.reference_seq_len // 64 + 1) * 64
    cache_lines = int(50e6 / 6.0e9 * table_bytes / 64)
    # k of the k-mer table: 12 at 6e9 BWT rows, one less per factor 4
    kk = max(6, int(round(12 - np.log(6.0e9 / idx.desc.reference_seq_len) / np.log(4))))
    out = np.zeros((4, 5, 3), np.float64)
    L.smem_study(C.byref(idx.desc), codes.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), C.c_int(len(reads)), C.c_longlong(cache_lines), C.c_int(kk),
                 out.ctypes.data_as(C.c_void_p))
    names = ["current layout", "half-size table (128 rows per line)", f"{kk}-mer table for the first {kk - 1} forward steps", "text check of unique pass-1 stretches"]
    phases = ["fwd1", "bwd1", "fwd2", "bwd2", "pass3"]
    print(f"index {table_bytes / 1e6:.0f} MB Occ table, cache model {cache_lines} lines ({cache_lines * 64 / 1e6:.1f} MB, 16-way LRU), {len(reads)} reads")
    base = out[0, :, 2].sum() / len(reads)
    for v in range(4):
        per = out[v] / len(reads)
        print(f"\n{names[v]}: index accesses {per[:, 0].sum():.0f}/read, lines {per[:, 1].sum():.0f}/read, DRAM lines {per[:, 2].sum():.0f}/read ({per[:, 2].sum() / base:.2f} of current)")
        print("   " + "  ".join(f"{p}: {per[i, 0]:.0f} acc / {per[i, 2]:.0f} miss" for i, p in enumerate(phases)))


if __name__ == "__main__":
    main()

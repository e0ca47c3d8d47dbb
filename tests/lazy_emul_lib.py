"""ctypes binding of tests/host_emul/libbm2lazyemul.so: the host emulation with the lazy extension's waves (test-only; see
tests/host_emul/lazy_emul.cpp).  Inputs and outputs as emul_lib.seed_chain_extend."""
from __future__ import annotations
import ctypes as C, os, subprocess
import numpy as np
import emul_lib as el

ROOT = el.ROOT
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import oracle_lib
        oracle_lib.lib()
        d = os.path.join(ROOT, "tests", "host_emul")
        so = os.path.join(d, "libbm2lazyemul.so")
        srcs = [os.path.join(d, "lazy_emul.cpp"), os.path.join(d, "emul.cpp")] + [os.path.join(ROOT, "bwa-mem2_b200", "csrc", f) for f in
                                                                                  ("fm_device.cuh", "chain_device.cuh", "ext_device.cuh", "hd.h")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-w", "-ffp-contract=off",
                                   "-I" + os.path.join(ROOT, "bwa-mem2_b200", "csrc"), "-I" + os.path.join(ROOT, "include"),
                                   os.path.join(d, "lazy_emul.cpp"), "-o", so, "-L" + os.path.join(ROOT, "oracle"), "-lbm2oracle",
                                   "-Wl,-rpath," + os.path.join(ROOT, "oracle")])
        _LIB = C.CDLL(so)
    return _LIB


def seed_chain_extend(index, opt, codes, offsets):
    """(regs, read offsets, stats): stats = jobs built, jobs never run, reads decided after the first wave, regs the final post-filter
    kept that were never extended."""
    capi = el._capi(); rb, keep = el._batch(codes, offsets)
    regs = C.c_void_p(); off = C.c_void_p(); n = C.c_int64()
    L = lib()
    L.lazy_emul_seed_chain_extend(C.byref(index.desc), C.byref(opt), C.byref(rb), C.byref(regs), C.byref(n), C.byref(off))
    a = el._arr(regs, n.value, capi.REG_DT)
    offs = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_int64)), shape=(rb.n_reads + 1,)).copy()
    el._free(regs, off)
    v = (C.c_int64 * 4)()
    L.lazy_emul_last_ext_stats(v)
    return a, offs, dict(jobs=v[0], skipped=v[1], done_wave1=v[2], kept_not_extended=v[3])

"""The ballot resolution of the warp post-filter scans (pf_scan_step_d in bwa-mem2_b200/csrc/ext_device.cuh, used by pf_scan_warp in
pipeline.cu for the tail's warp post-filter and the warp walk of the lazy extension): applied over the 32-box steps of a scan, it must
give the same v and stop in the same step as the sequential loop of pf_seed_purged_d, `for (i = 0; i < n_reg && v < lim; ++i)`, for
any box kinds (0 skipped, 1 counted, 2 hit) and any lim."""
import ctypes as C, os, subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    d = os.path.join(ROOT, "tests", "host_emul")
    src, so = os.path.join(d, "scan_step_emul.cpp"), os.path.join(d, "libbm2scanstep.so")
    deps = [src] + [os.path.join(ROOT, "bwa-mem2_b200", "csrc", f) for f in ("ext_device.cuh", "chain_device.cuh", "hd.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I" + os.path.join(ROOT, "bwa-mem2_b200", "csrc"),
                               "-I" + os.path.join(ROOT, "include"), src, "-o", so])
    return C.CDLL(so)


def _sequential(kind, lim):
    """(v, step of the box the loop stopped at, -1 when it ran off the end or never started)"""
    v = 0
    for i, k in enumerate(kind):
        if v >= lim:
            return v, (i - 1) // 32
        if k == 2:
            return v, i // 32
        v += int(k)
    return v, ((len(kind) - 1) // 32 if len(kind) and v >= lim > 0 else -1)


def _warp(fn, kind, lim):
    stop = C.c_int()
    v = fn(kind.ctypes.data_as(C.c_void_p), len(kind), lim, C.byref(stop))
    return v, stop.value


def test_step_resolution_matches_sequential_scan():
    fn = _lib().scan_step_emul
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)]
    rng = np.random.default_rng(5)
    n_cases = n_hit_stops = n_lim_stops = 0
    for case in range(400):
        n = int(rng.integers(1, 2001)) if case % 4 else int(rng.integers(1, 70))
        p_hit = [0.0, 0.001, 0.01, 0.1, 0.5][case % 5]
        p_skip = [0.0, 0.3, 0.7, 0.95][case % 4]
        kind = rng.choice(3, size=n, p=[p_skip * (1 - p_hit), (1 - p_skip) * (1 - p_hit), p_hit]).astype(np.int8)
        n_counted = int((kind == 1).sum())
        lims = range(0, n_counted + 3) if n_counted < 300 else sorted(set(rng.integers(0, n_counted + 3, 200).tolist()) | {0, 1, n_counted, n_counted + 1})
        for lim in lims:
            want = _sequential(kind, lim)
            assert _warp(fn, kind, lim) == want, (case, n, lim)
            n_cases += 1
            if want[1] >= 0:
                if want[0] < lim:
                    n_hit_stops += 1
                else:
                    n_lim_stops += 1
    assert n_cases > 20000 and n_hit_stops > 1000 and n_lim_stops > 1000

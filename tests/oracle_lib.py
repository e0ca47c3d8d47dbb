"""ctypes binding of oracle/libbm2oracle.so (CPU restatement; test infrastructure only)."""
from __future__ import annotations
import ctypes as C, os, subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None


class BswParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("a", "b", "o_del", "e_del", "o_ins", "e_ins", "zdrop", "end_bonus", "vector_quirks")]


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(ROOT, "oracle", "libbm2oracle.so")
        src = os.path.join(ROOT, "oracle", "bm2_oracle.cpp")
        if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "port"], stdout=subprocess.DEVNULL)
        _LIB = C.CDLL(so)
        _LIB.bm2o_extend_pairs.restype = C.c_int64
        _LIB.bm2o_bsw_extend.restype = C.c_int64
    return _LIB


def bsw_params(a=1, b=4, o_del=6, e_del=1, o_ins=6, e_ins=1, zdrop=100, end_bonus=5, vector_quirks=1):
    return BswParams(a, b, o_del, e_del, o_ins, e_ins, zdrop, end_bonus, vector_quirks)


def make_pairs(len1, len2, h0, idr, idq):
    from refdump import PAIR_DT
    n = len(len1)
    p = np.zeros(n, PAIR_DT)
    p["len1"] = len1; p["len2"] = len2; p["h0"] = h0; p["idr"] = idr; p["idq"] = idq
    p["id"] = np.arange(n)
    return p


def extend_pairs(pairs, ref, qer, w, params):
    """Runs the oracle in place on a PAIR_DT array; returns banded cell count."""
    ref = np.ascontiguousarray(ref, np.uint8); qer = np.ascontiguousarray(qer, np.uint8)
    assert pairs.flags.c_contiguous
    return lib().bm2o_extend_pairs(pairs.ctypes.data_as(C.c_void_p), ref.ctypes.data_as(C.c_void_p),
                                   qer.ctypes.data_as(C.c_void_p), C.c_int32(len(pairs)), C.c_int32(w), C.byref(params))


# ---- FM-index stages ----------------------------------------------------------------------------
def _capi():
    import sys
    from __graft_entry__ import load_package
    return load_package().capi


def collect_smems(index, opt, codes, offsets):
    capi = _capi()
    codes = np.ascontiguousarray(codes, np.uint8); offsets = np.ascontiguousarray(offsets, np.int64)
    rb = capi.ReadBatch(len(offsets) - 1, codes.ctypes.data, offsets.ctypes.data)
    out = C.c_void_p()
    L = lib()
    L.bm2o_collect_smems.restype = C.c_int64
    n = L.bm2o_collect_smems(C.byref(index.desc), C.byref(opt), C.byref(rb), C.byref(out))
    a = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_uint8)), shape=(max(n, 1) * capi.SMEM_DT.itemsize,))[:n * capi.SMEM_DT.itemsize].view(capi.SMEM_DT).copy()
    L.bm2o_free(out)
    return a


def sa_lookup(index, rows):
    rows = np.ascontiguousarray(rows, np.int64)
    out = np.empty_like(rows)
    lib().bm2o_sa_lookup(C.byref(index.desc), rows.ctypes.data_as(C.c_void_p), C.c_int64(len(rows)), out.ctypes.data_as(C.c_void_p))
    return out


def seed_chain(index, opt, codes, offsets):
    capi = _capi()
    codes = np.ascontiguousarray(codes, np.uint8); offsets = np.ascontiguousarray(offsets, np.int64)
    rb = capi.ReadBatch(len(offsets) - 1, codes.ctypes.data, offsets.ctypes.data)
    ch = C.c_void_p(); sd = C.c_void_p(); off = C.c_void_p(); nc = C.c_int64(); ns = C.c_int64()
    L = lib()
    rc = L.bm2o_seed_chain(C.byref(index.desc), C.byref(opt), C.byref(rb), C.byref(ch), C.byref(nc), C.byref(sd), C.byref(ns), C.byref(off))
    assert rc == 0
    def arr(p, n, dt):
        a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(n, 1) * dt.itemsize,))[:n * dt.itemsize].view(dt).copy()
        return a
    chains = arr(ch, nc.value, capi.CHAIN_DT); seeds = arr(sd, ns.value, capi.SEED_DT)
    offs = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_int64)), shape=(rb.n_reads + 1,)).copy()
    for p in (ch, sd, off):
        L.bm2o_free(p)
    return chains, seeds, offs


def seed_chain_extend(index, opt, codes, offsets):
    """-> (regs REG_DT array, read_off, bsw_cells, rc)"""
    capi = _capi()
    codes = np.ascontiguousarray(codes, np.uint8); offsets = np.ascontiguousarray(offsets, np.int64)
    rb = capi.ReadBatch(len(offsets) - 1, codes.ctypes.data, offsets.ctypes.data)
    regs = C.c_void_p(); off = C.c_void_p(); n = C.c_int64(); cells = C.c_int64()
    L = lib()
    rc = L.bm2o_seed_chain_extend(C.byref(index.desc), C.byref(opt), C.byref(rb), C.byref(regs), C.byref(n), C.byref(off), C.byref(cells))
    dt = capi.REG_DT
    a = np.ctypeslib.as_array(C.cast(regs, C.POINTER(C.c_uint8)), shape=(max(n.value, 1) * dt.itemsize,))[:n.value * dt.itemsize].view(dt).copy()
    offs = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_int64)), shape=(rb.n_reads + 1,)).copy()
    L.bm2o_free(regs); L.bm2o_free(off)
    return a, offs, cells.value, rc


def gen_cigar(index, opt, codes, offsets, reqs):
    """Oracle's bwa_gen_cigar2 restatement -> (recs CIGAR_REC_DT, cigar uint32[], md bytes, rc)."""
    capi = _capi()
    codes = np.ascontiguousarray(codes, np.uint8); offsets = np.ascontiguousarray(offsets, np.int64)
    reqs = np.ascontiguousarray(reqs, capi.CIGAR_REQ_DT)
    rb = capi.ReadBatch(len(offsets) - 1, codes.ctypes.data, offsets.ctypes.data)
    recs = C.c_void_p(); cig = C.c_void_p(); md = C.c_void_p(); n_ops = C.c_int64(); n_md = C.c_int64()
    L = lib()
    rc = L.bm2o_gen_cigar(C.byref(index.desc), C.byref(opt), C.byref(rb), reqs.ctypes.data_as(C.c_void_p), C.c_int64(len(reqs)),
                          C.byref(recs), C.byref(cig), C.byref(n_ops), C.byref(md), C.byref(n_md))
    if rc:
        return None, None, None, rc
    def arr(p, n, dt):
        dt = np.dtype(dt)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(n, 1) * dt.itemsize,))[:n * dt.itemsize].view(dt).copy()
    out = arr(recs, len(reqs), capi.CIGAR_REC_DT), arr(cig, n_ops.value, "<u4"), arr(md, n_md.value, "u1"), 0
    for p in (recs, cig, md):
        L.bm2o_free(p)
    return out


REG_CMP_FIELDS = ("rb", "re", "qb", "qe", "rid", "score", "truesc", "sub", "alt_sc", "csub", "sub_n", "w", "seedcov",
                  "secondary", "secondary_all", "seedlen0", "frac_rep", "hash")


def _regs_digest(off, cols):
    import hashlib
    h = hashlib.sha256(np.asarray(off, np.int64).tobytes())
    for name, v in cols:
        v = np.asarray(v)
        h.update(name.encode() + np.ascontiguousarray(v.astype(np.float64 if v.dtype.kind == "f" else np.int64)).tobytes())
    return h.hexdigest()


def regs_digest(regs, off):
    """SHA-256 of what regs_equal_to_dump compares, for REG_DT regs (ours): equal digests <=> regs_equal_to_dump(...) == []."""
    return _regs_digest(off, [(f, regs[f]) for f in REG_CMP_FIELDS] + [("n_comp", (regs["n_comp_is_alt"] << 2) >> 2),
                                                                        ("is_alt", (regs["n_comp_is_alt"] >> 30) & 3)])


def dump_digest(dump_regs, dump_off):
    """regs_digest of a reference regs dump (refdump.read_regs): the stored form of the reference's regs in tests/golden."""
    return _regs_digest(dump_off, [(f, dump_regs[f]) for f in REG_CMP_FIELDS] + [("n_comp", dump_regs["n_comp"]),
                                                                                  ("is_alt", dump_regs["is_alt"] & 3)])


def regs_equal_to_dump(regs, off, dump_regs, dump_off):
    """Compare REG_DT regs (ours) with refdump.REG_DT regs (reference dump). Returns list of differing reads."""
    bad = []
    if not np.array_equal(off, dump_off):
        bad = list(np.nonzero(np.diff(off) != np.diff(dump_off))[0][:20])
    same = len(regs) == len(dump_regs)
    if same:
        ok = np.ones(len(regs), bool)
        for f in REG_CMP_FIELDS:
            ok &= regs[f] == dump_regs[f]
        ok &= ((regs["n_comp_is_alt"] << 2) >> 2) == dump_regs["n_comp"]
        ok &= ((regs["n_comp_is_alt"] >> 30) & 3) == (dump_regs["is_alt"] & 3)
        if not ok.all():
            idx = np.nonzero(~ok)[0]
            rd = np.searchsorted(off, idx, side="right") - 1
            bad = sorted(set(bad) | set(rd.tolist()))
    return bad

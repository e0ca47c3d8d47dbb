"""Helpers of the bm2_baserecalibrator tests: the recalibration rule of tests/bqsr_util.py counted per read group, the report of several
covariates and the read groups of headers restated in Python, the host emulation tests/host_emul/baserecalibrator_emul.cpp, records with an
RG:Z tag."""
import ctypes as C
import os, struct, subprocess
import math
import numpy as np
from bqsr_util import (ARGUMENTS, CSRC, MAXC, NCTX, NCYC, NQ, ROOT, _table, bu, empirical_q, pack_bits, read_group, record_bases,  # noqa: F401
                       report_text)


# ---- the rule per read group, the report of several covariates, the host emulation ----

COUNTS = 2 * NQ * NCTX + 2 * NQ * NCYC + 2                                      # kBqsrCounts: one covariate's counters on the device


def rg_tag_value(rec):
    for tg, t, v in bu.fields(rec)["tags"]:
        if tg == "RG" and t == "Z":
            return v
    return None


def empty_tables():
    return dict(qual_obs=np.zeros(NQ, np.int64), qual_err=np.zeros(NQ, np.int64), ctx_obs=np.zeros((NQ, NCTX), np.int64),
                ctx_err=np.zeros((NQ, NCTX), np.int64), cyc_obs=np.zeros((NQ, NCYC), np.int64), cyc_err=np.zeros((NQ, NCYC), np.int64),
                reads=0, bases=0)


def count_rg(recs, ref, cov, jun, ids, id_cov, n_cov):
    """Records -> ([tables of each covariate], err (index, kind) or None): a record past the filters needs an RG:Z value among ids (kind 4
    without the tag, 5 for a value that is no ID), checked before the read errors 1..3; it counts into the tables of covariate id_cov."""
    ts, err = [empty_tables() for _ in range(n_cov)], None
    for i, r in enumerate(recs):
        st, bases = record_bases(r, ref, cov, jun)
        c = 0
        if st != 4:
            v = rg_tag_value(r)
            if v is None:
                st = 4 + 10
            elif v not in ids:
                st = 5 + 10
            else:
                c = id_cov[ids.index(v)]
        if st in (1, 2, 3, 14, 15):
            if err is None:
                err = (i, st - 10 if st > 10 else st)
            continue
        if st != 0:
            continue
        t = ts[c]
        t["reads"] += 1
        for q, cx, cyc, e in bases:
            t["bases"] += 1
            t["qual_obs"][q] += 1; t["qual_err"][q] += e
            if cx is not None:
                t["ctx_obs"][q, cx] += 1; t["ctx_err"][q, cx] += e
            t["cyc_obs"][q, cyc + MAXC] += 1; t["cyc_err"][q, cyc + MAXC] += e
    return ts, err


def report_text_rg(tables, names):
    """The report of several covariates: RecalTable0 one row per covariate, RecalTable1 and RecalTable2 each covariate's rows in turn (in the
    order given), the Quantized table's Count summed over them."""
    o = "#:GATKReport.v1.1:5\n"
    o += _table("Arguments", "Recalibration argument collection values used in this run", [("Argument", "%s"), ("Value", "%s")],
                [list(a) for a in ARGUMENTS])
    qsum = sum((t["qual_obs"] for t in tables), np.zeros(NQ, np.int64))
    o += _table("Quantized", "Quality quantization map", [("QualityScore", "%d"), ("Count", "%d"), ("QuantizedScore", "%d")],
                [[str(q), str(int(qsum[q])), str(q)] for q in range(NQ)])
    rows0, rows1, rows2 = [], [], []
    for t, rg in zip(tables, names):
        N, E, s = int(t["qual_obs"].sum()), int(t["qual_err"].sum()), 0.0
        for q in range(NQ):
            s += float(t["qual_obs"][q]) * 10.0 ** (q / -10.0)
        if N:
            qr = -10.0 * math.log10(s / N)
            rows0.append([rg, "M", "%.4f" % empirical_q(N, E, qr), "%.4f" % qr, str(N), "%.2f" % E])
        for q in range(NQ):
            n, e = int(t["qual_obs"][q]), int(t["qual_err"][q])
            if n:
                rows1.append([rg, str(q), "M", "%.4f" % empirical_q(n, e, q), str(n), "%.2f" % e])
            for c in range(NCTX):
                n, e = int(t["ctx_obs"][q, c]), int(t["ctx_err"][q, c])
                if n:
                    rows2.append([rg, str(q), "ACGT"[c >> 2] + "ACGT"[c & 3], "Context", "M", "%.4f" % empirical_q(n, e, q), str(n), "%.2f" % e])
            for y in np.nonzero(t["cyc_obs"][q])[0]:
                n, e = int(t["cyc_obs"][q, y]), int(t["cyc_err"][q, y])
                rows2.append([rg, str(q), str(int(y) - MAXC), "Cycle", "M", "%.4f" % empirical_q(n, e, q), str(n), "%.2f" % e])
    o += _table("RecalTable0", "", [("ReadGroup", "%s"), ("EventType", "%s"), ("EmpiricalQuality", "%.4f"), ("EstimatedQReported", "%.4f"),
                                    ("Observations", "%d"), ("Errors", "%.2f")], rows0)
    o += _table("RecalTable1", "", [("ReadGroup", "%s"), ("QualityScore", "%d"), ("EventType", "%s"), ("EmpiricalQuality", "%.4f"),
                                    ("Observations", "%d"), ("Errors", "%.2f")], rows1)
    o += _table("RecalTable2", "", [("ReadGroup", "%s"), ("QualityScore", "%d"), ("CovariateValue", "%s"), ("CovariateName", "%s"),
                                    ("EventType", "%s"), ("EmpiricalQuality", "%.4f"), ("Observations", "%d"), ("Errors", "%.2f")], rows2)
    return o


def read_groups(texts):
    """Headers -> (ids in order of first appearance, each one's covariate index, covariates in byte order); raises ValueError as the tool
    fails: an input without @RG, one ID with two covariates."""
    cov_of, order = {}, []
    for k, text in enumerate(texts):
        here = {}
        for line in text.split("\n"):
            if not line.startswith("@RG\t"):
                continue
            f = dict(x.split(":", 1) for x in line.split("\t")[1:] if ":" in x)
            i = f.get("ID", "")
            if i in here:
                continue
            here[i] = read_group(line)
            if i not in cov_of:
                cov_of[i] = here[i]; order.append(i)
            elif cov_of[i] != here[i]:
                raise ValueError("read group %s has covariate %s here" % (i, here[i]))
        if not here:
            raise ValueError("the header has no @RG line")
    covs = sorted(set(cov_of.values()), key=lambda c: c.encode())
    return order, [covs.index(cov_of[i]) for i in order], covs


def pac_of(ref):
    pac = np.zeros((ref.l_pac + 3) // 4, np.uint8)
    i = np.arange(ref.l_pac)
    np.bitwise_or.at(pac, i >> 2, (ref.codes.astype(np.uint8) << ((3 - (i & 3)) * 2)).astype(np.uint8))
    return pac


def build_rg_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bre_emul") / "libbreemul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "host_emul", "baserecalibrator_emul.cpp"), "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.bre_count.restype = C.c_int32
    lib.bre_count.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int64]
    lib.bre_map.restype = C.c_int64
    lib.bre_map.argtypes = [C.c_char_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]
    lib.bre_report.restype = C.c_int64
    lib.bre_report.argtypes = [C.c_char_p, C.c_int32, C.c_void_p, C.c_char_p, C.c_int64]
    lib.bre_read_groups.restype = C.c_int32
    lib.bre_read_groups.argtypes = [C.c_char_p, C.c_int32, C.c_char_p, C.c_char_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p]
    lib.bre_run.restype = C.c_int32
    lib.bre_run.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int64, C.c_int32, C.c_char_p, C.c_int64, C.c_void_p]
    return lib


def _dense(cnt, c):
    """One covariate's dict from the device-layout counters (the quality table summed over the cycles, as on the device)."""
    t = cnt[c * COUNTS:(c + 1) * COUNTS]
    a, b = NQ * NCTX, NQ * NCYC
    d = dict(ctx_obs=t[:a].reshape(NQ, NCTX).copy(), ctx_err=t[a:2 * a].reshape(NQ, NCTX).copy(), cyc_obs=t[2 * a:2 * a + b].reshape(NQ, NCYC).copy(),
             cyc_err=t[2 * a + b:2 * a + 2 * b].reshape(NQ, NCYC).copy(), reads=int(t[-2]), bases=int(t[-1]))
    d["qual_obs"], d["qual_err"] = d["cyc_obs"].sum(1), d["cyc_err"].sum(1)
    return d


def emul_count_rg(lib, data, starts, ref, cov, jun, ids, id_cov, n_cov):
    """The emulation's rule -> ([tables of each covariate], err (index, kind) or None, message)."""
    starts = np.ascontiguousarray(starts, np.int64)
    buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
    sb = starts if len(starts) else np.zeros(1, np.int64)
    blob = np.zeros(1 << 16, np.uint8)
    vals = np.array(list(id_cov) + [0], np.int32)
    assert lib.bre_map("\n".join(ids).encode(), len(ids), vals.ctypes.data, blob.ctypes.data, len(blob)) >= 0
    cw, jw = pack_bits(cov), pack_bits(jun)
    holes = np.array(ref.holes, np.int64).reshape(-1) if ref.holes else np.zeros(2, np.int64)
    off, ln, pac = np.array(ref.off, np.int64), np.array(ref.lens, np.int32), pac_of(ref)
    cnt, err = np.zeros(n_cov * COUNTS, np.int64), np.zeros(2, np.int64)
    msg = C.create_string_buffer(4096)
    lib.bre_count(buf.ctypes.data, sb.ctypes.data, len(starts), pac.ctypes.data, ref.l_pac, off.ctypes.data, ln.ctypes.data, len(off), cw.ctypes.data,
                  jw.ctypes.data, holes.ctypes.data, len(ref.holes), blob.ctypes.data, len(ids), cnt.ctypes.data, err.ctypes.data, msg, 4096)
    return [_dense(cnt, c) for c in range(n_cov)], None if err[1] == 0 else (int(err[0]), int(err[1])), msg.value.decode()


def emul_report_rg(lib, tables, names):
    cnt = np.zeros(len(tables) * COUNTS, np.int64)
    for c, t in enumerate(tables):
        cnt[c * COUNTS:(c + 1) * COUNTS] = np.concatenate([np.asarray(t[k], np.int64).reshape(-1) for k in ("ctx_obs", "ctx_err", "cyc_obs", "cyc_err")]
                                                          + [np.array([t["reads"], t["bases"]], np.int64)])
    n = lib.bre_report("\n".join(names).encode(), len(names), cnt.ctypes.data, None, 0)
    out = C.create_string_buffer(n + 1)
    lib.bre_report("\n".join(names).encode(), len(names), cnt.ctypes.data, out, n + 1)
    return out.value.decode()


def emul_read_groups(lib, texts, names):
    out = C.create_string_buffer(1 << 16)
    ic, cn = np.zeros(4096, np.int32), np.zeros(2, np.int32)
    if lib.bre_read_groups(b"\0".join(t.encode() for t in texts) + b"\0", len(texts), "\n".join(names).encode(), out, 1 << 16, ic.ctypes.data, 4096,
                           cn.ctypes.data):
        raise ValueError(out.value.decode())
    a, b = out.value.decode().split("\n")
    return a.split("\t")[:-1], ic[:cn[0]].tolist(), b.split("\t")[:-1]


def emul_run(lib, prefix, inputs, vcfs, window=1 << 28, threads=2):
    """The emulated tool -> (table text, stats) or raises ValueError with the error."""
    out = C.create_string_buffer(1 << 24)
    st = np.zeros(6, np.int64)
    if lib.bre_run(prefix.encode(), "\n".join(inputs).encode(), "\n".join(vcfs).encode(), window, threads, out, 1 << 24, st.ctypes.data):
        raise ValueError(out.value.decode())
    return out.value.decode(), dict(records=int(st[0]), windows=int(st[1]), counted_reads=int(st[2]), counted_bases=int(st[3]),
                                    read_groups=int(st[4]), known_sites=int(st[5]))


def with_rg(rec, v):
    """The record with an RG:Z tag of value v appended."""
    tag = b"RGZ" + v.encode() + b"\0"
    return struct.pack("<i", len(rec) - 4 + len(tag)) + rec[4:] + tag

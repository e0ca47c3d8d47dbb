"""Helpers of the bm2_applybqsr tests: the apply rule of bwa-mem2_b200/csrc/bqsr_device.cuh and the table parser and deltas of bqsr_report.h
restated in Python (built on tests/bqsr_util.py), the host emulation tests/host_emul/applybqsr_emul.cpp, GATK-shaped tables and crafted
records for each branch of the rule."""
import ctypes as C
import os, struct, subprocess
import numpy as np
import bam_util as bu
import bqsr_util as bq

ROOT, CSRC = bq.ROOT, bq.CSRC
NQ, NCTX, NCYC, MAXC = bq.NQ, bq.NCTX, bq.NCYC, bq.MAXC
APPLY, KEEP, ERR_CYCLES, ERR_QUAL = 0, 1, 4, 5
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_applybqsr")


# ---- the table ----

def _cells(line):
    return [c for c in line.split(" ") if c]


def parse_tables(text):
    """A GATKReport -> {table name: (header cells, [row cells])} (the first table of each name)."""
    lines = text.split("\n")
    out, i = {}, 1
    while i < len(lines):
        if lines[i].startswith("#:GATKTable:") and lines[i][12:13].isdigit():
            nc, nr = (int(x) for x in lines[i][12:].split(":")[:2])
            name = lines[i + 1][12:].split(":")[0]
            hdr = _cells(lines[i + 2])
            rows = [_cells(lines[i + 3 + k]) for k in range(nr)]
            out.setdefault(name, (hdr, rows))
            i += 3 + nr
        else:
            i += 1
    return out


def dense(text):
    """The dense tables of a report: (read groups, P [n, 94], D_ctx [n, 94, 16], D_cyc [n, 94, 1001]), float64, by bqsr_report.h's rule."""
    t = parse_tables(text)

    def rows(name):
        hdr, rs = t[name]
        return [dict(zip(hdr, r)) for r in rs if dict(zip(hdr, r))["EventType"] == "M"]

    rgs, r0 = [], {}
    for r in rows("RecalTable0"):
        rgs.append(r["ReadGroup"])
        r0[r["ReadGroup"]] = (float(r["EstimatedQReported"]), int(r["Observations"]), float(r["Errors"]))
    q1, c2, y2 = {}, {}, {}
    for r in rows("RecalTable1"):
        q1[(r["ReadGroup"], int(r["QualityScore"]))] = (int(r["Observations"]), float(r["Errors"]))
    for r in rows("RecalTable2"):
        v = r["CovariateValue"]
        key = (r["ReadGroup"], int(r["QualityScore"]), v)
        (c2 if r["CovariateName"] == "Context" else y2)[key] = (int(r["Observations"]), float(r["Errors"]))

    def EQ(ne, prior):
        return float(bq.empirical_q(ne[0], int(ne[1] + 0.5), prior))

    n = len(rgs)
    P, Cx, Y = np.zeros((n, NQ)), np.zeros((n, NQ, NCTX)), np.zeros((n, NQ, NCYC))
    for k, rg in enumerate(rgs):
        E, n0, e0 = r0[rg]
        G = EQ((n0, e0), E) - E
        EG = E + G
        for q in range(NQ):
            Dq = EQ(q1[(rg, q)], EG) - EG if (rg, q) in q1 else 0.0
            p = EG + Dq
            P[k, q] = p
            for c in range(NCTX):
                key = (rg, q, "ACGT"[c >> 2] + "ACGT"[c & 3])
                if key in c2:
                    Cx[k, q, c] = EQ(c2[key], p) - p
            for y in range(-MAXC, MAXC + 1):
                key = (rg, q, str(y))
                if y and key in y2:
                    Y[k, q, y + MAXC] = EQ(y2[key], p) - p
    return rgs, P, Cx, Y


def _fmt_table(name, cols, rows, order=None):
    order = order or list(range(len(cols)))
    return bq._table(name, "", [cols[k] for k in order], [[r[k] for k in order] for r in rows])


def gatk_table(rng, rgs, priors=None, shuffle=False, args=None):
    """A GATK-shaped report: several read groups, M, I and D rows, fractional Errors, rows missing at each level (a read group without a
    RecalTable1 row for some qualities, contexts and cycles left out).  priors: each read group's EstimatedQReported."""
    o = "#:GATKReport.v1.1:5\n"
    a = dict(bq.ARGUMENTS)
    a.update(args or {})
    o += bq._table("Arguments", "Recalibration argument collection values used in this run", [("Argument", "%s"), ("Value", "%s")],
                   [[k, v] for k, v in a.items()])
    o += bq._table("Quantized", "Quality quantization map", [("QualityScore", "%d"), ("Count", "%d"), ("QuantizedScore", "%d")],
                   [[str(q), "0", str(q)] for q in range(NQ)])
    r0, r1, r2 = [], [], []
    for k, rg in enumerate(rgs):
        E = priors[k] if priors else float(rng.uniform(20, 38))
        n0 = int(rng.integers(10**5, 10**8))
        for ev in "MID":
            r0.append([rg, ev, "%.4f" % 30, "%.4f" % (E if ev == "M" else 45.0), str(n0), "%.2f" % (n0 * float(rng.uniform(1e-4, 3e-2)))])
        for q in sorted(set(int(x) for x in rng.integers(2, 45, 12))):
            if rng.random() < 0.15:
                continue                                                      # a quality without a RecalTable1 row, but with table 2 rows
            n = int(rng.integers(100, 10**7))
            for ev in "MID":
                r1.append([rg, str(q), ev, "%.4f" % q, str(n), "%.2f" % (n * float(rng.uniform(1e-5, 0.1)))])
        for q in sorted(set(int(x) for x in rng.integers(2, 45, 12))):
            for c in rng.choice(16, int(rng.integers(3, 16)), replace=False):
                n = int(rng.integers(10, 10**6))
                r2.append([rg, str(q), "ACGT"[c >> 2] + "ACGT"[c & 3], "Context", "M", "%.4f" % q, str(n), "%.2f" % (n * float(rng.uniform(0, 0.2)))])
            for y in rng.choice(np.r_[-MAXC:0, 1:MAXC + 1], int(rng.integers(5, 200)), replace=False):
                n = int(rng.integers(1, 10**6))
                for ev in "MI":
                    r2.append([rg, str(q), str(int(y)), "Cycle", ev, "%.4f" % q, str(n), "%.2f" % (n * float(rng.uniform(0, 0.2)))])
    cols0 = [("ReadGroup", "%s"), ("EventType", "%s"), ("EmpiricalQuality", "%.4f"), ("EstimatedQReported", "%.4f"), ("Observations", "%d"),
             ("Errors", "%.2f")]
    cols1 = [("ReadGroup", "%s"), ("QualityScore", "%d"), ("EventType", "%s"), ("EmpiricalQuality", "%.4f"), ("Observations", "%d"), ("Errors", "%.2f")]
    cols2 = [("ReadGroup", "%s"), ("QualityScore", "%d"), ("CovariateValue", "%s"), ("CovariateName", "%s"), ("EventType", "%s"),
             ("EmpiricalQuality", "%.4f"), ("Observations", "%d"), ("Errors", "%.2f")]
    perm = (lambda n: [int(x) for x in rng.permutation(n)]) if shuffle else (lambda n: None)
    return o + _fmt_table("RecalTable0", cols0, r0, perm(6)) + _fmt_table("RecalTable1", cols1, r1, perm(6)) + \
        _fmt_table("RecalTable2", cols2, r2, perm(8))


# ---- the per-record rule ----

def rg_value(rec):
    for tg, t, v in bu.fields(rec)["tags"]:
        if tg == "RG" and t == "Z":
            return v
    return None


def apply_record(rec, ids, id_table, tabs):
    """One record -> (status, the record with its new qualities, bases changed); status APPLY, KEEP, ERR_CYCLES or ERR_QUAL (then the record
    is returned as it was)."""
    _, P, Cx, Y = tabs
    v = rg_value(rec)
    k = ids.index(v) if v is not None and v in ids else None
    bs, rid, pos, lrn, mapq, bin_, ncig, flag, L = struct.unpack("<iiiBBHHHi", rec[:24])
    qoff = 36 + lrn + 4 * ncig + (L + 1) // 2
    qual = list(rec[qoff:qoff + L])
    if k is None or id_table[k] < 0 or L == 0 or qual[0] == 0xFF:
        return KEEP, rec, 0
    if L > MAXC:
        return ERR_CYCLES, rec, 0
    if any(q > 93 for q in qual):
        return ERR_QUAL, rec, 0
    r = id_table[k]
    sb = rec[36 + lrn + 4 * ncig:qoff]
    seq = ["=ACMGRSVTWYHKDBN"[(sb[j // 2] >> (4 * (1 - j % 2))) & 15] for j in range(L)]
    good = [j for j in range(L) if qual[j] > 2]
    tl, tr = (good[0], good[-1] + 1) if good else (L, L)
    letter = lambda j: 4 if j < tl or j >= tr else bq._code(seq[j])
    rev, f = bool(flag & 16), -1 if flag & 1 and flag & 0x80 else 1
    out, changed = bytearray(rec), 0
    for j in range(L):
        q = qual[j]
        if q < 6:
            continue
        cyc = (L - j if rev else j + 1) * f
        if not rev:
            pair = None if j == 0 else (letter(j - 1), letter(j))
        else:
            pair = None if j == L - 1 else tuple(4 if x == 4 else 3 - x for x in (letter(j + 1), letter(j)))
        cx = None if pair is None or 4 in pair else pair[0] * 4 + pair[1]
        d = P[r, q] + ((0.0 + (Cx[r, q, cx] if cx is not None else 0.0)) + Y[r, q, cyc + MAXC])
        nq = int(d + 0.5) if d > 0 else int(d - 0.5)
        nq = min(max(nq, 1), 93)
        if nq != q:
            out[qoff + j] = nq
            changed += 1
    return APPLY, bytes(out), changed


def header_map(text, rgs):
    """The header's @RG IDs and each one's read group index in rgs (its PU, else its ID), or -1."""
    ids, tab = [], []
    for line in text.split("\n"):
        if line.startswith("@RG\t"):
            f = dict(x.split(":", 1) for x in line.split("\t")[1:] if ":" in x)
            ids.append(f.get("ID", ""))
            c = bq.read_group(line)
            tab.append(rgs.index(c) if c in rgs else -1)
    return ids, tab


def with_tags(rec, tags: bytes):
    return struct.pack("<i", len(rec) - 4 + len(tags)) + rec[4:] + tags


def rg_tag(v):
    return b"RGZ" + v.encode() + b"\0"


def crafted(ref, rng, rgs_ids):
    """Records for each branch: forward, reverse, second of a pair, soft clips, all-low-quality, N bases, q < 6, each flag, unknown and
    missing read groups, other tags before RG:Z, QUAL '*', l_seq 0."""
    out = []
    g = rgs_ids

    def q(n, lo=2, hi=45):
        return [int(x) for x in rng.integers(lo, hi, n)]

    def rd(name, flag, pos, cigar, rg, quals=None, tags=b"", mut=0.05, seq=None):
        L = sum(n for n, op in cigar if op in (0, 1, 4, 7, 8))
        s = seq if seq is not None else bq.mutate(ref.seq(0, pos, L + 5), rng, mut)[:L].replace("N", "A")
        r = bq.make_rec(name, flag, 0 if not flag & 4 else -1, pos if not flag & 4 else -1, cigar, s, quals if quals is not None else q(L))
        return with_tags(r, tags + (rg_tag(rg) if rg is not None else b""))

    for k, rg in enumerate(g):
        out.append(rd("fwd%d" % k, 0, 1000 + k, [(100, 0)], rg))
        out.append(rd("rev%d" % k, 16, 1100, [(100, 0)], rg, mut=0.2))
        out.append(rd("second%d" % k, 0x1 | 0x80 | 0x10, 1200, [(90, 0)], rg))
        out.append(rd("second_fwd%d" % k, 0x1 | 0x80 | 0x20, 1250, [(90, 0)], rg))
        out.append(rd("first%d" % k, 0x1 | 0x40 | 0x20, 1300, [(90, 0)], rg))
    rg = g[0]
    out.append(rd("softclip", 0, 1400, [(10, 4), (70, 0), (20, 4)], rg))
    out.append(rd("softclip_rev", 16, 1500, [(5, 4), (90, 0), (5, 4)], rg))
    out.append(rd("all_low", 0, 1600, [(50, 0)], rg, quals=[2] * 50))
    out.append(rd("tails", 16, 1700, [(70, 0)], rg, quals=[0, 2, 1] + q(60, 6) + [2, 2, 0, 1, 2, 2, 1]))
    out.append(rd("n_bases", 0, 1800, [(60, 0)], rg, seq="ACGTN" * 12))
    out.append(rd("low_q", 0, 1900, [(64, 0)], rg, quals=[k % 9 for k in range(64)]))
    out.append(rd("q93", 0, 2000, [(40, 0)], rg, quals=[93] * 20 + [6] * 20))
    out.append(rd("len500", 0, 2100, [(500, 0)], rg))
    for fl in (0x4, 0x100, 0x800, 0x400, 0x200, 0x4 | 0x1 | 0x80):
        out.append(rd("flag_%x" % fl, fl, 2200, [(50, 0)] if not fl & 4 else [], rg, seq=None if not fl & 4 else "ACGTACGTAC" * 5, quals=q(50)))
    out.append(rd("other_tags", 0, 2300, [(50, 0)], rg, tags=b"NMC\x02" + b"XAZabc\0" + b"ZBBc\x03\x00\x00\x00\x01\x02\x03" + b"XFf\0\0\x80\x3f"))
    out.append(rd("no_rg", 0, 2400, [(50, 0)], None, tags=b"NMC\x01"))
    out.append(rd("unknown_rg", 0, 2500, [(50, 0)], "nosuchgroup"))
    out.append(with_tags(bq.make_rec("qual_star", 0, 0, 2600, [(50, 0)], ref.seq(0, 2600, 50).replace("N", "A"), None), rg_tag(rg)))
    out.append(with_tags(bq.make_rec("lseq0", 4, -1, -1, [], "", []), rg_tag(rg)))
    return out


def random_records(ref, rng, n, ids):
    recs = bq.random_records(ref, rng, n)
    out = []
    for k, r in enumerate(recs):
        x = rng.random()
        if x < 0.05:
            out.append(r)
        elif x < 0.08:
            out.append(with_tags(r, rg_tag("missing")))
        else:
            out.append(with_tags(r, (b"NMC\x01" if rng.random() < 0.5 else b"") + rg_tag(ids[int(rng.integers(0, len(ids)))])))
    return out


def apply_all(recs, ids, id_table, tabs):
    """-> (records, first error (index, kind 1 cycles / 2 quality) or None, recal, kept, changed)."""
    out, err, recal, kept, changed = [], None, 0, 0, 0
    for i, r in enumerate(recs):
        st, nr, ch = apply_record(r, ids, id_table, tabs)
        if st >= ERR_CYCLES:
            if err is None:
                err = (i, st - ERR_CYCLES + 1)
            out.append(r)
            continue
        recal += st == APPLY; kept += st == KEEP; changed += ch
        out.append(nr)
    return out, err, recal, kept, changed


# ---- the host emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("applybqsr_emul") / "libapplybqsremul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "host_emul", "applybqsr_emul.cpp"), "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.aq_parse.argtypes = [C.c_char_p, C.c_char_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_int64]
    lib.aq_parse.restype = C.c_int32
    lib.aq_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_void_p, C.c_void_p]
    lib.aq_read.argtypes = [C.c_char_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_char_p, C.c_int64]
    lib.aq_read.restype = C.c_int32
    lib.aq_free.argtypes = [C.c_void_p]
    return lib


def emul_dense(lib, text, path="t.txt", max_rg=8):
    """-> (read groups, P, D_ctx, D_cyc) as dense() gives them, or raises ValueError with the parser's message."""
    P, Cx, Y = np.zeros((max_rg, NQ)), np.zeros((max_rg, NQ, NCTX)), np.zeros((max_rg, NQ, NCYC))
    names, err = C.create_string_buffer(1 << 16), C.create_string_buffer(4096)
    n = lib.aq_parse(text.encode(), path.encode(), max_rg, P.ctypes.data, Cx.ctypes.data, Y.ctypes.data, names, 1 << 16, err, 4096)
    if n < 0:
        raise ValueError(err.value.decode())
    rgs = names.value.decode().split("\n")[:n] if n else []
    return rgs, P[:n], Cx[:n], Y[:n]


def emul_apply(lib, recs, ids, id_table, tabs):
    """-> apply_all's tuple, from the emulation."""
    data, starts = bq.flatten(recs)
    buf = np.frombuffer(bytearray(data), np.uint8).copy() if data else np.zeros(1, np.uint8)
    sb = starts if len(starts) else np.zeros(1, np.int64)
    tb = np.array(id_table if id_table else [0], np.int32)
    P, Cx, Y = (np.ascontiguousarray(x, np.float64) for x in tabs[1:])
    cnt, err = np.zeros(3, np.int64), np.zeros(2, np.int64)
    lib.aq_apply(buf.ctypes.data, sb.ctypes.data, len(starts), "\n".join(ids).encode(), tb.ctypes.data, len(ids), len(tabs[0]),
                 P.ctypes.data if P.size else None, Cx.ctypes.data if Cx.size else None, Y.ctypes.data if Y.size else None, cnt.ctypes.data, err.ctypes.data)
    raw = buf.tobytes()
    out = [raw[s:s + (starts[i + 1] if i + 1 < len(starts) else len(data)) - s] for i, s in enumerate(starts)]
    return out, (None if err[0] < 0 else (int(err[0]), int(err[1]))), int(cnt[0]), int(cnt[1]), int(cnt[2])


def emul_read(lib, path, window, threads=2):
    """The window reader over a BAM file -> (header text, records bytes, windows) or raises ValueError; also returns the warning."""
    recs, nrec, text, nw = C.c_void_p(), C.c_int64(), C.c_void_p(), C.c_int64()
    err, warn = C.create_string_buffer(4096), C.create_string_buffer(4096)
    rc = lib.aq_read(path.encode(), window, threads, C.byref(recs), C.byref(nrec), C.byref(text), C.byref(nw), err, warn, 4096)
    if rc:
        raise ValueError(err.value.decode())
    out = (C.string_at(text).decode(), C.string_at(recs, nrec.value) if nrec.value else b"", nw.value, warn.value.decode())
    lib.aq_free(recs); lib.aq_free(text)
    return out

"""Helpers of the bm2_markdup tests: its rule (bwa-mem2_b200/csrc/markdup_bam.h over markdup_device.cuh) restated in Python over the records
of several BAM files - merge, header, pairing, per-library keys, marking, read-group optical links and the metrics text - the host emulation
tests/host_emul/markdup_bam_emul.cpp, BAM files written from records, and random records of several lanes and libraries."""
import ctypes as C
import math, os, struct, subprocess, zlib
import numpy as np
import bam_util as bu
import bam_sort_util as bsu
import markdup_util as mu
import markdup_metrics_util as mm

ROOT = mu.ROOT
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_markdup")
REC_DT = np.dtype([("end", "<u8"), ("hash", "<u8"), ("score", "<i4"), ("kind", "<i4"), ("rg", "<i4"), ("lib", "<i4"), ("tile", "<i4"), ("x", "<i4"), ("y", "<i4"),
                   ("loc", "<i4")])
NONE, FRAG, HALF, UNMAPPED_HALF = 0, 1, 2, 3
UNKNOWN = "Unknown Library"


class MarkdupError(Exception):
    pass


# ---- files ----

def bgzf(data: bytes, member=65280) -> bytes:
    out = b""
    for at in range(0, len(data), member):
        chunk = data[at:at + member]
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        body = c.compress(chunk) + c.flush()
        out += b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(body) + 25) + body + \
            struct.pack("<II", zlib.crc32(chunk), len(chunk))
    return out + bu.EOF_BLOCK


def bam_bytes(text, refs, recs):
    h = b"BAM\x01" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for n, ln in refs:
        h += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", ln)
    return h + b"".join(recs)


def write_bam(path, text, refs, recs, member=65280):
    with open(path, "wb") as f:
        f.write(bgzf(bam_bytes(text, refs, recs), member))


def read_bam(path):
    """-> (header text, [(name, length)], [record bytes])"""
    raw = bu.inflate(open(path, "rb").read())
    lt = struct.unpack_from("<i", raw, 4)[0]
    text = raw[8:8 + lt].decode()
    at = 8 + lt
    n = struct.unpack_from("<i", raw, at)[0]; at += 4
    refs = []
    for _ in range(n):
        ln = struct.unpack_from("<i", raw, at)[0]
        refs.append((raw[at + 4:at + 3 + ln].decode(), struct.unpack_from("<i", raw, at + 4 + ln)[0]))
        at += 8 + ln
    return text, refs, [r for _, r in bu.records(raw[at:])]


def rec(rid, pos, flag, name, cigar=((60, 0),), mrid=-1, mpos=-1, rg=None, qual=30, extra=b""):
    tags = extra + (b"RGZ" + rg.encode() + b"\0" if rg is not None else b"")
    r = bsu.make_rec(rid, pos, flag, cigar, name.encode(), extra=tags)
    r = r[:24] + struct.pack("<ii", mrid, mpos) + r[32:]
    return mu.with_qual(r, qual) if qual != 30 else r


def key(r):
    rid, pos = struct.unpack_from("<ii", r, 4)
    flag = struct.unpack_from("<H", r, 18)[0]
    return ((rid & 0xFFFFFFFF) << 32) | (((pos + 1) & 0xFFFFFFFF) << 1) | ((flag >> 4) & 1)


def sort_recs(recs):
    return sorted(recs, key=key)


def header(rgs=(), pgs=(), cos=(), sq=(("c0", 100000), ("c1", 100000), ("c2", 100000)), so="coordinate"):
    t = "@HD\tVN:1.6\tSO:%s\n" % so + "".join("@SQ\tSN:%s\tLN:%d\n" % s for s in sq)
    t += "".join(l + "\n" for l in rgs) + "".join(l + "\n" for l in pgs) + "".join(l + "\n" for l in cos)
    return t, list(sq)


# ---- the rule ----

def tag(line, t):
    for f in line.split("\t")[1:]:
        if f.startswith(t):
            return f[len(t):]
    return ""


def set_tag(line, t, v):
    fs = line.split("\t")
    for k in range(1, len(fs)):
        if fs[k].startswith(t):
            fs[k] = t + v
            break
    return "\t".join(fs)


def merge_headers(names, texts, refs, cl):
    hd, sq, rg, pg, co = [], [], [], [], []
    rg_line, pg_lines, pg_ids, lbs, ids, first_last = {}, set(), set(), [], [], ""
    for i, t in enumerate(texts):
        if refs[i] != refs[0]:
            raise MarkdupError(names[i] + ": its @SQ lines differ")
        so, ren = None, {}
        for l in [x for x in t.rstrip("\0").split("\n") if x]:
            if l.startswith("@HD\t"):
                so = tag(l, "SO:") if so is None else so
                if i == 0 and not hd:
                    hd.append(l)
            elif l.startswith("@SQ\t"):
                if i == 0:
                    sq.append(l)
            elif l.startswith("@RG\t"):
                rid = tag(l, "ID:")
                if rid in rg_line:
                    if rg_line[rid] != l:
                        raise MarkdupError(names[i] + ": read group " + rid + " differs")
                    continue
                rg_line[rid] = l; rg.append(l); ids.append(rid); lbs.append(tag(l, "LB:"))
            elif l.startswith("@PG\t"):
                pid, pp = tag(l, "ID:"), tag(l, "PP:")
                m = set_tag(l, "PP:", ren[pp]) if pp and pp in ren else l
                if m in pg_lines:
                    ren[pid] = pid
                    if i == 0:
                        first_last = pid
                    continue
                nid, k = pid, 1
                while nid in pg_ids:
                    nid, k = "%s.%d" % (pid, k), k + 1
                if nid != pid:
                    m = set_tag(m, "ID:", nid)
                ren[pid] = nid
                if i == 0:
                    first_last = nid
                pg_lines.add(m); pg_ids.add(nid); pg.append(m)
            elif l.startswith("@CO\t"):
                co.append(l)
        if (so or "") != "coordinate":
            raise MarkdupError(names[i] + ": not coordinate-sorted")
    nid, k = "bm2_markdup", 1
    while nid in pg_ids:
        nid, k = "bm2_markdup.%d" % k, k + 1
    pg.append("@PG\tID:%s\tPN:bm2_markdup%s\tVN:b200-r2\tCL:%s" % (nid, "\tPP:" + first_last if first_last else "", cl))
    libs = sorted(set([x for x in lbs if x] + [UNKNOWN]), key=lambda s: s.encode())
    return "".join(l + "\n" for l in hd + sq + rg + pg + co), ids, [libs.index(x or UNKNOWN) for x in lbs], libs


def _rg_value(r):
    f = bu.fields(r)
    for tg, t, v in f["tags"]:
        if tg == "RG" and t == "Z":
            return v
    return None


def name_hash(name: bytes):
    """dup_name_hash: 64-bit FNV-1a"""
    h = 14695981039346656037
    for c in name:
        h = ((h ^ c) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def pair_halves(halves, names):
    """bm2_markdup_pair's rule: halves [(hash, rg, name bytes)] in ordinal order -> partner index or -1 of each; a half joins the first
    earlier unjoined half of the same (hash, read group) whose name is the same"""
    part, open_ = [-1] * len(halves), {}
    for i, (h, rg, nm) in enumerate(halves):
        k = (h, rg, nm)
        if k in open_:
            j = open_.pop(k)
            part[i], part[j] = j, i
        else:
            open_[k] = i
    return part


def record_info(r, ids, rg_lib, unknown):
    """mdb_record_kernel restated: a REC_DT tuple and the field dict"""
    f = bu.fields(r)
    v = _rg_value(r)
    rg, lib = len(ids), unknown
    if v is not None:
        rg = ids.index(v) if v in ids else -1
        lib = rg_lib[rg] if rg >= 0 else unknown
    kind, end, score, loc, t, x, y = NONE, 0, 0, 0, 0, 0, 0
    fl = f["flag"]
    if not fl & 0x900:
        if fl & 4:
            kind = UNMAPPED_HALF if (fl & 1) and not (fl & 8) else NONE
        else:
            kind = HALF if (fl & 1) and not (fl & 8) else FRAG
            end, score = mu.end_key(mu.end_of(f)), mu.read_score(f)
            if kind == HALF:
                lc = mm.location(f["qname"])
                if lc:
                    loc, (t, x, y) = mm.HAS, lc
    h = name_hash(f["qname"].encode()) if kind in (HALF, UNMAPPED_HALF) else 0
    return (end, h, score, kind, rg, lib, t, x, y, loc), f, v


def markdup(inputs, cl="bm2_markdup", args="", d=100):
    """inputs: [(name, header text, refs, [records in file order])] -> (output header text, marked records, metrics text, stats dict).
    Raises MarkdupError for every error of the rule."""
    names = [n for n, _, _, _ in inputs]
    text, ids, rg_lib, libs = merge_headers(names, [t for _, t, _, _ in inputs], [r for _, _, r, _ in inputs], cl)
    unknown = libs.index(UNKNOWN)
    for n, _, _, rs in inputs:
        for a, b in zip(rs, rs[1:]):
            if key(b) < key(a):
                raise MarkdupError(n + ": out of coordinate order")
    merged = sorted([(key(r), i, k, r) for i, (_, _, _, rs) in enumerate(inputs) for k, r in enumerate(rs)], key=lambda t: t[:3])
    recs = [t[3] for t in merged]
    nl = len(libs)
    pe, fe = [[] for _ in range(nl)], [[] for _ in range(nl)]
    locs = {}
    secsup, unmapped, seen = [0] * nl, [0] * nl, [False] * nl
    held, other, pairs = {}, {}, []
    for o, r in enumerate(recs):
        info, f, v = record_info(r, ids, rg_lib, unknown)
        end, _, score, kind, rg, lib = info[:6]
        seen[lib] = True
        if f["flag"] & 0x900:
            secsup[lib] += 1
        elif f["flag"] & 4:
            unmapped[lib] += 1
        if kind == FRAG:
            fe[lib].append((end, 0, o, score, mu.FRAG))
            continue
        if kind not in (HALF, UNMAPPED_HALF):
            continue
        rgk = rg if rg >= 0 else other.setdefault(v, len(ids) + 1 + len(other))
        k = (f["qname"], rgk)
        if k not in held:
            held[k] = (o, info, f)
            continue
        ho, hinfo, hf = held.pop(k)
        if hinfo[3] == UNMAPPED_HALF and kind == UNMAPPED_HALF:
            continue
        if hinfo[3] != kind:
            raise MarkdupError("read %s lacks flag 0x8, but its mate is unmapped" % f["qname"])
        ks, sc = [hinfo[0], end], [hinfo[2], score]
        pe[lib].append((min(ks), max(ks), ho, sc[0] + sc[1], mu.PAIR))
        fe[lib] += [(ks[j], 0, ho, sc[j], mu.PAIR_END) for j in range(2)]
        locs[ho] = (hinfo[9] | mm.pair_class([hf, f]) | (rgk << 2), hinfo[6], hinfo[7], hinfo[8])
        pairs.append((ho, o))
    bad = [v for v in held.values() if v[1][3] == HALF]
    if bad:
        raise MarkdupError("read %s: its mate never appears" % min(bad, key=lambda v: v[0])[2]["qname"])
    dups, rows = set(), []
    stats = dict(records=len(recs), pairs=sum(map(len, pe)), fragments=sum(e[4] == mu.FRAG for x in fe for e in x), dup_pair_templates=0,
                 dup_fragment_templates=0, dup_optical_pairs=0)
    for l in range(nl):
        pd, fd = mu.resolve(pe[l]), mu.resolve(fe[l])
        groups = {}
        for e in pe[l]:
            groups.setdefault(e[:2], []).append(locs[e[2]])
        opt = sum(mm.optical_count(g, d) for g in groups.values())
        dups |= set(pd) | set(fd)
        stats["dup_pair_templates"] += len(pd); stats["dup_fragment_templates"] += len(fd); stats["dup_optical_pairs"] += opt
        if seen[l]:
            rows.append((libs[l], dict(unpaired=sum(e[4] == mu.FRAG for e in fe[l]), pairs=len(pe[l]), secsup=secsup[l], unmapped=unmapped[l],
                                       unpaired_dups=len(fd), pair_dups=len(pd), optical=opt)))
    for a, b in pairs:
        if a in dups:
            dups.add(b)
    out = []
    for o, r in enumerate(recs):
        fl = struct.unpack_from("<H", r, 18)[0] & ~0x400
        out.append(mu.set_flag(r, fl | (0x400 if o in dups else 0)))
    stats["dup_records"] = sum(1 for o in range(len(recs)) if o in dups)
    stats["libraries"] = len(rows)
    return text, out, metrics_text(rows, args), stats


def metrics_text(rows, args):
    """rows: [(library, the seven counts as in markdup_metrics_util.metrics_text)] -> bm2_markdup's metrics file"""
    o = "## htsjdk.samtools.metrics.StringHeader\n# bm2_markdup%s\n\n" % ((" " + args) if args else "")
    o += "## METRICS CLASS\tpicard.sam.DuplicationMetrics\n" + "\t".join(mm.COLUMNS) + "\n"
    for lib, m in rows:
        L = mm.library_size(m["pairs"] - m["optical"], m["pairs"] - m["pair_dups"])
        den = m["unpaired"] + 2 * m["pairs"]
        pct = (m["unpaired_dups"] + 2 * m["pair_dups"]) / den if den else 0.0
        o += "\t".join([lib] + [str(m[k]) for k in ("unpaired", "pairs", "secsup", "unmapped", "unpaired_dups", "pair_dups", "optical")]
                       + [mm.fmt(pct), "" if L is None else str(L)]) + "\n"
    if len(rows) == 1:
        m = rows[0][1]
        L = mm.library_size(m["pairs"] - m["optical"], m["pairs"] - m["pair_dups"])
        if L is not None:
            o += "\n## HISTOGRAM\tjava.lang.Double\nBIN\tCoverageMult\n"
            for x in range(1, 101):
                o += "%d.0\t%s\n" % (x, mm.fmt(L * (1 - math.exp(-(x * m["pairs"]) / L)) / (m["pairs"] - m["pair_dups"])))
    return o


def markdup_files(paths, cl="bm2_markdup", args="", d=100):
    ins = []
    for p in paths:
        t, refs, rs = read_bam(p)
        ins.append((p, t, refs, rs))
    return markdup(ins, cl, args, d)


# ---- random records ----

def random_lanes(rng, n_pairs, lanes, dup_rate=0.3, contigs=3, span=20000):
    """Records of n_pairs pairs plus fragments, secondaries, supplementaries and unmapped mates, spread over lanes: [(rg id, library)].
    Duplicates are planted within a library (a copy of a pair or fragment in the same or another lane of its library), named near their
    original on its tile or elsewhere.  -> {rg id: [records]}, each lane's list unsorted."""
    out = {rg: [] for rg, _ in lanes}
    spots, used = [], set()

    def name(lane_i, t, x, y):
        return "M01:77:FC:%d:%d:%d:%d" % (lane_i + 1, t, x, y)

    def cig(rev):
        lc = int(rng.choice([0, 0, 3]))
        return ((lc, 4), (60 - lc, 0)) if lc and not rev else ((60 - lc, 0), (lc, 4)) if lc else ((60, 0),)

    k = 0
    for i in range(n_pairs):
        li = int(rng.integers(0, len(lanes)))
        rg, lib = lanes[li]
        if spots and rng.random() < dup_rate:
            s = spots[int(rng.integers(0, len(spots)))]
            same = [j for j, (_, lb) in enumerate(lanes) if lb == s["lib"]]
            li = same[int(rng.integers(0, len(same)))]
            rg = lanes[li][0]
            t, x, y = s["loc"]
            if rng.random() < 0.6:
                x, y = x + int(rng.integers(-80, 81)), y + int(rng.integers(-80, 81))
            else:
                t += 1
            a, b = s["a"], s["b"]
            kind = s["kind"]
        else:
            t, x, y = 1101 + int(rng.integers(0, 2)), int(rng.integers(1000, 20000)), int(rng.integers(1000, 20000))
            a = (int(rng.integers(0, contigs)), int(rng.integers(0, span)), int(rng.integers(0, 2)))
            b = (a[0] if rng.random() < 0.85 else int(rng.integers(0, contigs)), a[1] + int(rng.integers(-300, 600)), 1 - a[2])
            b = (b[0], max(b[1], 0), b[2])
            kind = int(rng.choice([0, 0, 0, 0, 1, 2]))          # 0 pair, 1 fragment, 2 mate unmapped
            spots.append(dict(lib=lib, loc=(t, x, y), a=a, b=b, kind=kind))
        while (li, t, x, y) in used:                              # names are unique within a lane
            x += 1
        used.add((li, t, x, y))
        nm = name(li, t, x, y) + ":%d" % k if rng.random() < 0.02 else name(li, t, x, y)
        k += 1
        q = int(rng.choice([30, 20, 35]))
        if kind == 0:
            fa, fb = 0x1 | 0x40 | (16 if a[2] else 0) | (32 if b[2] else 0), 0x1 | 0x80 | (16 if b[2] else 0) | (32 if a[2] else 0)
            out[rg].append(rec(a[0], a[1], fa, nm, cig(a[2]), b[0], b[1], rg, q))
            out[rg].append(rec(b[0], b[1], fb, nm, cig(b[2]), a[0], a[1], rg, q))
            if rng.random() < 0.1:
                out[rg].append(rec(a[0], a[1] + 40, 0x1 | 0x40 | 0x800, nm, ((30, 4), (30, 0)), b[0], b[1], rg))
            if rng.random() < 0.1:
                out[rg].append(rec(b[0], b[1] + 7, 0x1 | 0x80 | 0x100 | 0x400, nm, ((60, 0),), a[0], a[1], rg))
        elif kind == 1:
            out[rg].append(rec(a[0], a[1], 16 if a[2] else 0, nm, cig(a[2]), rg=rg, qual=q))
        else:
            out[rg].append(rec(a[0], a[1], 0x1 | 0x40 | 0x8 | (16 if a[2] else 0), nm, cig(a[2]), a[0], a[1], rg, q))
            out[rg].append(rec(a[0], a[1], 0x1 | 0x80 | 0x4 | 0x400, nm, (), a[0], a[1], rg))
    return out


# ---- the emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("markdup_bam_emul") / "libmdbemul.so")
    he = os.path.join(ROOT, "tests", "host_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + mu.CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(he, "markdup_bam_emul.cpp"), os.path.join(he, "markdup_metrics_emul.cpp"), os.path.join(he, "markdup_emul.cpp"),
                           os.path.join(he, "bam_sort_emul.cpp"), os.path.join(he, "bgzf_emul.cpp"), "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.mdb_emul_records.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.mdb_emul_pair.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.mdb_emul_resolve_ex.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.mdb_emul_run.argtypes = [C.c_char_p] * 6 + [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_char_p, C.c_int]
    return lib


STAT_NAMES = ("records", "pairs", "fragments", "pending_max", "dup_pair_templates", "dup_fragment_templates", "dup_records", "dup_optical_pairs",
              "dup_sig_runs", "dup_sig_bytes", "windows", "libraries")


def emul_run(lib, paths, out, metrics, bai="", args="", cl="bm2_markdup", threads=2, window=256 << 20, sig_bytes=1 << 30, d=100):
    """-> (exit code, message, stats dict)"""
    st = np.zeros(12, np.int64)
    err = C.create_string_buffer(4096)
    rc = lib.mdb_emul_run("\n".join(paths).encode(), out.encode(), metrics.encode(), bai.encode(), args.encode(), cl.encode(), threads, window,
                          sig_bytes, d, st.ctypes.data, err, 4096)
    return rc, err.value.decode(), dict(zip(STAT_NAMES, (int(v) for v in st)))


def emul_records(lib, recs, ids, libs, n_lib, unknown):
    data = b"".join(recs)
    starts = np.array(np.cumsum([0] + [len(r) for r in recs[:-1]]), np.int64) if recs else np.zeros(1, np.int64)
    out, cnt = np.zeros(max(len(recs), 1), REC_DT), np.zeros(2 * n_lib, np.int64)
    buf = np.frombuffer(data + b"\0", np.uint8)
    lib.mdb_emul_records(buf.ctypes.data, starts.ctypes.data, len(recs), "\n".join(ids).encode(), np.array(libs + [0], np.int32).ctypes.data, len(ids),
                         n_lib, unknown, out.ctypes.data, cnt.ctypes.data)
    return out[:len(recs)], cnt


HALF_DT = np.dtype([("hash", "<u8"), ("rg", "<i4"), ("name_len", "<i4"), ("name_off", "<i8")])


def halves_array(halves):
    """[(hash, rg, name bytes)] -> (HALF_DT array, names bytes)"""
    a, names = np.zeros(max(len(halves), 1), HALF_DT), b""
    for i, (h, rg, nm) in enumerate(halves):
        a[i] = (h, rg, len(nm), len(names))
        names += nm
    return a[:len(halves)], names


def emul_pair(lib, halves):
    a, names = halves_array(halves)
    out = np.zeros(max(len(halves), 1), np.int32)
    buf = np.frombuffer(names + b"\0", np.uint8)
    lib.mdb_emul_pair(np.ascontiguousarray(a).ctypes.data if len(halves) else None, len(halves), buf.ctypes.data, out.ctypes.data)
    return out[:len(halves)].tolist()


def emul_resolve_ex(lib, entries, d):
    e = np.ascontiguousarray(entries, mm.LOC_DT)
    dd, nd, no = np.zeros(max(len(e), 1), np.int64), C.c_int64(), C.c_int64()
    lib.mdb_emul_resolve_ex(e.ctypes.data, len(e), d, dd.ctypes.data, C.byref(nd), C.byref(no))
    return dd[:nd.value], no.value

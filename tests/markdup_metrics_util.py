"""Helpers of the duplication-metrics tests: the location, optical and metrics rules of bwa-mem2_b200/csrc/markdup_device.cuh and
markdup_metrics.h restated in Python, the host emulation tests/host_emul/markdup_metrics_emul.cpp, the metrics computed from a BAM's records,
and reads with planted duplicates under Illumina-style names."""
import ctypes as C
import math, os, subprocess
import numpy as np
import bam_util as bu
import markdup_util as mu

ROOT = mu.ROOT
CSRC = mu.CSRC
LOC_DT = np.dtype([("k1", "<u8"), ("k2", "<u8"), ("tid", "<i8"), ("score", "<i4"), ("kind", "<i4"), ("tile", "<i4"), ("x", "<i4"), ("y", "<i4"),
                   ("loc", "<i4")])
HAS, REV = 1, 2
MAX_SET = 300_000
COLUMNS = ["LIBRARY", "UNPAIRED_READS_EXAMINED", "READ_PAIRS_EXAMINED", "SECONDARY_OR_SUPPLEMENTARY_RDS", "UNMAPPED_READS", "UNPAIRED_READ_DUPLICATES",
           "READ_PAIR_DUPLICATES", "READ_PAIR_OPTICAL_DUPLICATES", "PERCENT_DUPLICATION", "ESTIMATED_LIBRARY_SIZE"]


# ---- the rule ----

def parse_int(field):
    """Picard's rapidParseInt: an optional '-', then the digits up to the first non-digit, as a wrapping Java int; None without a digit."""
    i, neg = 0, field[:1] == b"-"
    if neg:
        i = 1
    v, any_ = 0, False
    while i < len(field) and 48 <= field[i] <= 57:
        v = (v * 10 + field[i] - 48) & 0xFFFFFFFF
        any_ = True
        i += 1
    if not any_:
        return None
    if neg:
        v = (-v) & 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def location(name):
    """A QNAME (bytes or str) -> (tile, x, y), or None."""
    f = (name.encode() if isinstance(name, str) else name).split(b":")
    if len(f) not in (5, 7):
        return None
    v = [parse_int(x) for x in f[-3:]]
    return None if None in v else tuple(v)


def optical_count(members, d):
    """members: [(loc bits, tile, x, y)] of one pair group -> its optical count, by a breadth-first search over the link relation."""
    n = len(members)
    if n < 2 or n > MAX_SET:
        return 0
    a = np.array([m[:4] for m in members], np.int64).reshape(-1, 4)
    seen = np.zeros(n, bool)
    comps = 0
    for s in range(n):
        if seen[s]:
            continue
        comps += 1
        seen[s] = True
        if not a[s, 0] & HAS:
            continue
        todo = [s]
        while todo:
            i = todo.pop()
            nb = np.nonzero(~seen & (a[:, 0] & HAS != 0) & (a[:, 0] == a[i, 0]) & (a[:, 1] == a[i, 1]) & (np.abs(a[:, 2] - a[i, 2]) <= d)
                            & (np.abs(a[:, 3] - a[i, 3]) <= d))[0]
            seen[nb] = True
            todo += nb.tolist()
    return n - comps


def library_size(pairs, unique):
    """Picard's estimateLibrarySize; None when undefined."""
    if pairs <= 0 or pairs - unique <= 0:
        return None
    c, n = float(unique), float(pairs)
    f = lambda x: c / x - 1 + math.exp(-n / x)
    m, M = 1.0, 100.0
    while f(M * c) > 0:
        M *= 10.0
    for _ in range(40):
        r = (m + M) / 2.0
        u = f(r * c)
        if u == 0:
            break
        if u > 0:
            m = r
        else:
            M = r
    return int(c * (m + M) / 2.0)


def fmt(v):
    s = "%.6f" % v
    s = s.rstrip("0")
    return s[:-1] if s.endswith(".") else s


def metrics_text(m, args, library="Unknown Library"):
    """m: dict of the seven counts (unpaired, pairs, secsup, unmapped, unpaired_dups, pair_dups, optical) -> the file's text."""
    L = library_size(m["pairs"] - m["optical"], m["pairs"] - m["pair_dups"])
    den = m["unpaired"] + 2 * m["pairs"]
    pct = (m["unpaired_dups"] + 2 * m["pair_dups"]) / den if den else 0.0
    o = "## htsjdk.samtools.metrics.StringHeader\n# bm2_mem%s\n\n" % ((" " + args) if args else "")
    o += "## METRICS CLASS\tpicard.sam.DuplicationMetrics\n" + "\t".join(COLUMNS) + "\n"
    o += "\t".join([library] + [str(m[k]) for k in ("unpaired", "pairs", "secsup", "unmapped", "unpaired_dups", "pair_dups", "optical")]
                   + [fmt(pct), "" if L is None else str(L)]) + "\n"
    if L is not None:
        o += "\n## HISTOGRAM\tjava.lang.Double\nBIN\tCoverageMult\n"
        for x in range(1, 101):
            o += "%d.0\t%s\n" % (x, fmt(L * (1 - math.exp(-(x * m["pairs"]) / L)) / (m["pairs"] - m["pair_dups"])))
    return o


def pair_class(fs):
    """The class bits of a pair template from its two primaries' field dicts."""
    f = fs[0] if (fs[0]["flag"] & 0x40) or not (fs[1]["flag"] & 0x40) else fs[1]
    return REV if f["flag"] & 16 else 0


def metrics_of(templates, d):
    """templates: [(tid, [field dicts in record order])] -> the seven counts of the rule."""
    pe, fe, loc = [], [], {}
    secsup = unmapped = 0
    for tid, fs in templates:
        p, f = mu.template_entries(fs, tid)
        pe += p; fe += f
        for x in fs:
            secsup += (x["flag"] & 0x900) != 0
            unmapped += (x["flag"] & 0x900) == 0 and (x["flag"] & 4) != 0
        if p:
            prim = [x for x in fs if not x["flag"] & 0x900]
            lc = location(fs[0]["qname"])
            loc[tid] = ((HAS if lc else 0) | pair_class(prim),) + (lc or (0, 0, 0))
    groups = {}
    for e in pe:
        groups.setdefault((e[0], e[1]), []).append(loc[e[2]])
    return dict(unpaired=sum(e[4] == mu.FRAG for e in fe), pairs=len(pe), secsup=secsup, unmapped=unmapped,
                unpaired_dups=len(mu.resolve(fe)), pair_dups=len(mu.resolve(pe)), optical=sum(optical_count(g, d) for g in groups.values()))


def parse_metrics(text):
    """The file's value row as a dict, and its histogram rows."""
    lines = text.split("\n")
    k = lines.index("\t".join(COLUMNS))
    row = dict(zip(COLUMNS, lines[k + 1].split("\t")))
    hist = lines[lines.index("BIN\tCoverageMult") + 1:-1] if "BIN\tCoverageMult" in lines else []
    return row, hist


# ---- the emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("markdup_metrics_emul") / "libmmemul.so")
    he = os.path.join(ROOT, "tests", "host_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(he, "markdup_metrics_emul.cpp"), os.path.join(he, "markdup_emul.cpp"), os.path.join(he, "bam_sort_emul.cpp"),
                           os.path.join(he, "bgzf_emul.cpp"), "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.mm_optical_group.argtypes = [C.c_void_p, C.c_int64, C.c_int64]
    lib.mm_optical_group.restype = C.c_int64
    lib.mm_name_location.argtypes = [C.c_char_p, C.c_int, C.c_void_p]
    lib.mm_signatures_ex.argtypes = [C.c_void_p] * 4 + [C.c_int64] + [C.c_void_p] * 5
    lib.mm_resolve_ex.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.mm_metrics_text.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int64]
    lib.mm_metrics_text.restype = C.c_int64
    lib.mm_library_size.argtypes = [C.c_int64, C.c_int64]
    lib.mm_library_size.restype = C.c_int64
    return lib


def emul_location(lib, name):
    out = np.zeros(4, np.int32)
    lib.mm_name_location(name, len(name), out.ctypes.data)
    return tuple(int(v) for v in out[1:]) if out[0] else None


def members_array(members):
    a = np.zeros(max(len(members), 1), LOC_DT)
    for i, (loc, t, x, y) in enumerate(members):
        a[i]["kind"], a[i]["loc"], a[i]["tile"], a[i]["x"], a[i]["y"] = mu.PAIR, loc, t, x, y
    return a


def emul_optical(lib, members, d):
    a = members_array(members)
    return int(lib.mm_optical_group(a.ctypes.data, len(members), d))


def emul_signatures_ex(lib, data, first, ids):
    st = np.array([a for a, _ in bu.records(data)], np.int64)
    n = len(ids)
    p, f = np.zeros(max(n, 1), LOC_DT), np.zeros(max(2 * n, 1), mu.DUP_ENTRY_DT)
    np_, nf, counts = C.c_int64(), C.c_int64(), np.zeros(2, np.int64)
    lib.mm_signatures_ex(mu._buf(data).ctypes.data, mu._buf(st, np.int64).ctypes.data, mu._buf(first, np.int64).ctypes.data, mu._buf(ids, np.int64).ctypes.data,
                         n, p.ctypes.data, C.byref(np_), f.ctypes.data, C.byref(nf), counts.ctypes.data)
    return p[:np_.value], f[:nf.value], (int(counts[0]), int(counts[1]))


def emul_resolve_ex(lib, entries, d, resolve_=True):
    e = np.ascontiguousarray(entries, LOC_DT)
    srt, dd, nd, no = np.zeros(max(len(e), 1), LOC_DT), np.zeros(max(len(e), 1), np.int64), C.c_int64(), C.c_int64()
    lib.mm_resolve_ex(mu._buf(e, LOC_DT).ctypes.data, len(e), int(resolve_), d, srt.ctypes.data, dd.ctypes.data, C.byref(nd), C.byref(no))
    return (dd[:nd.value], no.value) if resolve_ else srt[:len(e)]


def emul_metrics_text(lib, m, args, library="Unknown Library"):
    v = np.array([m[k] for k in ("unpaired", "pairs", "secsup", "unmapped", "unpaired_dups", "pair_dups", "optical")], np.int64)
    buf = C.create_string_buffer(1 << 16)
    n = lib.mm_metrics_text(v.ctypes.data, library.encode(), args.encode(), buf, 1 << 16)
    assert n < 1 << 16
    return buf.value.decode()


# ---- located groups and records ----

def random_group(rng, n, d, classes=2, tiles=2, no_loc=0.1, spread=None):
    """n members around a few spots, with chains at about d apart."""
    spread = spread or 3 * d + 3
    out = []
    for _ in range(n):
        if rng.random() < no_loc:
            out.append((int(rng.integers(0, 2)) * REV, 0, 0, 0))
            continue
        out.append((HAS | int(rng.integers(0, classes)) * REV, 1101 + int(rng.integers(0, tiles)), int(rng.integers(0, spread)), int(rng.integers(0, spread))))
    return out


def located_entries(rng, n, n_groups, d):
    """Located pair entries of n_groups keys of random sizes; names parse into members of random_group."""
    keys = [(mu.end_key((0, int(k), 0)), mu.end_key((0, int(k) + 300, 1))) for k in rng.permutation(n * 4)[:n_groups]]
    tids = rng.permutation(n * 3)[:n]
    a = np.zeros(n, LOC_DT)
    mem = random_group(rng, n, d)
    for i in range(n):
        k1, k2 = keys[int(rng.integers(0, len(keys)))] if rng.random() < 0.97 else keys[0]
        a[i] = (k1, k2, int(tids[i]), int(rng.choice([0, 100, 2000])), mu.PAIR) + tuple(mem[i][1:]) + (mem[i][0],)
    return a


def illumina_name(tile, x, y, lane=1):
    return "M01:77:000000000-ABCDE:%d:%d:%d:%d" % (lane, tile, x, y)

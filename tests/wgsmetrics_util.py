"""Helpers of the bm2_wgsmetrics tests: Picard CollectWgsMetrics's loop restated in Python as the rule of bwa-mem2_b200/csrc/wgs_device.cuh
and wgs_metrics.h states it (per locus, the records in file order, a set of read names), the metrics file's text, small references written
as .ann / .amb files, crafted and random coordinate-sorted records, and the host emulation tests/host_emul/wgsmetrics_emul.cpp."""
import ctypes as C
import math, os, struct, subprocess
from collections import defaultdict
import numpy as np
import bam_util as bu
import bqsr_util as bq

ROOT, CSRC = bq.ROOT, bq.CSRC
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_wgsmetrics")
NOCALL = "Nn."
KX = (1, 5, 10, 15, 20, 25, 30, 40, 50, 60, 70, 80, 90, 100)
DEFAULTS = dict(min_mapq=20, min_baseq=20, cap=250, count_unpaired=False)


class Ref:
    """Contigs (names, lengths, offsets in the concatenated reference) and .amb holes (offset, length, letter)."""

    def __init__(self, contigs, holes=()):
        self.names = [n for n, _ in contigs]
        self.lens = [ln for _, ln in contigs]
        self.off = list(np.cumsum([0] + self.lens[:-1]))
        self.l_pac = int(sum(self.lens))
        self.holes = list(holes)
        self.nocall = np.zeros(self.l_pac, bool)
        for b, n, c in self.holes:
            if c in NOCALL:
                self.nocall[b:b + n] = True

    def nocall_ranges(self):
        return [(b, b + n) for b, n, c in self.holes if c in NOCALL]

    def write(self, prefix):
        ann = "%d %d 11\n" % (self.l_pac, len(self.names))
        for n, o, ln in zip(self.names, self.off, self.lens):
            ann += "0 %s (null)\n%d %d %d\n" % (n, o, ln, sum(1 for b, k, _ in self.holes if o <= b < o + ln))
        open(prefix + ".ann", "w").write(ann)
        amb = "%d %d %d\n" % (self.l_pac, len(self.names), len(self.holes)) + "".join("%d %d %s\n" % h for h in self.holes)
        open(prefix + ".amb", "w").write(amb)

    @staticmethod
    def read(prefix):
        lines = open(prefix + ".ann").read().split("\n")
        n = int(lines[0].split()[1])
        contigs = [(lines[1 + 2 * k].split()[1], int(lines[2 + 2 * k].split()[1])) for k in range(n)]
        amb = open(prefix + ".amb").read().split("\n")
        holes = [(int(a.split()[0]), int(a.split()[1]), a.split()[2]) for a in amb[1:1 + int(amb[0].split()[2])]]
        return Ref(contigs, holes)


# ---- the rule ----

def _blocks(cigar):
    """(ref offset, read offset, length) of the M / = / X blocks, the reference length, the query length."""
    out, r, q = [], 0, 0
    for op in cigar:
        n, t = op >> 4, op & 15
        if t in (0, 7, 8):
            out.append((r, q, n))
        if t in (0, 2, 3, 7, 8):
            r += n
        if t in (0, 1, 4, 7, 8):
            q += n
    return out, r, q


ERRORS = {1: "has no base qualities", 2: "does not lie inside a contig", 3: "has a CIGAR that does not match its record"}


def metrics(recs, ref, min_mapq=20, min_baseq=20, cap=250, count_unpaired=False):
    """Records in file order -> (hist [cap + 1], exc [MAPQ, DUPE, UNPAIRED, BASEQ, OVERLAP, CAPPED], counted, err) where err is None or
    (index, kind, name) of the first read error (then hist and exc are None)."""
    exc = [0] * 6
    loci = defaultdict(list)                              # g -> [(name, high quality)] in file order
    counted = 0
    for i, r in enumerate(recs):
        f = bu.fields(r)
        flag, rid, pos = f["flag"], f["rid"], f["pos"]
        if flag & 4 or rid == -1 or flag & 0x200:
            continue
        blocks, rlen, qlen = _blocks(f["cigar"])
        if rid < 0 or rid >= len(ref.names) or pos < 0 or pos + rlen > ref.lens[rid]:
            return None, None, counted, (i, 2, f["qname"])
        aligned = sum(n for _, _, n in blocks)
        if f["mapq"] < min_mapq:
            exc[0] += aligned; continue
        if flag & 0x400:
            exc[1] += aligned; continue
        if not count_unpaired and (not flag & 1 or flag & 8):
            exc[2] += aligned; continue
        if flag & 0x100:
            continue
        if f["l_seq"] == 0 or f["qual"][0] == 0xFF:
            return None, None, counted, (i, 1, f["qname"])
        if qlen != f["l_seq"]:
            return None, None, counted, (i, 3, f["qname"])
        counted += 1
        g0 = ref.off[rid] + pos
        for ro, qo, n in blocks:
            for k in range(n):
                loci[g0 + ro + k].append((f["qname"], f["qual"][qo + k] >= min_baseq and f["seq"][qo + k] != "N"))
    pile = np.zeros(ref.l_pac, np.int64)
    for g, lst in loci.items():                           # Picard's per-locus loop
        if ref.nocall[g]:
            continue
        names = set()
        for name, hq in lst:
            if not hq:
                exc[3] += 1
            elif name in names:
                exc[4] += 1
            else:
                names.add(name)
                pile[g] += 1
    p = pile[~ref.nocall]
    exc[5] = int(np.maximum(p - cap, 0).sum())
    hist = np.bincount(np.minimum(p, cap), minlength=cap + 1).astype(np.int64)
    return hist, exc, counted, None


def _d(v):
    s = "%.6f" % v
    s = s.rstrip("0")
    return s[:-1] if s.endswith(".") else s


def _median(pairs, n):
    if n <= 0:
        return 0.0

    def kth(k):
        s = 0
        for v, c in pairs:
            s += c
            if s >= k:
                return v
        return pairs[-1][0]
    return kth((n + 1) // 2) if n % 2 else (kth(n // 2) + kth(n // 2 + 1)) / 2.0


def text(hist, exc, args):
    """The metrics file, by the formulas of wgs_metrics.h."""
    cap = len(hist) - 1
    T = int(sum(int(h) for h in hist))
    Cv = int(sum(d * int(h) for d, h in enumerate(hist)))
    mean = Cv / T if T else 0.0
    ss = 0.0
    for d, h in enumerate(hist):
        ss += float(h) * ((float(d) - mean) * (float(d) - mean))
    sd = math.sqrt(ss / float(T - 1)) if T > 1 else 0.0
    v = [(float(d), int(h)) for d, h in enumerate(hist) if h]
    med = _median(v, T)
    mad = _median(sorted((abs(x - med), c) for x, c in v), T)
    excl = sum(exc)
    den = excl + Cv
    pct = lambda a, b: a / b if b else 0.0
    o = "## htsjdk.samtools.metrics.StringHeader\n# bm2_wgsmetrics" + (" " + args if args else "") + "\n\n"
    o += "## METRICS CLASS\tpicard.analysis.WgsMetrics\n"
    cols = ["GENOME_TERRITORY", "MEAN_COVERAGE", "SD_COVERAGE", "MEDIAN_COVERAGE", "MAD_COVERAGE", "PCT_EXC_MAPQ", "PCT_EXC_DUPE",
            "PCT_EXC_UNPAIRED", "PCT_EXC_BASEQ", "PCT_EXC_OVERLAP", "PCT_EXC_CAPPED", "PCT_EXC_TOTAL"] + ["PCT_%dX" % k for k in KX] + \
        ["HET_SNP_SENSITIVITY", "HET_SNP_Q"]
    o += "\t".join(cols) + "\n"
    vals = [str(T)] + [_d(x) for x in (mean, sd, med, mad)] + [_d(pct(x, den)) for x in exc] + [_d(pct(excl, den))]
    vals += [_d(pct(int(sum(int(h) for h in hist[k:])), T)) for k in KX] + ["", ""]
    o += "\t".join(vals) + "\n\n## HISTOGRAM\tjava.lang.Integer\ncoverage\thigh_quality_coverage_count\n"
    o += "".join("%d\t%d\n" % (d, h) for d, h in enumerate(hist))
    return o


# ---- records ----

def rec(name, flag, rid, pos, cigar, quals, seq=None, mapq=60, mrid=None, mpos=-1):
    """A record: cigar (length, op) pairs; quals a list (None: QUAL '*'); seq defaults to A's."""
    L = sum(n for n, op in cigar if op in (0, 1, 4, 7, 8))
    s = seq if seq is not None else "ACGT" * (L // 4) + "ACGT"[:L % 4]
    return bq.make_rec(name, flag, rid, pos, cigar, s, quals, mapq=mapq, mrid=(rid if flag & 1 else -1) if mrid is None else mrid, mpos=mpos)


def key(r):
    f = bu.fields(r)
    return ((f["rid"] & 0xFFFFFFFF) << 32) | (((f["pos"] + 1) & 0xFFFFFFFF) << 1) | (1 if f["flag"] & 16 else 0)


def sort_recs(recs):
    return [r for _, r in sorted(((key(r), i), r) for i, r in enumerate(recs))]


def random_pairs(ref, rng, n_pairs, max_len=150):
    """n_pairs random pairs (and some supplementaries) with random CIGARs (clips, insertions, deletions, skips), flags, MAPQs and qualities,
    coordinate-sorted.  Mates often overlap."""
    out = []

    def cigar(L):
        c, left = [], L
        if rng.random() < 0.2:
            s = int(rng.integers(1, 15)); c.append((s, 4)); left -= s
        tail = int(rng.integers(1, 15)) if rng.random() < 0.2 else 0
        left -= tail
        while left > 0:
            m = min(left, int(rng.integers(3, 60)))
            c.append((m, int(rng.choice([0, 0, 0, 7, 8])))); left -= m
            if left > 3 and rng.random() < 0.3:
                x = rng.random()
                if x < 0.4:
                    i = int(rng.integers(1, min(4, left))); c.append((i, 1)); left -= i
                elif x < 0.9:
                    c.append((int(rng.integers(1, 6)), 2))
                else:
                    c.append((int(rng.integers(1, 30)), 3))
        if tail:
            c.append((tail, 4))
        return c

    def one(name, flag, rid, pos, L, mapq):
        c = cigar(L)
        rl = sum(n for n, op in c if op in (0, 2, 3, 7, 8))
        pos = max(0, min(pos, ref.lens[rid] - rl))
        L = sum(n for n, op in c if op in (0, 1, 4, 7, 8))
        q = [int(x) for x in (rng.integers(0, 41, L) if rng.random() < 0.7 else rng.choice([2, 19, 20, 21, 37], L))]
        s = "".join("ACGTN"[int(x)] for x in rng.choice(5, L, p=[0.245, 0.245, 0.245, 0.245, 0.02]))
        return bq.make_rec(name, flag, rid, pos, c, s, q, mapq=mapq, mrid=rid if flag & 1 else -1)

    for k in range(n_pairs):
        rid = int(rng.integers(0, len(ref.names)))
        if ref.lens[rid] < 400:
            continue
        L1, L2 = int(rng.integers(20, max_len)), int(rng.integers(20, max_len))
        p1 = int(rng.integers(0, ref.lens[rid] - 1))
        p2 = max(0, p1 + int(rng.integers(-60, 200)))
        mq = lambda: int(rng.choice([0, 5, 19, 20, 60, 60, 60]))
        extra = int(rng.choice([0, 0, 0, 0, 0x400, 0x100, 0x200, 0x8]))
        f1, f2 = 0x1 | 0x40 | 0x20 | extra, 0x1 | 0x80 | 0x10 | (extra if extra != 0x100 else 0)
        if rng.random() < 0.05:
            f1 &= ~1
        name = "t%d" % k
        out.append(one(name, f1, rid, p1, L1, mq()))
        if rng.random() < 0.93:
            out.append(one(name, f2, rid, p2, L2, mq()))
        if rng.random() < 0.05:
            out.append(one(name, 0x1 | 0x800 | 0x40, rid, p1 + int(rng.integers(-30, 30)), int(rng.integers(20, 60)), 60))
        if rng.random() < 0.02:
            out.append(one("u%d" % k, 0x4, -1, -1, 30, 0))
    return sort_recs(out)


# ---- the host emulation ----

def build_emul(tmp_path_factory, collide=False):
    so = str(tmp_path_factory.mktemp("wgs_emul") / ("libwgsemul%s.so" % ("_c" if collide else "")))
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-I" + os.path.join(ROOT, "include")] +
                          (["-DWGS_HASH_MASK=0"] if collide else []) +
                          [os.path.join(ROOT, "tests", "host_emul", "wgsmetrics_emul.cpp"), "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.wm_new.restype = C.c_void_p
    lib.wm_new.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.wm_add.restype = C.c_int32
    lib.wm_add.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_char_p, C.c_int64]
    lib.wm_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.wm_free.argtypes = [C.c_void_p]
    lib.wm_text.restype = C.c_int64
    lib.wm_text.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_char_p, C.c_char_p, C.c_int64]
    lib.wm_run.restype = C.c_int32
    lib.wm_run.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_char_p, C.c_char_p,
                           C.c_int64, C.c_void_p]
    return lib


def windows(recs, sizes):
    """Split recs into windows of the given record counts (cycled)."""
    out, i, k = [], 0, 0
    while i < len(recs):
        n = sizes[k % len(sizes)]
        out.append(recs[i:i + n]); i += n; k += 1
    return out


def emul_run(lib, ref, wins, min_mapq=20, min_baseq=20, cap=250, count_unpaired=False, check_order=True):
    """The emulation's add per window, then finish -> (hist, exc, counted, None, records, carried_max), or (None, None, None, error message)."""
    off = np.array(ref.off, np.int64); ln = np.array(ref.lens, np.int32)
    nc = np.array(ref.nocall_ranges(), np.int64).reshape(-1)
    ncb = nc if len(nc) else np.zeros(2, np.int64)
    h = lib.wm_new(off.ctypes.data, ln.ctypes.data, len(off), ref.l_pac, ncb.ctypes.data, len(nc) // 2, min_mapq, min_baseq, cap, int(count_unpaired))
    try:
        err = C.create_string_buffer(4096)
        for w in wins:
            data, starts = bq.flatten(w)
            buf = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
            sb = starts if len(starts) else np.zeros(1, np.int64)
            if lib.wm_add(h, buf.ctypes.data, sb.ctypes.data, len(w), int(check_order), err, 4096):
                return None, None, None, err.value.decode()
        hist, exc, st = np.zeros(cap + 1, np.int64), np.zeros(6, np.int64), np.zeros(3, np.int64)
        lib.wm_finish(h, hist.ctypes.data, exc.ctypes.data, st.ctypes.data)
        return hist, [int(x) for x in exc], int(st[1]), None, int(st[0]), int(st[2])
    finally:
        lib.wm_free(h)


def emul_text(lib, hist, exc, args):
    hist = np.ascontiguousarray(hist, np.int64); e = np.array(exc, np.int64)
    n = lib.wm_text(hist.ctypes.data, len(hist) - 1, e.ctypes.data, args.encode(), None, 0)
    out = C.create_string_buffer(n + 1)
    lib.wm_text(hist.ctypes.data, len(hist) - 1, e.ctypes.data, args.encode(), out, n + 1)
    return out.value.decode()


def emul_tool(lib, prefix, bam, window=1 << 28, threads=2, min_mapq=20, min_baseq=20, cap=250, count_unpaired=False, args=""):
    """The emulated tool over files -> (text, stats) or raises ValueError with the error."""
    out = C.create_string_buffer(1 << 22)
    st = np.zeros(4, np.int64)
    rc = lib.wm_run(prefix.encode(), bam.encode(), window, threads, min_mapq, min_baseq, cap, int(count_unpaired), args.encode(), out, 1 << 22,
                    st.ctypes.data)
    if rc:
        raise ValueError(out.value.decode())
    return out.value.decode(), dict(records=int(st[0]), counted_records=int(st[1]), windows=int(st[2]), carried_max=int(st[3]))


def bam_bytes(ref, recs, text="@HD\tVN:1.6\tSO:coordinate\n", refs=None):
    """A BGZF BAM file of recs under a header whose reference list is ref's (or refs: [(name, length)])."""
    refs = refs if refs is not None else list(zip(ref.names, ref.lens))
    h = b"BAM\x01" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for n, ln in refs:
        h += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", ln)
    return bq.bgzf(h + b"".join(recs))

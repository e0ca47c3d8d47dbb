"""Helpers of the recalibration-table tests: the rule of bwa-mem2_b200/csrc/bqsr_device.cuh, the empirical quality and report text of
bqsr_report.h and the known-site bitsets of known_sites.h restated in Python, the host emulation tests/host_emul/bqsr_emul.cpp, BAM records
built from parts, crafted records for each rule and random ones."""
import ctypes as C
import gzip, math, os, struct, subprocess, zlib
import numpy as np
import bam_util as bu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bwa-mem2_b200", "csrc")
NQ, NCTX, NCYC, MAXC = 94, 16, 1001, 500
ERR_NAMES = {1: "no qualities", 2: "cycles", 3: "quality"}


# ---- the index ----

class Ref:
    """The forward codes, contigs and .amb holes of an index."""

    def __init__(self, prefix):
        lines = open(prefix + ".ann").read().split("\n")
        self.l_pac = int(lines[0].split()[0])
        n = int(lines[0].split()[1])
        self.names, self.off, self.lens = [], [], []
        for k in range(n):
            self.names.append(lines[1 + 2 * k].split()[1])
            o, ln = (int(x) for x in lines[2 + 2 * k].split()[:2])
            self.off.append(o); self.lens.append(ln)
        pac = np.frombuffer(open(prefix + ".pac", "rb").read(), np.uint8)
        i = np.arange(self.l_pac)
        self.codes = ((pac[i >> 2] >> ((3 - (i & 3)) * 2)) & 3).astype(np.uint8)
        amb = open(prefix + ".amb").read().split("\n")
        nh = int(amb[0].split()[2])
        self.holes = [(int(amb[1 + k].split()[0]), int(amb[1 + k].split()[0]) + int(amb[1 + k].split()[1])) for k in range(nh)]
        self.hole_mask = np.zeros(self.l_pac, bool)
        for b, e in self.holes:
            self.hole_mask[b:e] = True

    def seq(self, rid, pos, n):
        """The contig's bases [pos, pos + n) as ACGT (N inside holes)."""
        g = self.off[rid] + pos
        return "".join("N" if self.hole_mask[x] else "ACGT"[self.codes[x]] for x in range(g, g + n))


# ---- known sites ----

def sites_bits(ref, sites):
    """sites: [(rid, 1-based POS, REF length)] -> (covered, junction) as bool arrays over the reference."""
    cov, jun = np.zeros(ref.l_pac, bool), np.zeros(ref.l_pac, bool)
    for rid, p, n in sites:
        g = ref.off[rid] + p - 1
        cov[g:g + n] = True
        jun[g:g + n - 1] = True
    return cov, jun


def pack_bits(mask):
    w = np.zeros((len(mask) + 63) // 64 * 64, np.uint8)
    w[:len(mask)] = mask
    return np.packbits(w, bitorder="little").view("<u8").copy()


def vcf_text(ref, sites, header=True):
    out = "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n" if header else ""
    for rid, p, n in sites:
        r = ref.seq(rid, p - 1, n).replace("N", "A")
        out += "%s\t%d\t.\t%s\t%s\t.\tPASS\t.\n" % (ref.names[rid], p, r, "G" if r[0] != "G" else "C")
    return out


def bgzf(data: bytes) -> bytes:
    """BGZF members of at most 65280 input bytes each, and the end-of-file member."""
    out = b""
    for at in range(0, len(data), 65280):
        chunk = data[at:at + 65280]
        c = zlib.compressobj(6, zlib.DEFLATED, -15)
        body = c.compress(chunk) + c.flush()
        out += b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(body) + 25) + body + \
            struct.pack("<II", zlib.crc32(chunk), len(chunk))
    return out + bu.EOF_BLOCK


def random_sites(ref, rng, every=30):
    sites = []
    for rid, ln in enumerate(ref.lens):
        for p in np.sort(rng.choice(np.arange(1, ln - 5), size=max(ln // every, 1), replace=False)):
            sites.append((rid, int(p), int(rng.choice([1, 1, 1, 2, 3, 4]))))
    return sites


# ---- the rule ----

def _code(c):
    return "ACGT".index(c) if c in "ACGT" else 4


def count(recs, ref, cov, jun):
    """Records (bytes) -> dict of the dense tables (qual_*, ctx_*, cyc_*), reads, bases, err (index, kind) or None."""
    t = dict(qual_obs=np.zeros(NQ, np.int64), qual_err=np.zeros(NQ, np.int64), ctx_obs=np.zeros((NQ, NCTX), np.int64),
             ctx_err=np.zeros((NQ, NCTX), np.int64), cyc_obs=np.zeros((NQ, NCYC), np.int64), cyc_err=np.zeros((NQ, NCYC), np.int64),
             reads=0, bases=0, err=None)
    for i, r in enumerate(recs):
        st, bases = record_bases(r, ref, cov, jun)
        if st in (1, 2, 3):
            if t["err"] is None:
                t["err"] = (i, st)
            continue
        if st != 0:
            continue
        t["reads"] += 1
        for q, cx, cyc, e in bases:
            t["bases"] += 1
            t["qual_obs"][q] += 1; t["qual_err"][q] += e
            if cx is not None:
                t["ctx_obs"][q, cx] += 1; t["ctx_err"][q, cx] += e
            t["cyc_obs"][q, cyc + MAXC] += 1; t["cyc_err"][q, cyc + MAXC] += e
    return t


def record_bases(rec, ref, cov, jun):
    """One record -> (status, [(quality, context or None, cycle, error)]): status 0 counted, 1 no qualities, 2 over 500 cycles, 3 a quality
    above 93, 4 filtered, 5 empty after clipping."""
    f = bu.fields(rec)
    flag, cig, L0 = f["flag"], [(c >> 4, c & 15) for c in f["cigar"]], f["l_seq"]
    if flag & (0x4 | 0x100 | 0x800 | 0x400 | 0x200) or f["mapq"] in (0, 255) or not 0 <= f["rid"] < len(ref.names) or not cig or L0 <= 0:
        return 4, []
    qual = f["qual"]
    if qual[0] == 0xFF:
        return 1, []
    rlen = sum(n for n, op in cig if op in (0, 2, 3, 7, 8))
    sl = sr = 0
    seen = False
    for n, op in cig:
        if op == 4:
            if seen:
                sr += n
            else:
                sl += n
        elif op != 5:
            seen = True
    lo, hi = sl, L0 - sr
    rev = bool(flag & 16)
    start, end, ms, T = f["pos"] + 1, f["pos"] + rlen, f["next_pos"] + 1, f["tlen"]
    aligned, k, g = [], 0, start
    for n, op in cig:
        if op in (0, 7, 8):
            aligned += [(k + j, g + j) for j in range(n)]
            k += n; g += n
        elif op in (1, 4):
            k += n
        elif op in (2, 3):
            g += n
    if T != 0 and flag & 1 and not flag & 4 and not flag & 8 and bool(flag & 16) != bool(flag & 32) and (end > ms if rev else start <= ms + T):
        b = ms - 1 if rev else start + abs(T)
        if start <= b <= end:
            if rev:
                ks = [kk for kk, p in aligned if p <= b]
                lo = max(lo, max(ks) + 1 if ks else 0)
            else:
                ks = [kk for kk, p in aligned if p >= b]
                hi = min(hi, min(ks) if ks else L0)
    if hi <= lo:
        return 5, []
    if hi - lo > 500:
        return 2, []
    if any(qual[k] > 93 for k in range(lo, hi)):
        return 3, []
    good = [k for k in range(lo, hi) if qual[k] > 2]
    tl, tr = (good[0], good[-1] + 1) if good else (hi, hi)
    seq = f["seq"]
    letter = lambda k: 4 if k < tl or k >= tr else _code(seq[k])
    g0 = ref.off[f["rid"]] + f["pos"]
    out, k, g = [], 0, g0
    f_ = -1 if flag & 1 and flag & 0x80 else 1
    for n, op in cig:
        if op in (0, 7, 8, 1):
            for j in range(n):
                kk = k + j
                if not lo <= kk < hi:
                    continue
                ins = op == 1
                gg = g - 1 if ins else g + j
                b, q = _code(seq[kk]), qual[kk]
                if b == 4 or q < 6:
                    continue
                if ins and (0 <= gg and gg + 1 < ref.l_pac and jun[gg]) or (not ins and cov[gg]):
                    continue
                e = 0 if ins else int((4 if ref.hole_mask[gg] else int(ref.codes[gg])) != b)
                i, Lc = kk - lo, hi - lo
                cyc = (Lc - i if rev else i + 1) * f_
                if not rev:
                    pair = None if kk == lo else (letter(kk - 1), letter(kk))
                else:
                    pair = None if kk == hi - 1 else tuple(4 if x == 4 else 3 - x for x in (letter(kk + 1), letter(kk)))
                cx = None if pair is None or 4 in pair else pair[0] * 4 + pair[1]
                out.append((int(q), cx, cyc, e))
            k += n
            if op != 1:
                g += n
        elif op == 4:
            k += n
        elif op in (2, 3):
            g += n
    return 0, out


# ---- empirical quality and the report ----

def empirical_q(n, e, prior):
    N, E = n + 2, e + 1
    kmax = 2147483646
    if N > kmax:
        frac = kmax / N
        E = math.floor(E * frac + 0.5)
        N = kmax
    best, arg = 0.0, 0
    for Q in range(61):
        d = min(abs(int(Q - prior)), 40)
        x = 0.9 * math.exp(-(d * d) / 0.5)
        lp = math.log10(x) if x > 0 else -math.inf                      # C's log10(0)
        l10p = Q / -10.0
        one = 1.0 - 10.0 ** l10p
        ll = E * l10p + (N - E) * (math.log10(one) if one > 0 else -math.inf)
        if not math.isfinite(ll):
            ll = -1.7976931348623157e308
        v = lp + ll
        if Q == 0 or v > best:
            best, arg = v, Q
    return min(arg, 93)


ARGUMENTS = [("binary_tag_name", "null"), ("covariate", "ReadGroupCovariate,QualityScoreCovariate,ContextCovariate,CycleCovariate"),
             ("default_platform", "null"), ("deletions_default_quality", "45"), ("force_platform", "null"), ("indels_context_size", "3"),
             ("insertions_default_quality", "45"), ("low_quality_tail", "2"), ("maximum_cycle_value", "500"), ("mismatches_context_size", "2"),
             ("mismatches_default_quality", "-1"), ("no_standard_covs", "false"), ("quantizing_levels", "16"), ("recalibration_report", "null"),
             ("run_without_dbsnp", "false"), ("solid_nocall_strategy", "THROW_EXCEPTION"), ("solid_recal_mode", "SET_Q_ZERO")]


def _table(name, desc, cols, rows):
    o = "#:GATKTable:%d:%d%s:;\n#:GATKTable:%s:%s\n" % (len(cols), len(rows), "".join(":" + f for _, f in cols), name, desc)
    w = [max([len(c)] + [len(r[k]) for r in rows]) for k, (c, _) in enumerate(cols)]
    for r in [[c for c, _ in cols]] + rows:
        o += "  ".join(x.ljust(w[k]) if cols[k][1] == "%s" else x.rjust(w[k]) for k, x in enumerate(r)) + "\n"
    return o + "\n"


def report_text(t, rg):
    o = "#:GATKReport.v1.1:5\n"
    o += _table("Arguments", "Recalibration argument collection values used in this run", [("Argument", "%s"), ("Value", "%s")],
                [list(a) for a in ARGUMENTS])
    o += _table("Quantized", "Quality quantization map", [("QualityScore", "%d"), ("Count", "%d"), ("QuantizedScore", "%d")],
                [[str(q), str(int(t["qual_obs"][q])), str(q)] for q in range(NQ)])
    N, E, s = int(t["qual_obs"].sum()), int(t["qual_err"].sum()), 0.0
    for q in range(NQ):
        s += float(t["qual_obs"][q]) * 10.0 ** (q / -10.0)
    rows0 = []
    if N:
        qr = -10.0 * math.log10(s / N)
        rows0.append([rg, "M", "%.4f" % empirical_q(N, E, qr), "%.4f" % qr, str(N), "%.2f" % E])
    o += _table("RecalTable0", "", [("ReadGroup", "%s"), ("EventType", "%s"), ("EmpiricalQuality", "%.4f"), ("EstimatedQReported", "%.4f"),
                                    ("Observations", "%d"), ("Errors", "%.2f")], rows0)
    rows1, rows2 = [], []
    for q in range(NQ):
        n, e = int(t["qual_obs"][q]), int(t["qual_err"][q])
        if n:
            rows1.append([rg, str(q), "M", "%.4f" % empirical_q(n, e, q), str(n), "%.2f" % e])
        for c in range(NCTX):
            n, e = int(t["ctx_obs"][q, c]), int(t["ctx_err"][q, c])
            if n:
                rows2.append([rg, str(q), "ACGT"[c >> 2] + "ACGT"[c & 3], "Context", "M", "%.4f" % empirical_q(n, e, q), str(n), "%.2f" % e])
        for y in range(NCYC):
            n, e = int(t["cyc_obs"][q, y]), int(t["cyc_err"][q, y])
            if n:
                rows2.append([rg, str(q), str(y - MAXC), "Cycle", "M", "%.4f" % empirical_q(n, e, q), str(n), "%.2f" % e])
    o += _table("RecalTable1", "", [("ReadGroup", "%s"), ("QualityScore", "%d"), ("EventType", "%s"), ("EmpiricalQuality", "%.4f"),
                                    ("Observations", "%d"), ("Errors", "%.2f")], rows1)
    o += _table("RecalTable2", "", [("ReadGroup", "%s"), ("QualityScore", "%d"), ("CovariateValue", "%s"), ("CovariateName", "%s"),
                                    ("EventType", "%s"), ("EmpiricalQuality", "%.4f"), ("Observations", "%d"), ("Errors", "%.2f")], rows2)
    return o


def read_group(line):
    f = dict(x.split(":", 1) for x in line.replace("\\t", "\t").split("\t")[1:] if ":" in x)
    return f.get("PU") or f.get("ID")


# ---- the host emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bqsr_emul") / "libbqsremul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "host_emul", "bqsr_emul.cpp"), "-o", so, "-lz"])
    lib = C.CDLL(so)
    lib.bqsr_emul_count.argtypes = [C.c_void_p] * 2 + [C.c_int64] + [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32] + [C.c_void_p] * 3 + \
        [C.c_int64] + [C.c_void_p] * 8
    lib.bqsr_emul_empirical.argtypes = [C.c_int64, C.c_int64, C.c_double]
    lib.bqsr_emul_report.argtypes = [C.c_char_p] + [C.c_void_p] * 6
    lib.bqsr_emul_report.restype = C.c_void_p
    lib.bqsr_emul_read_group.argtypes = [C.c_char_p]
    lib.bqsr_emul_read_group.restype = C.c_void_p
    lib.bqsr_emul_sites.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int64]
    lib.bqsr_emul_sites.restype = C.c_int64
    lib.bqsr_emul_free.argtypes = [C.c_void_p]
    return lib


def _z(dt, shape):
    return np.zeros(shape, dt)


def emul_count(lib, data, starts, ref, cov, jun):
    starts = np.ascontiguousarray(starts, np.int64)
    buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
    sb = starts if len(starts) else np.zeros(1, np.int64)
    cw, jw = pack_bits(cov), pack_bits(jun)
    holes = np.array(ref.holes, np.int64).reshape(-1) if ref.holes else np.zeros(2, np.int64)
    off = np.array(ref.off, np.int64)
    t = dict(qual_obs=_z(np.int64, NQ), qual_err=_z(np.int64, NQ), ctx_obs=_z(np.int64, (NQ, NCTX)), ctx_err=_z(np.int64, (NQ, NCTX)),
             cyc_obs=_z(np.int64, (NQ, NCYC)), cyc_err=_z(np.int64, (NQ, NCYC)))
    rb, err = np.zeros(2, np.int64), np.zeros(2, np.int64)
    lib.bqsr_emul_count(buf.ctypes.data, sb.ctypes.data, len(starts), ref.codes.ctypes.data, ref.l_pac, off.ctypes.data, len(ref.off),
                        cw.ctypes.data, jw.ctypes.data, holes.ctypes.data, len(ref.holes),
                        *(t[k].ctypes.data for k in ("qual_obs", "qual_err", "ctx_obs", "ctx_err", "cyc_obs", "cyc_err")), rb.ctypes.data, err.ctypes.data)
    t.update(reads=int(rb[0]), bases=int(rb[1]), err=None if err[0] < 0 else (int(err[0]), int(err[1])))
    return t


def emul_report(lib, t, rg):
    p = lib.bqsr_emul_report(rg.encode(), *(np.ascontiguousarray(t[k], np.int64).ctypes.data
                                            for k in ("qual_obs", "qual_err", "ctx_obs", "ctx_err", "cyc_obs", "cyc_err")))
    s = C.string_at(p).decode()
    lib.bqsr_emul_free(p)
    return s


def emul_read_group(lib, line):
    p = lib.bqsr_emul_read_group(line.encode())
    s = C.string_at(p).decode()
    lib.bqsr_emul_free(p)
    return s


def emul_sites(lib, paths, ref):
    """-> (covered, junction, records) as bool arrays, or raises ValueError with the reader's message."""
    words = (ref.l_pac + 63) // 64
    cw, jw = np.zeros(words, np.uint64), np.zeros(words, np.uint64)
    err = C.create_string_buffer(4096)
    off, ln = np.array(ref.off, np.int64), np.array(ref.lens, np.int64)
    n = lib.bqsr_emul_sites("\n".join(paths).encode(), "\n".join(ref.names).encode(), off.ctypes.data, ln.ctypes.data, len(ref.names), ref.l_pac,
                            cw.ctypes.data, jw.ctypes.data, err, 4096)
    if n < 0:
        raise ValueError(err.value.decode())
    unpack = lambda w: np.unpackbits(w.view(np.uint8), bitorder="little")[:ref.l_pac].astype(bool)
    return unpack(cw), unpack(jw), n


def same_tables(a, b):
    keys = ("qual_obs", "qual_err", "ctx_obs", "ctx_err", "cyc_obs", "cyc_err")
    return all(np.array_equal(np.asarray(a[k]).reshape(-1), np.asarray(b[k]).reshape(-1)) for k in keys) and a["reads"] == b["reads"] and \
        a["bases"] == b["bases"]


# ---- records ----

def make_rec(name, flag, rid, pos, cigar, seq, qual, mapq=60, mrid=-1, mpos=-1, tlen=0):
    """One BAM record; cigar: (length, op) pairs; seq: a string; qual: a list of qualities, or None for QUAL '*'."""
    ops = [(n << 4) | op for n, op in cigar]
    L = len(seq)
    end = pos + (sum(n for n, op in cigar if op in (0, 2, 3, 7, 8)) or 1)
    bin_ = bu.reg2bin(pos, end) if rid >= 0 and pos >= 0 else 4680
    sb = bytearray((L + 1) // 2)
    for k, c in enumerate(seq):
        sb[k // 2] |= "=ACMGRSVTWYHKDBN".index(c) << (4 * (1 - k % 2))
    q = bytes([0xFF] * L) if qual is None else bytes(qual)
    nm = name.encode()
    body = struct.pack("<iiBBHHHiiii", rid, pos, len(nm) + 1, mapq, bin_, len(ops), flag, L, mrid, mpos, tlen)
    body += nm + b"\0" + struct.pack("<%dI" % len(ops), *ops) + bytes(sb) + q
    return struct.pack("<i", len(body)) + body


def flatten(recs):
    data, starts = b"", []
    for r in recs:
        starts.append(len(data)); data += r
    return data, np.array(starts, np.int64)


def mutate(s, rng, rate):
    return "".join("ACGT"[("ACGT".index(c) + 1 + int(rng.integers(0, 3))) % 4] if c in "ACGT" and rng.random() < rate else c for c in s)


def crafted(ref, rng):
    """Records for each rule: soft clips, adaptor clipping of both strands (overlapping pairs, T = 0, same strand, boundary outside), a read
    clipped to nothing, indels next to and inside sites, N bases, qualities 0..5, low-quality tails, reverse contexts, both mates' cycles, a
    read over an .amb hole, every excluded flag and MAPQ 0 / 255."""
    out = []
    rid = 0
    hole_b = ref.holes[0][0] - ref.off[[k for k in range(len(ref.off)) if ref.off[k] <= ref.holes[0][0]][-1]]
    hole_rid = [k for k in range(len(ref.off)) if ref.off[k] <= ref.holes[0][0]][-1]

    def q(n, lo=2, hi=41):
        return [int(x) for x in rng.integers(lo, hi, n)]

    def rd(name, flag, pos, cigar, mut=0.05, quals=None, r=rid, **kw):
        L = sum(n for n, op in cigar if op in (0, 1, 4, 7, 8))
        s = mutate(ref.seq(r, pos, L + 20), rng, mut)[:L].replace("N", "A")
        return make_rec(name, flag, r, pos, cigar, s, quals if quals is not None else q(L), **kw)

    out.append(rd("softclip_both", 0, 1000, [(7, 4), (80, 0), (13, 4)]))
    out.append(rd("softclip_rev", 16, 1100, [(3, 4), (90, 0), (9, 4)]))
    for name, flag, pos, mpos, tlen in [("adapt_fwd", 0x1 | 0x2 | 0x20 | 0x40, 2000, 2030, 90), ("adapt_rev", 0x1 | 0x2 | 0x10 | 0x80, 1990, 2000, -90),
                                        ("adapt_fwd_long", 0x1 | 0x2 | 0x20 | 0x40, 2200, 2300, 400), ("adapt_rev_outside", 0x1 | 0x10 | 0x80, 2500, 2400, -300),
                                        ("adapt_t0", 0x1 | 0x20 | 0x40, 2600, 2610, 0), ("adapt_same_strand", 0x1 | 0x40, 2700, 2710, 60),
                                        ("adapt_mate_unmapped", 0x1 | 0x8 | 0x20 | 0x40, 2800, 2810, 60), ("adapt_rev_sc", 0x1 | 0x10 | 0x80, 2905, 2900, -70),
                                        ("adapt_fwd_sc", 0x1 | 0x20 | 0x40, 3000, 3010, 50)]:
        cig = [(100, 0)] if "sc" not in name else [(5, 4), (90, 0), (5, 4)]
        out.append(rd(name, flag, pos, cig, mpos=mpos, mrid=rid, tlen=tlen))
    out.append(rd("clipped_to_nothing", 0, 3500, [(50, 4), (10, 2), (50, 4)]))
    out.append(rd("adapt_rev_two_left", 0x1 | 0x10 | 0x80, 3500, [(60, 0), (40, 4)], mpos=3558, mrid=rid, tlen=-20))
    out.append(rd("adapt_fwd_first", 0x1 | 0x20 | 0x40, 3600, [(100, 0)], mpos=3500, mrid=rid, tlen=-1))
    for k, cig in enumerate([[(40, 0), (3, 1), (40, 0)], [(40, 0), (4, 2), (40, 0)], [(20, 0), (1, 1), (20, 0), (2, 2), (30, 0)],
                             [(2, 4), (3, 1), (60, 0)], [(60, 0), (2, 1), (3, 4)]]):
        out.append(rd("indel%d" % k, 16 * (k % 2), 5000 + 13 * k, cig))
    out.append(make_rec("n_bases", 0, rid, 6000, [(60, 0)], "ACGTN" * 12, q(60)))
    out.append(rd("low_quals", 0, 6100, [(70, 0)], quals=[k % 8 for k in range(70)]))
    out.append(rd("tails", 0, 6200, [(70, 0)], quals=[2, 1, 0, 2] + q(60, 6) + [2, 2, 1, 0, 2, 2]))
    out.append(rd("tails_rev", 16, 6300, [(70, 0)], quals=[0, 2] + q(62, 6) + [1, 2, 2, 2, 0, 1]))
    out.append(rd("all_tail", 0, 6400, [(30, 0)], quals=[2] * 30))
    out.append(rd("rev_context", 16, 6500, [(100, 0)], mut=0.2))
    out.append(rd("first_of_pair", 0x1 | 0x40 | 0x20, 6600, [(100, 0)], mrid=rid, mpos=6800, tlen=300))
    out.append(rd("second_of_pair", 0x1 | 0x80 | 0x10, 6800, [(100, 0)], mrid=rid, mpos=6600, tlen=-300))
    out.append(rd("second_fwd", 0x1 | 0x80 | 0x20, 6900, [(100, 0)], mrid=rid, mpos=7100, tlen=300))
    out.append(rd("hole", 0, max(hole_b - 40, 0), [(100, 0)], r=hole_rid))
    out.append(rd("hole_rev", 16, hole_b + 5, [(30, 0), (2, 1), (30, 0)], r=hole_rid))
    for fl in (0x4, 0x100, 0x800, 0x400, 0x200):
        out.append(rd("flag_%x" % fl, fl, 7000, [(50, 0)]))
    out.append(rd("mapq0", 0, 7000, [(50, 0)], mapq=0))
    out.append(rd("mapq255", 0, 7000, [(50, 0)], mapq=255))
    out.append(rd("hard_clip", 0, 7100, [(10, 5), (50, 0), (3, 5)]))
    out.append(rd("eq_x", 0, 7200, [(20, 7), (1, 8), (20, 0)], mut=0))
    return out


def random_records(ref, rng, n):
    out = []
    for k in range(n):
        rid = int(rng.integers(0, len(ref.names)))
        L = int(rng.choice([50, 100, 151, 250]))
        cig, left = [], L
        if rng.random() < 0.3:
            s = int(rng.integers(1, 20)); cig.append((s, 4)); left -= s
        tail = int(rng.integers(1, 20)) if rng.random() < 0.3 else 0
        left -= tail
        while left > 0:
            m = min(left, int(rng.integers(5, 80)))
            cig.append((m, 0)); left -= m
            if left > 3 and rng.random() < 0.3:
                if rng.random() < 0.5:
                    i = int(rng.integers(1, min(4, left))); cig.append((i, 1)); left -= i
                else:
                    cig.append((int(rng.integers(1, 5)), 2))
        if tail:
            cig.append((tail, 4))
        while cig[-1][1] != 0 and cig[-1][1] != 4:
            cig.pop()
        L = sum(n_ for n_, op in cig if op in (0, 1, 4))
        rl = sum(n_ for n_, op in cig if op in (0, 2))
        pos = int(rng.integers(0, ref.lens[rid] - rl - 1))
        s = mutate(ref.seq(rid, pos, min(L, ref.lens[rid] - pos)).ljust(L, "A"), rng, 0.03).replace("N", "C")
        s = "".join("N" if rng.random() < 0.005 else c for c in s)
        flag = int(rng.choice([0, 16, 0x1 | 0x40 | 0x20, 0x1 | 0x80 | 0x10, 0x1 | 0x40 | 0x10, 0x1 | 0x80 | 0x20, 0x1 | 0x40, 0x400, 0x100, 0x1 | 0x8 | 0x40]))
        mpos, tlen = -1, 0
        if flag & 1:
            mpos = max(0, pos + int(rng.integers(-300, 300)))
            tlen = int(rng.integers(-500, 500))
        qual = [int(x) for x in rng.integers(0, 42, L)] if rng.random() < 0.5 else [int(x) for x in rng.choice([2, 12, 23, 37], L)]
        out.append(make_rec("r%d" % k, flag, rid, pos, cig, s, qual, mapq=int(rng.choice([0, 5, 60, 60])), mrid=rid if flag & 1 else -1, mpos=mpos,
                            tlen=tlen))
    return out

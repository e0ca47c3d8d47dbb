"""Helpers of the bm2_multiplemetrics tests: Picard CollectAlignmentSummaryMetrics's and CollectInsertSizeMetrics's per-record loops restated
in Python as the README states the rule (record by record, no code shared with bwa-mem2_b200/csrc/mm_device.cuh or mm_metrics.h), the two
files' text, small references written as .ann / .amb / .pac files, crafted and random records in any order, and the host emulation
tests/host_emul/multiplemetrics_emul.cpp."""
import ctypes as C
import math, os, struct, subprocess
from collections import Counter
import numpy as np
import bam_util as bu
import bqsr_util as bq

ROOT, CSRC = bq.ROOT, bq.CSRC
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_multiplemetrics")
MAX_LSEQ = 1 << 20
CATS = ("FIRST_OF_PAIR", "SECOND_OF_PAIR", "UNPAIRED")
ORIENTS = ("FR", "RF", "TANDEM")
# Picard's default adapters (IlluminaUtil.IlluminaAdapterPair SINGLE_END, PAIRED_END, INDEXED; 5' then 3')
ADAPTERS = ("AATGATACGGCGACCACCGACAGGTTCAGAGTTCTACAGTCCGACGATC", "AGATCGGAAGAGCTCGTATGCCGTCTTCTGCTTG",
            "AATGATACGGCGACCACCGAGATCTACACTCTTTCCCTACACGACGCTCTTCCGATCT", "AGATCGGAAGAGCGGTTCAGCAGGAATGCCGAGACCGATCTCGTATGCCGTCTTCTGCTTG",
            "AATGATACGGCGACCACCGAGATCTACACTCTTTCCCTACACGACGCTCTTCCGATCT",
            "AGATCGGAAGAGCACACGTCTGAACTCCAGTCACNNNNNNNNATCTCGTATGCCGTCTTCTGCTTG")
ERRORS = {1: "has l_seq 0 or above 1048576", 2: "does not lie inside a contig of the reference", 3: "has a CIGAR that does not match its record"}


def revcomp(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


class Ref:
    """Contigs, .amb holes (offset, length, letter) and a base code (0..3) per locus, as bm2_index writes them."""

    def __init__(self, contigs, holes=(), codes=None, seed=7):
        self.names = [n for n, _ in contigs]
        self.lens = [ln for _, ln in contigs]
        self.off = [int(x) for x in np.cumsum([0] + self.lens[:-1])]
        self.l_pac = int(sum(self.lens))
        self.holes = list(holes)
        self.codes = codes if codes is not None else np.random.default_rng(seed).integers(0, 4, self.l_pac).astype(np.uint8)
        t = np.frombuffer(b"ACGT", np.uint8)[self.codes].copy()
        for b, n, c in self.holes:
            t[b:b + n] = ord(c.upper())
        self.text = t.tobytes().decode()                      # the reference letter at each locus

    def letter(self, g):
        return self.text[g]

    def write(self, prefix):
        ann = "%d %d 11\n" % (self.l_pac, len(self.names))
        for n, o, ln in zip(self.names, self.off, self.lens):
            ann += "0 %s (null)\n%d %d %d\n" % (n, o, ln, sum(1 for b, k, _ in self.holes if o <= b < o + ln))
        open(prefix + ".ann", "w").write(ann)
        open(prefix + ".amb", "w").write("%d %d %d\n" % (self.l_pac, len(self.names), len(self.holes)) + "".join("%d %d %s\n" % h for h in self.holes))
        pac = bytearray((self.l_pac + 3) // 4)
        for i, c in enumerate(self.codes):
            pac[i // 4] |= int(c) << (2 * (3 - i % 4))
        if self.l_pac % 4 == 0:
            pac.append(0)
        pac.append(self.l_pac % 4)
        open(prefix + ".pac", "wb").write(bytes(pac))

    @staticmethod
    def read(prefix):
        lines = open(prefix + ".ann").read().split("\n")
        n = int(lines[0].split()[1])
        contigs = [(lines[1 + 2 * k].split()[1], int(lines[2 + 2 * k].split()[1])) for k in range(n)]
        amb = open(prefix + ".amb").read().split("\n")
        holes = [(int(a.split()[0]), int(a.split()[1]), a.split()[2]) for a in amb[1:1 + int(amb[0].split()[2])]]
        l_pac = int(lines[0].split()[0])
        pac = np.frombuffer(open(prefix + ".pac", "rb").read(), np.uint8)
        i = np.arange(l_pac)
        return Ref(contigs, holes, ((pac[i >> 2] >> ((3 - (i & 3)) * 2)) & 3).astype(np.uint8))


# ---- the rule ----

def _orientation(f, ref_len):
    """htsjdk SamPairUtil.getPairOrientation."""
    rev, mrev = bool(f["flag"] & 0x10), bool(f["flag"] & 0x20)
    if rev == mrev:
        return "TANDEM"
    start = f["pos"] + 1
    pos5 = f["next_pos"] + 1 if rev else start
    neg5 = start + ref_len - 1 if rev else start + f["tlen"]
    return "FR" if pos5 < neg5 else "RF"


def _is_adapter(seq):
    if len(seq) < 16:
        return False
    for a in ADAPTERS:
        for k in (a[:16], revcomp(a[:16])):
            if sum(1 for x, y in zip(seq[:16], k) if x != "N" and x != y) <= 1:
                return True
    return False


def _new_cat():
    return dict(total=0, pf=0, noise=0, adapter=0, aligned=0, in_pairs=0, improper=0, forward=0, soft=0, hard=0, sc3_sum=0, sc3_reads=0,
                indels=0, bases=0, mism=0, hq_reads=0, hq_bases=0, q20=0, hq_mism=0, chim_den=0, chim=0,
                lengths=Counter(), read_mism=Counter(), nocall=Counter())


def metrics(recs, ref):
    """Records in any order -> (cats {name: counters}, inserts {orientation: Counter}, err) where err is None or (index, kind, name) of the
    first read error by index."""
    cats = {c: _new_cat() for c in CATS}
    inserts = {o: Counter() for o in ORIENTS}
    for i, r in enumerate(recs):
        f = bu.fields(r)
        flag = f["flag"]
        if flag & 0x900:
            continue
        L = f["l_seq"]
        if L == 0 or L > MAX_LSEQ:
            return None, None, (i, 1, f["qname"])
        pf = not flag & 0x200
        aligned = pf and not flag & 4
        ops = [(c >> 4, c & 15) for c in f["cigar"]]
        ref_len = sum(n for n, t in ops if t in (0, 2, 3, 7, 8))
        if aligned:
            if f["rid"] < 0 or f["rid"] >= len(ref.names) or f["pos"] < 0 or f["pos"] + ref_len > ref.lens[f["rid"]]:
                return None, None, (i, 2, f["qname"])
            if sum(n for n, t in ops if t in (0, 1, 4, 7, 8)) != L:
                return None, None, (i, 3, f["qname"])
        m = cats["UNPAIRED" if not flag & 1 else "FIRST_OF_PAIR" if flag & 0x40 else "SECOND_OF_PAIR"]
        seq, qual = f["seq"], f["qual"]
        m["total"] += 1
        m["lengths"][L] += 1
        for k, b in enumerate(seq):
            if b == "N":
                m["nocall"][L - 1 - k if flag & 0x10 else k] += 1
        tags = {t: v for t, _, v in f["tags"]}
        if pf:
            m["pf"] += 1
            if tags.get("XN") == 1 and any(t == "XN" and ty in "cCsSiI" for t, ty, _ in f["tags"]):
                m["noise"] += 1
            if flag & 4 and _is_adapter(seq):
                m["adapter"] += 1
        if aligned:
            m["aligned"] += 1
            mated = flag & 1 and not flag & 8
            m["in_pairs"] += bool(mated)
            m["improper"] += bool(flag & 1 and not flag & 2)
            m["forward"] += not flag & 0x10
            m["soft"] += sum(n for n, t in ops if t == 4)
            m["hard"] += sum(n for n, t in ops if t == 5)
            m["indels"] += sum(1 for n, t in ops if t in (1, 2))
            core = [(n, t) for n, t in ops if t != 5]
            end = core[0] if flag & 0x10 else core[-1]
            if end[1] == 4:
                m["sc3_sum"] += end[0]; m["sc3_reads"] += 1
            hq = f["mapq"] >= 20
            g, q, mism, q20 = ref.off[f["rid"]] + f["pos"], 0, 0, 0
            for n, t in ops:
                if t in (0, 7, 8):
                    for k in range(n):
                        mism += seq[q + k] != ref.letter(g + k)
                        q20 += qual[0] != 0xFF and qual[q + k] >= 20
                if t in (0, 2, 3, 7, 8):
                    g += n
                if t in (0, 1, 4, 7, 8):
                    q += n
            aligned_bases = sum(n for n, t in ops if t in (0, 7, 8))
            m["bases"] += aligned_bases
            m["mism"] += mism
            if hq:
                m["hq_reads"] += 1; m["hq_bases"] += aligned_bases; m["q20"] += q20; m["hq_mism"] += mism
                m["read_mism"][mism] += 1
                m["chim_den"] += 1
                if mated:
                    chim = f["next_rid"] != f["rid"] or abs(f["tlen"]) > 100000 or _orientation(f, ref_len) != "FR"
                else:
                    chim = "SA" in tags
                m["chim"] += bool(chim)
        if flag & 1 and not flag & (4 | 8 | 0x40 | 0x400) and f["tlen"] != 0:
            inserts[_orientation(f, ref_len)][abs(f["tlen"])] += 1
    return cats, inserts, None


# ---- the files ----

def _d(v):
    s = "%.6f" % v
    s = s.rstrip("0")
    return s[:-1] if s.endswith(".") else s


def _kth(items, k):
    s = 0
    for v, c in items:
        s += c
        if s >= k:
            return v
    return items[-1][0]


def _median(items, n):
    if n <= 0:
        return 0.0
    return float(_kth(items, (n + 1) // 2)) if n % 2 else (_kth(items, n // 2) + _kth(items, n // 2 + 1)) / 2.0


def hist_stats(h):
    """htsjdk Histogram: n, mean, sd (n - 1), median, mad, mode (smallest tied), min, max of a Counter."""
    items = sorted((k, c) for k, c in h.items() if c)
    n = sum(c for _, c in items)
    if not n:
        return dict(n=0, mean=0.0, sd=0.0, median=0.0, mad=0.0, mode=0.0, min=0, max=0)
    mean = sum(float(k) * c for k, c in items) / n
    ss = 0.0
    for k, c in items:
        ss += float(c) * ((float(k) - mean) * (float(k) - mean))
    med = _median([(float(k), c) for k, c in items], n)
    mad = _median(sorted((abs(float(k) - med), c) for k, c in items), n)
    best = max(c for _, c in items)
    return dict(n=n, mean=mean, sd=math.sqrt(ss / (n - 1)) if n > 1 else 0.0, median=med, mad=mad,
                mode=float(min(k for k, c in items if c == best)), min=items[0][0], max=items[-1][0])


SUMMARY_COLS = ("CATEGORY TOTAL_READS PF_READS PCT_PF_READS PF_NOISE_READS PF_READS_ALIGNED PCT_PF_READS_ALIGNED PF_ALIGNED_BASES "
                "PF_HQ_ALIGNED_READS PF_HQ_ALIGNED_BASES PF_HQ_ALIGNED_Q20_BASES PF_HQ_MEDIAN_MISMATCHES PF_MISMATCH_RATE PF_HQ_ERROR_RATE "
                "PF_INDEL_RATE MEAN_READ_LENGTH SD_READ_LENGTH MEDIAN_READ_LENGTH MAD_READ_LENGTH MIN_READ_LENGTH MAX_READ_LENGTH "
                "READS_ALIGNED_IN_PAIRS PCT_READS_ALIGNED_IN_PAIRS PF_READS_IMPROPER_PAIRS PCT_PF_READS_IMPROPER_PAIRS BAD_CYCLES STRAND_BALANCE "
                "PCT_CHIMERAS PCT_ADAPTER PCT_SOFTCLIP PCT_HARDCLIP AVG_POS_3PRIME_SOFTCLIP_LENGTH SAMPLE LIBRARY READ_GROUP").split()
INSERT_COLS = ("MEDIAN_INSERT_SIZE MODE_INSERT_SIZE MEDIAN_ABSOLUTE_DEVIATION MIN_INSERT_SIZE MAX_INSERT_SIZE MEAN_INSERT_SIZE "
               "STANDARD_DEVIATION READ_PAIRS PAIR_ORIENTATION WIDTH_OF_10_PERCENT WIDTH_OF_20_PERCENT WIDTH_OF_30_PERCENT WIDTH_OF_40_PERCENT "
               "WIDTH_OF_50_PERCENT WIDTH_OF_60_PERCENT WIDTH_OF_70_PERCENT WIDTH_OF_80_PERCENT WIDTH_OF_90_PERCENT WIDTH_OF_95_PERCENT "
               "WIDTH_OF_99_PERCENT SAMPLE LIBRARY READ_GROUP").split()


def _bad_cycles(m):
    return sum(1 for v in m["nocall"].values() if m["total"] and v / m["total"] >= 0.8)


def _row(name, m, bad):
    r = lambda a, b: _d(a / b if b else 0.0)
    L, M = hist_stats(m["lengths"]), hist_stats(m["read_mism"])
    v = [name, m["total"], m["pf"], r(m["pf"], m["total"]), m["noise"], m["aligned"], r(m["aligned"], m["pf"]), m["bases"], m["hq_reads"],
         m["hq_bases"], m["q20"], _d(M["median"]), r(m["mism"], m["bases"]), r(m["hq_mism"], m["hq_bases"]), r(m["indels"], m["bases"]),
         _d(L["mean"]), _d(L["sd"]), _d(L["median"]), _d(L["mad"]), L["min"], L["max"], m["in_pairs"], r(m["in_pairs"], m["aligned"]),
         m["improper"], r(m["improper"], m["aligned"]), bad, r(m["forward"], m["aligned"]), r(m["chim"], m["chim_den"]),
         r(m["adapter"], m["pf"]), r(m["soft"], m["bases"]), r(m["hard"], m["bases"]), r(m["sc3_sum"], m["sc3_reads"]), "", "", ""]
    return "\t".join(str(x) for x in v) + "\n"


def _header(args, cls):
    return "## htsjdk.samtools.metrics.StringHeader\n# bm2_multiplemetrics" + (" " + args if args else "") + "\n\n## METRICS CLASS\t" + cls + "\n"


def summary_text(cats, args):
    o = _header(args, "picard.analysis.AlignmentSummaryMetrics") + "\t".join(SUMMARY_COLS) + "\n"
    first, second, un = cats["FIRST_OF_PAIR"], cats["SECOND_OF_PAIR"], cats["UNPAIRED"]
    if first["total"]:
        o += _row("FIRST_OF_PAIR", first, _bad_cycles(first)) + _row("SECOND_OF_PAIR", second, _bad_cycles(second))
        pair = {k: first[k] + second[k] for k in first}
        o += _row("PAIR", pair, _bad_cycles(first) + _bad_cycles(second))
    if un["total"] or not first["total"]:
        o += _row("UNPAIRED", un, _bad_cycles(un))
    return o


def insert_text(inserts, args):
    o = _header(args, "picard.analysis.InsertSizeMetrics") + "\t".join(INSERT_COLS) + "\n"
    total = sum(sum(h.values()) for h in inserts.values())
    if not total:
        return o
    shown, trimmed = [], {}
    for name in ORIENTS:
        h = inserts[name]
        n = sum(h.values())
        if not n / total >= 0.05:
            continue
        s = hist_stats(h)
        widths = {p: 0 for p in (10, 20, 30, 40, 50, 60, 70, 80, 90, 95, 99)}
        low = high = s["median"]
        covered = 0.0
        while low >= s["min"] or high <= s["max"]:                  # Picard's loop
            covered += h.get(int(low), 0)
            if low != high:
                covered += h.get(int(high), 0)
            frac = covered / n
            dist = int(high - low) + 1
            for p in widths:
                if frac >= p / 100 and widths[p] == 0:
                    widths[p] = dist
            low -= 1; high += 1
        top = int(s["median"] + 10 * s["mad"])
        t = Counter({k: c for k, c in h.items() if k <= top})
        ts = hist_stats(t)
        shown.append(name); trimmed[name] = t
        v = [_d(s["median"]), _d(s["mode"]), _d(s["mad"]), s["min"], s["max"], _d(ts["mean"]), _d(ts["sd"]), n, name] + list(widths.values()) + ["", "", ""]
        o += "\t".join(str(x) for x in v) + "\n"
    o += "\n## HISTOGRAM\tjava.lang.Integer\ninsert_size" + "".join("\tAll_Reads.%s_count" % s.lower() for s in shown) + "\n"
    for k in sorted(set().union(*(trimmed[s].keys() for s in shown))):
        o += str(k) + "".join("\t%d" % trimmed[s].get(k, 0) for s in shown) + "\n"
    return o


def files(recs, ref, args=""):
    cats, ins, err = metrics(recs, ref)
    assert err is None, err
    return summary_text(cats, args), insert_text(ins, args)


# ---- records ----

def tag_i(name, v, t="i"):
    return name.encode() + t.encode() + struct.pack("<" + {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I"}[t], v)


def tag_z(name, v):
    return name.encode() + b"Z" + v.encode() + b"\0"


def rec(name, flag, rid, pos, cigar, quals=30, seq=None, mapq=60, mrid=None, mpos=-1, tlen=0, tags=b""):
    """A record: cigar (length, op) pairs; quals an int (every base), a list, or None (QUAL '*'); seq defaults to A C G T repeated; tags as
    bytes (tag_i, tag_z)."""
    L = sum(n for n, op in cigar if op in (0, 1, 4, 7, 8)) if seq is None else len(seq)
    s = seq if seq is not None else ("ACGT" * (L // 4 + 1))[:L]
    q = [quals] * L if isinstance(quals, int) else quals
    mrid = (rid if flag & 1 else -1) if mrid is None else mrid
    r = bq.make_rec(name, flag, rid, pos, cigar, s, q, mapq=mapq, mrid=mrid, mpos=mpos, tlen=tlen)
    return struct.pack("<i", len(r) - 4 + len(tags)) + r[4:] + tags


def ref_seq(ref, rid, pos, n):
    return "".join(ref.letter(ref.off[rid] + pos + k) for k in range(n))


def random_records(ref, rng, n_pairs, max_len=150):
    """n_pairs random templates: pairs with both, one or no end mapped, in any order and with every flag the rule reads (secondary,
    supplementary, QC fail, duplicate, proper, strands), MAPQs on both sides of 20, clips, indels, N bases, reads copied from the reference
    with some errors, XN and SA tags, adapter reads, and TLENs of every orientation, some above 100 000 and 2^20; single-end reads too.
    Shuffled."""
    out = []

    def cigar(L):
        c, left = [], L
        if rng.random() < 0.1:
            c.append((int(rng.integers(1, 10)), 5))
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
        if rng.random() < 0.1:
            c.append((int(rng.integers(1, 10)), 5))
        return c

    def one(name, flag, rid, pos, L, mapq, mrid, mpos, tlen):
        tags = b""
        if rng.random() < 0.1:
            tags += tag_i("XN", int(rng.choice([0, 1, 1, 2])), str(rng.choice(["c", "C", "s", "i"])))
        if rng.random() < 0.1:
            tags += tag_z("SA", "c1,100,+,30M,60,0;")
        if rng.random() < 0.05:
            tags += tag_z("RG", "g1")
        q = [int(x) for x in (rng.integers(0, 41, L) if rng.random() < 0.7 else rng.choice([2, 19, 20, 21, 37], L))]
        if flag & 4:
            if rng.random() < 0.5:
                a = ADAPTERS[int(rng.integers(0, 6))][:16]
                a = revcomp(a) if rng.random() < 0.5 else a
                s = list(a + "".join("ACGT"[int(x)] for x in rng.integers(0, 4, max(L - 16, 0))))[:L]
                for _ in range(int(rng.choice([0, 1, 2]))):
                    s[int(rng.integers(0, min(16, L)))] = str(rng.choice(list("ACGTN")))
                s = "".join(s)
            else:
                s = "".join("ACGTN"[int(x)] for x in rng.choice(5, L, p=[0.24, 0.24, 0.24, 0.24, 0.04]))
            return rec(name, flag, rid, pos, [], q, seq=s, mapq=0, mrid=mrid, mpos=mpos, tlen=tlen, tags=tags)
        c = cigar(L)
        rl = sum(n for n, op in c if op in (0, 2, 3, 7, 8))
        pos = max(0, min(pos, ref.lens[rid] - rl))
        L = sum(n for n, op in c if op in (0, 1, 4, 7, 8))
        s = list(ref_seq(ref, rid, pos, rl).replace(".", "N"))[:L] + ["A"] * max(0, L - rl)
        s = "".join(("ACGTN"[int(rng.integers(0, 5))] if rng.random() < 0.05 else b) for b in s[:L])
        q = q[:L] + [30] * max(0, L - len(q))
        return rec(name, flag, rid, pos, c, q if rng.random() < 0.95 else None, seq=s, mapq=mapq, mrid=mrid, mpos=mpos, tlen=tlen, tags=tags)

    for k in range(n_pairs):
        rid = int(rng.integers(0, len(ref.names)))
        if ref.lens[rid] < 400:
            continue
        L1, L2 = int(rng.integers(5, max_len)), int(rng.integers(5, max_len))
        p1 = int(rng.integers(0, ref.lens[rid] - 200))
        p2 = max(0, min(ref.lens[rid] - 200, p1 + int(rng.integers(-60, 300))))
        mq = lambda: int(rng.choice([0, 5, 19, 20, 60, 60, 60]))
        name = "t%d" % k
        if rng.random() < 0.15:                                          # single-end
            f = int(rng.choice([0, 0x10, 0x4, 0x400, 0x200, 0x100, 0x800]))
            out.append(one(name, f, -1 if f & 4 else rid, -1 if f & 4 else p1, L1, mq(), -1, -1, 0))
            continue
        s1, s2 = int(rng.integers(0, 2)), int(rng.integers(0, 2))
        u1, u2 = rng.random() < 0.07, rng.random() < 0.07
        mrid2 = rid if rng.random() < 0.9 else (rid + 1) % len(ref.names)
        tl = int(rng.choice([abs(p2 - p1) + L2, abs(p2 - p1) + 1, 100000, 100001, 1 << 20, (1 << 20) + 5, 3000000, 0, int(rng.integers(1, 500))]))
        tl = tl if p1 <= p2 else -tl
        extra = int(rng.choice([0, 0, 0, 0, 0x400, 0x200, 0x2, 0x2, 0x2]))
        f1 = 0x1 | 0x40 | extra | (0x10 if s1 else 0) | (0x20 if s2 else 0) | (0x4 if u1 else 0) | (0x8 if u2 else 0)
        f2 = 0x1 | 0x80 | extra | (0x10 if s2 else 0) | (0x20 if s1 else 0) | (0x4 if u2 else 0) | (0x8 if u1 else 0)
        out.append(one(name, f1, -1 if u1 else rid, -1 if u1 else p1, L1, mq(), mrid2, p2, 0 if u1 or u2 else tl))
        out.append(one(name, f2, -1 if u2 else mrid2, -1 if u2 else p2, L2, mq(), rid, p1, 0 if u1 or u2 else -tl))
        if rng.random() < 0.05:
            out.append(one(name, 0x1 | 0x800 | 0x40, rid, p1, int(rng.integers(20, 60)), 60, rid, p2, 0))
        if rng.random() < 0.05:
            out.append(one(name, 0x1 | 0x100 | 0x80, rid, p2, int(rng.integers(20, 60)), 0, rid, p1, 0))
    order = rng.permutation(len(out))
    return [out[i] for i in order]


# ---- the host emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mm_emul") / "libmmemul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "host_emul", "multiplemetrics_emul.cpp"), "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.mme_new.restype = C.c_void_p
    lib.mme_new.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int64]
    lib.mme_add.restype = C.c_int32
    lib.mme_add.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_char_p, C.c_int64]
    lib.mme_counts.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.mme_text.restype = C.c_int64
    lib.mme_text.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.c_char_p, C.c_int64]
    lib.mme_free.argtypes = [C.c_void_p]
    lib.mme_run.restype = C.c_int32
    lib.mme_run.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.c_int32, C.c_char_p, C.c_char_p, C.c_int64, C.c_void_p]
    return lib


def pac_bytes(ref):
    pac = np.zeros((ref.l_pac + 3) // 4, np.uint8)
    i = np.arange(ref.l_pac)
    np.bitwise_or.at(pac, i >> 2, (ref.codes.astype(np.uint8) << ((3 - (i & 3)) * 2)).astype(np.uint8))
    return pac


def hole_arrays(ref):
    h = np.array([(b, b + n) for b, n, _ in ref.holes], np.int64).reshape(-1)
    return (h if len(h) else np.zeros(2, np.int64)), "".join(c for _, _, c in ref.holes).encode()


def windows(recs, sizes):
    """Split recs into windows of the given record counts (cycled)."""
    out, i, k = [], 0, 0
    while i < len(recs):
        n = sizes[k % len(sizes)]
        out.append(recs[i:i + n]); i += n; k += 1
    return out


def emul_run(lib, ref, wins, args=""):
    """The emulation's add per window -> (summary text, insert text, counts [3][21], pairs [3], None) or (None, None, None, None, error)."""
    off = np.array(ref.off, np.int64); ln = np.array(ref.lens, np.int32)
    pac = pac_bytes(ref)
    hb, hc = hole_arrays(ref)
    h = lib.mme_new(off.ctypes.data, ln.ctypes.data, len(off), ref.l_pac, pac.ctypes.data, hb.ctypes.data, hc, len(ref.holes))
    try:
        err = C.create_string_buffer(4096)
        for w in wins:
            data, starts = bq.flatten(w)
            buf = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
            sb = starts if len(starts) else np.zeros(1, np.int64)
            if lib.mme_add(h, buf.ctypes.data, sb.ctypes.data, len(w), err, 4096):
                return None, None, None, None, err.value.decode()
        counts, pairs = np.zeros((3, 21), np.int64), np.zeros(3, np.int64)
        lib.mme_counts(h, counts.ctypes.data, pairs.ctypes.data)
        texts = []
        for which in (0, 1):
            n = lib.mme_text(h, which, args.encode(), None, 0)
            out = C.create_string_buffer(n + 1)
            lib.mme_text(h, which, args.encode(), out, n + 1)
            texts.append(out.value.decode())
        return texts[0], texts[1], counts, pairs, None
    finally:
        lib.mme_free(h)


def emul_tool(lib, prefix, bam, window=1 << 28, threads=2, args=""):
    """The emulated tool over files -> (summary, insert, stats) or raises ValueError with the error."""
    out = C.create_string_buffer(1 << 22)
    st = np.zeros(2, np.int64)
    if lib.mme_run(prefix.encode(), bam.encode(), window, threads, args.encode(), out, 1 << 22, st.ctypes.data):
        raise ValueError(out.value.decode())
    a = out.value.decode()
    b = C.string_at(C.addressof(out) + len(a.encode()) + 1).decode()
    return a, b, dict(records=int(st[0]), windows=int(st[1]))


def bam_bytes(ref, recs, text="@HD\tVN:1.6\tSO:unsorted\n", refs=None):
    refs = refs if refs is not None else list(zip(ref.names, ref.lens))
    h = b"BAM\x01" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for n, ln in refs:
        h += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", ln)
    return bq.bgzf(h + b"".join(recs))


KEYS = ("total", "pf", "noise", "adapter", "aligned", "in_pairs", "improper", "forward", "soft", "hard", "sc3_sum", "sc3_reads", "indels", "bases",
        "mism", "hq_reads", "hq_bases", "q20", "hq_mism", "chim_den", "chim")


def from_device(d):
    """Context.mm_finish's dict -> metrics()'s (cats, inserts), so that the files come from Python's text functions."""
    cats = {}
    for c, name in enumerate(CATS):
        m = _new_cat()
        for k, key in enumerate(KEYS):
            m[key] = int(d["counts"][c][k])
        for src, dst in (("len_hist", "lengths"), ("mism_hist", "read_mism"), ("nocall", "nocall")):
            m[dst] = Counter({k: int(v) for k, v in enumerate(d[src][c]) if v})
        cats[name] = m
    inserts = {o: Counter({k: int(v) for k, v in enumerate(d["insert_hist"][i]) if v}) for i, o in enumerate(ORIENTS)}
    for x in d["insert_big"]:
        inserts[ORIENTS[int(x) >> 32]][int(x) & 0xFFFFFFFF] += 1
    return cats, inserts

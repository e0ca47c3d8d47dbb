"""Helpers of the duplicate-marking tests: the rule of bwa-mem2_b200/csrc/markdup_device.cuh restated in Python from bam_util.fields, the
host emulation tests/host_emul/markdup_emul.cpp, records and templates built field by field, and reads with planted duplicates drawn from an
index's reference."""
import ctypes as C
import os, struct, subprocess
import numpy as np
import bam_util as bu
import bam_sort_util as bs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bwa-mem2_b200", "csrc")
DUP_ENTRY_DT = np.dtype([("k1", "<u8"), ("k2", "<u8"), ("tid", "<i8"), ("score", "<i4"), ("kind", "<i4")])
PAIR, FRAG, PAIR_END = 0, 1, 2


# ---- the rule ----

def end_of(f):
    """(refID, unclipped 5' coordinate, reverse) of a mapped record."""
    rev = bool(f["flag"] & 16)
    cig = f["cigar"]
    ops = cig if not rev else cig[::-1]
    clip = 0
    for c in ops:
        if c & 15 not in (4, 5):
            break
        clip += c >> 4
    if not rev:
        return f["rid"], f["pos"] - clip, 0
    rl = bu.ref_len(cig)
    return f["rid"], f["pos"] + (rl or 1) - 1 + clip, 1


def end_key(e):
    rid, coord, rev = e
    return (rid << 34) | ((coord + (1 << 32)) << 1) | rev


def read_score(f):
    q = f["qual"]
    if f["l_seq"] == 0 or q[0] == 0xFF:
        return 0
    return min(sum(x for x in q if x >= 15), 16383)


def template_entries(fs, tid):
    """A template's records (field dicts, in record order) -> (pair entries, fragment-space entries) as (k1, k2, tid, score, kind)."""
    prim = [f for f in fs if not f["flag"] & 0x900]
    if len(prim) == 2 and not prim[0]["flag"] & 4 and not prim[1]["flag"] & 4:
        ks = [end_key(end_of(f)) for f in prim]
        sc = [read_score(f) for f in prim]
        return [(min(ks), max(ks), tid, sc[0] + sc[1], PAIR)], [(ks[k], 0, tid, sc[k], PAIR_END) for k in range(2)]
    if len(prim) in (1, 2):
        for f in prim:
            if not f["flag"] & 4:
                return [], [(end_key(end_of(f)), 0, tid, read_score(f), FRAG)]
    return [], []


def resolve(entries):
    """Entries of one space -> the duplicates' template ids, in the sort order (k1, k2, score descending, tid)."""
    srt = sorted(entries, key=lambda e: (e[0], e[1], -e[3], e[2]))
    out, g0 = [], 0
    while g0 < len(srt):
        g1 = g0
        while g1 < len(srt) and srt[g1][:2] == srt[g0][:2]:
            g1 += 1
        grp = srt[g0:g1]
        has_pe = any(e[4] == PAIR_END for e in grp)
        first = next((k for k, e in enumerate(grp) if e[4] != PAIR_END), None)
        out += [e[2] for k, e in enumerate(grp) if e[4] != PAIR_END and (has_pe or k != first)]
        g0 = g1
    return out


def duplicates(templates):
    """templates: [(tid, [field dicts])] -> (pair-space duplicates, fragment-space duplicates, templates with an entry)."""
    pe, fe = [], []
    for tid, fs in templates:
        p, f = template_entries(fs, tid)
        pe += p; fe += f
    return resolve(pe), resolve(fe), len(pe) + sum(e[4] == FRAG for e in fe)


def set_flag(rec, flag):
    return rec[:18] + struct.pack("<H", flag) + rec[20:]


def apply_flags(recs, tid_of, dups):
    """recs: record bytes; tid_of(record) -> its template id; the records of the templates in dups, unless unmapped, with 0x400."""
    out = []
    for r in recs:
        f = bu.fields(r)
        out.append(set_flag(r, f["flag"] | 0x400) if tid_of(r) in dups and not f["flag"] & 4 else r)
    return out


# ---- records ----

def with_qual(rec, qual):
    """A record (bam_sort_util.make_rec) with its QUAL replaced: bytes of l_seq, one value (int) for every base, or None for '*'."""
    lrn, ncig = rec[12], struct.unpack_from("<H", rec, 16)[0]
    lseq = struct.unpack_from("<i", rec, 20)[0]
    at = 36 + lrn + 4 * ncig + (lseq + 1) // 2
    q = bytes([0xFF]) * lseq if qual is None else bytes([qual]) * lseq if isinstance(qual, int) else bytes(qual)
    assert len(q) == lseq
    return rec[:at] + q + rec[at + lseq:]


def random_templates(rng, n, paired=True, piles=40, start_tid=0):
    """n templates of crafted records: a few contigs and few positions (piles of duplicates), clips on both strands, unmapped mates placed at
    their mate, both unmapped, secondary and supplementary records, mates on other contigs, QUAL '*' and CG:B,I now and then.
    -> [(tid, [record bytes])], tids increasing with gaps as reads of pairs give."""
    out, tid = [], start_tid
    spots = [(int(rng.integers(0, 3)), int(rng.integers(0, 5000)), int(rng.integers(0, 2))) for _ in range(piles)]

    def one(name, flag, rid, pos, rev, l=60):
        lc, tc = int(rng.choice([0, 0, 3, 7])), int(rng.choice([0, 0, 4]))
        hard = bool(rng.integers(0, 5) == 0)
        cig = ([(lc, 5 if hard else 4)] if lc else []) + [(l - lc - tc, 0)] + ([(tc, 4)] if tc else [])
        if rng.integers(0, 15) == 0:
            cig = [(lc or 2, 4)] + [(1, 0), (1, 2)] * 300 + [(1, 0)]
            r = bs.make_rec(rid, pos, flag | (16 if rev else 0), name=name, cg=cig)
        else:
            r = bs.make_rec(rid, pos, flag | (16 if rev else 0), cigar=tuple(cig), name=name)
        lseq = struct.unpack_from("<i", r, 20)[0]
        q = None if rng.integers(0, 12) == 0 else rng.choice([2, 10, 14, 15, 20, 30, 38], lseq)
        return with_qual(r, None if q is None else q.astype(np.uint8))

    def unmapped(name, flag, rid, pos):
        r = bs.make_rec(rid, pos, flag | 4, name=name, l_seq=60)
        return with_qual(r, rng.integers(2, 41, 60).astype(np.uint8))

    for k in range(n):
        name = b"t%d" % tid
        rid, pos, rev = spots[int(rng.integers(0, piles))]
        pos = max(0, pos + int(rng.choice([0, 0, 0, 1, 5])))
        kind = int(rng.integers(0, 10))
        recs = []
        if not paired:
            if kind == 0:
                recs.append(unmapped(name, 0, -1, -1))
            else:
                recs.append(one(name, 0, rid, pos, rev))
                if kind == 1:
                    recs.append(one(name, 0x800, rid, pos + 3000, 1 - rev))
                if kind == 2:
                    recs.append(one(name, 0x100, 1 - rid if rid < 2 else 0, pos, rev))
            out.append((tid, recs)); tid += 1
            continue
        mrid, mpos = (rid, pos + int(rng.choice([200, 300, 300]))) if kind != 3 else ((rid + 1) % 3, pos)
        if kind == 4:          # mate unmapped, placed at its mate
            recs += [one(name, 0x1 | 0x40 | 0x8, rid, pos, rev), unmapped(name, 0x1 | 0x80, rid, pos)]
        elif kind == 5:        # both unmapped
            recs += [unmapped(name, 0x1 | 0x40 | 0x8, -1, -1), unmapped(name, 0x1 | 0x80 | 0x8, -1, -1)]
        else:
            recs.append(one(name, 0x1 | 0x40, rid, pos, rev))
            if kind == 6:
                recs.append(one(name, 0x1 | 0x40 | 0x800, rid, pos + 2000, rev))
            recs.append(one(name, 0x1 | 0x80, mrid, mpos, 1 - rev))
            if kind == 7:
                recs.append(one(name, 0x1 | 0x80 | 0x100, mrid, mpos + 50, rev))
        out.append((tid, recs)); tid += 2
    return out


def flatten(templates):
    """-> (records bytes, tmpl_first, tmpl_id)."""
    data, first, ids, k = b"", [0], [], 0
    for tid, recs in templates:
        data += b"".join(recs); k += len(recs); first.append(k); ids.append(tid)
    return data, np.array(first, np.int64), np.array(ids, np.int64)


def entries_array(entries):
    a = np.zeros(len(entries), DUP_ENTRY_DT)
    for i, e in enumerate(entries):
        a[i] = e
    return a


def random_entries(rng, n, space):
    """Entries of one space with many equal keys and scores (piles and ties); the fragment space mixes in pair ends."""
    keys = [end_key((int(rng.integers(0, 4)), int(rng.integers(-50, 60)), int(rng.integers(0, 2)))) for _ in range(max(n // 12, 1))]
    out = []
    tids = rng.permutation(n * 3)[:n]
    for k in range(n):
        a = keys[int(rng.integers(0, len(keys)))]
        if space == PAIR:
            b = keys[int(rng.integers(0, len(keys)))]
            out.append((min(a, b), max(a, b), int(tids[k]), int(rng.choice([0, 100, 100, 2000, 32766])), PAIR))
        else:
            out.append((a, 0, int(tids[k]), int(rng.choice([0, 50, 50, 16383])), int(rng.choice([FRAG, FRAG, PAIR_END]))))
    return out


# ---- the emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("markdup_emul") / "libmarkdupemul.so")
    he = os.path.join(ROOT, "tests", "host_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(he, "markdup_emul.cpp"), os.path.join(he, "bam_sort_emul.cpp"), os.path.join(he, "bgzf_emul.cpp"),
                           "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.markdup_emul_signatures.argtypes = [C.c_void_p] * 4 + [C.c_int64] + [C.c_void_p] * 4
    lib.markdup_emul_resolve.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.markdup_emul_file.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                      C.c_char_p, C.c_int, C.c_char_p, C.c_void_p, C.c_char_p, C.c_int]
    return lib


def _buf(a, dt=np.uint8):
    a = np.frombuffer(a, np.uint8) if isinstance(a, bytes) else np.ascontiguousarray(a, dt)
    return a if len(a) else np.zeros(1, a.dtype)


def emul_signatures(lib, data, first, ids):
    st = np.array([a for a, _ in bu.records(data)], np.int64)
    n = len(ids)
    p, f = np.zeros(max(n, 1), DUP_ENTRY_DT), np.zeros(max(2 * n, 1), DUP_ENTRY_DT)
    np_, nf = C.c_int64(), C.c_int64()
    lib.markdup_emul_signatures(_buf(data).ctypes.data, _buf(st, np.int64).ctypes.data, _buf(first, np.int64).ctypes.data, _buf(ids, np.int64).ctypes.data,
                                n, p.ctypes.data, C.byref(np_), f.ctypes.data, C.byref(nf))
    return p[:np_.value], f[:nf.value]


def emul_resolve(lib, entries, resolve_=True):
    e = np.ascontiguousarray(entries, DUP_ENTRY_DT)
    srt, d, nd = np.zeros(max(len(e), 1), DUP_ENTRY_DT), np.zeros(max(len(e), 1), np.int64), C.c_int64()
    lib.markdup_emul_resolve(_buf(e, DUP_ENTRY_DT).ctypes.data, len(e), int(resolve_), srt.ctypes.data, d.ctypes.data, C.byref(nd))
    return d[:nd.value] if resolve_ else srt[:len(e)]


STAT_NAMES = ("runs", "windows", "sig_runs", "sig_bytes", "templates", "pair_dups", "frag_dups", "records", "spill_bytes")


def emul_file(lib, templates, run_bytes, sig_bytes, tmp_prefix, out_path, chunk_tmpl=50, threads=2):
    data, first, ids = flatten(templates)
    n_reads = int(ids.max()) + 2 if len(ids) else 0
    stats = np.zeros(9, np.int64); err = C.create_string_buffer(512)
    rc = lib.markdup_emul_file(_buf(data).ctypes.data, len(data), _buf(first, np.int64).ctypes.data, _buf(ids, np.int64).ctypes.data, len(ids), chunk_tmpl,
                               run_bytes, sig_bytes, n_reads, tmp_prefix.encode(), threads, out_path.encode(), stats.ctypes.data, err, 512)
    assert rc == 0, err.value
    return dict(zip(STAT_NAMES, (int(x) for x in stats)))


# ---- reads with planted duplicates ----

def load_reference(prefix):
    """The contigs of an index (<prefix>.ann, <prefix>.pac) as strings of ACGT."""
    lines = open(prefix + ".ann").read().split("\n")
    n = int(lines[0].split()[1])
    pac = np.frombuffer(open(prefix + ".pac", "rb").read(), np.uint8)
    out = []
    for k in range(n):
        name = lines[1 + 2 * k].split()[1]
        off, ln = (int(x) for x in lines[2 + 2 * k].split()[:2])
        i = np.arange(off, off + ln)
        codes = (pac[i >> 2] >> ((3 - (i & 3)) * 2)) & 3
        out.append((name, "".join("ACGT"[c] for c in codes)))
    return out


def revcomp(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


def planted_pairs(ref, rng, n_base=60, L=100):
    """Pairs of reads (name, r1, q1, r2, q2) drawn from ref with duplicates planted: copies under new names with new qualities (some with
    qualities equal to the original's, so the tie rule decides), copies whose first bases are changed (bwa clips them: the same unclipped
    5' end at another pos), copies with R1 and R2 swapped, copies with another insert (not duplicates), copies whose mate is random sequence
    (a fragment against pair ends) and chimeric reads (supplementary records)."""
    contigs = [s for _, s in ref if len(s) > 2000]
    pairs = []

    def q():
        return bytes(int(x) + 33 for x in rng.integers(2, 41, L))

    def mutate5(s, k=10):
        return "".join("ACGT"[("ACGT".index(c) + 1 + int(rng.integers(0, 3))) % 4] for c in s[:k]) + s[k:]

    for b in range(n_base):
        c = contigs[int(rng.integers(0, len(contigs)))]
        ins = int(rng.integers(250, 450))
        s = int(rng.integers(0, len(c) - ins - 1))
        r1, r2 = c[s:s + L], revcomp(c[s + ins - L:s + ins])
        q1, q2 = q(), q()
        pairs.append(("b%d" % b, r1, q1, r2, q2))
        for k in range(int(rng.integers(0, 4))):
            same = k == 0 and b % 3 == 0
            pairs.append(("b%dc%d" % (b, k), r1, q1 if same else q(), r2, q2 if same else q()))
        if b % 4 == 1:
            pairs.append(("b%dm" % b, mutate5(r1), q(), mutate5(r2), q()))
        if b % 5 == 2:
            pairs.append(("b%ds" % b, r2, q(), r1, q()))
        if b % 4 == 3:
            i2 = ins + 37
            if s + i2 < len(c):
                pairs.append(("b%di" % b, r1, q(), revcomp(c[s + i2 - L:s + i2]), q()))
        if b % 3 == 1:
            rnd = "".join("ACGT"[x] for x in rng.integers(0, 4, L))
            for k in range(2):
                pairs.append(("b%dr%d" % (b, k), r1, q(), rnd, q()))
        if b % 6 == 0:
            c2 = contigs[int(rng.integers(0, len(contigs)))]
            s2 = int(rng.integers(0, len(c2) - L))
            chim = r1[:L // 2] + c2[s2:s2 + L // 2]
            for k in range(2):
                pairs.append(("b%dx%d" % (b, k), chim, q(), r2, q()))
    order = rng.permutation(len(pairs))
    return [pairs[i] for i in order]


def fastq(recs):
    return "".join("@%s\n%s\n+\n%s\n" % (n, s, q.decode()) for n, s, q in recs).encode()


def fasta(recs):
    return "".join(">%s\n%s\n" % (n, s) for n, s, _ in recs).encode()

"""Helpers of the GC bias tests of bm2_multiplemetrics: Picard CollectGcBiasMetrics restated in Python as the README states the rule (no
code shared with bwa-mem2_b200/csrc/mm_device.cuh or mm_gcbias.h).  The reference windows two ways - GcBiasUtils.calculateGc with its rolling
state, written literally, for small references, and cumulative sums per contig in numpy for large ones - the per-record rule, the detail and
summary files' text, and the host emulation tests/host_emul/gcbias_emul.cpp.  References and records come from multiplemetrics_util."""
import ctypes as C
import math, os, subprocess
import numpy as np
import bam_util as bu
import bqsr_util as bq
import multiplemetrics_util as mu

W, BINS = 100, 101
DETAIL_COLS = ("ACCUMULATION_LEVEL READS_USED GC WINDOWS READ_STARTS MEAN_BASE_QUALITY NORMALIZED_COVERAGE ERROR_BAR_WIDTH SAMPLE LIBRARY "
               "READ_GROUP").split()
SUMMARY_COLS = ("ACCUMULATION_LEVEL READS_USED WINDOW_SIZE TOTAL_CLUSTERS ALIGNED_READS AT_DROPOUT GC_DROPOUT GC_NC_0_19 GC_NC_20_39 "
                "GC_NC_40_59 GC_NC_60_79 GC_NC_80_100 SAMPLE LIBRARY READ_GROUP").split()
PROGRAMS = ("CollectAlignmentSummaryMetrics", "CollectInsertSizeMetrics", "CollectGcBiasMetrics")


# ---- the reference windows ----

class _State:
    def __init__(self):
        self.init, self.gc, self.n, self.prior = True, 0, 0, None


def _is_gc(b):
    return b in ("G", "C")


def calculate_gc(bases, start, end, state):
    """GcBiasUtils.calculateGc: the window's bin, or -1 when it has more than 4 Ns; after the first window only the base entering and the
    base leaving change the counts."""
    if state.init:
        state.init = False
        state.gc = state.n = 0
        for i in range(start, end):
            if _is_gc(bases[i]):
                state.gc += 1
            elif bases[i] == "N":
                state.n += 1
    else:
        new = bases[end - 1]
        if _is_gc(new):
            state.gc += 1
        elif new == "N":
            state.n += 1
        if _is_gc(state.prior):
            state.gc -= 1
        elif state.prior == "N":
            state.n -= 1
    state.prior = bases[start]
    if state.n > 4:
        return -1
    return (state.gc * 100) // (end - start)


def ref_windows_literal(ref):
    """calculateRefWindowsByGc: per contig, the windows 1 <= i < L - W; mu.Ref.text holds the upper-cased letters."""
    out = [0] * BINS
    for o, L in zip(ref.off, ref.lens):
        bases = ref.text[o:o + L]
        state = _State()
        for i in range(1, L - W):
            b = calculate_gc(bases, i, i + W, state)
            if b != -1:
                out[b] += 1
    return out


def classes(ref):
    """(is GC, is N) per locus, as uint8 arrays."""
    t = np.frombuffer(ref.text.encode(), np.uint8)
    return ((t == ord("G")) | (t == ord("C"))).astype(np.int64), (t == ord("N")).astype(np.int64)


def ref_windows_numpy(ref, cls=None):
    """The same histogram from cumulative sums per contig."""
    g, n = classes(ref) if cls is None else cls
    out = np.zeros(BINS, np.int64)
    for o, L in zip(ref.off, ref.lens):
        if L - W <= 1:
            continue
        cg = np.concatenate(([0], np.cumsum(g[o:o + L])))
        cn = np.concatenate(([0], np.cumsum(n[o:o + L])))
        i = np.arange(1, L - W)
        gc, nn = cg[i + W] - cg[i], cn[i + W] - cn[i]
        keep = nn <= 4
        out += np.bincount(gc[keep] * 100 // W, minlength=BINS)
    return out


def window_bin(ref, g):
    s = ref.text[g:g + W]
    n = s.count("N")
    return -1 if n > 4 else (s.count("G") + s.count("C")) * 100 // W


# ---- the records ----

def reads(recs, ref):
    """Records in any order -> (dict(reads, bases, errors [101], clusters, aligned), err) where err is None or (index, kind, name) of the
    first read error by index (kinds as multiplemetrics_util.ERRORS)."""
    x = dict(reads=[0] * BINS, bases=[0] * BINS, errors=[0] * BINS, clusters=0, aligned=0)
    for i, r in enumerate(recs):
        f = bu.fields(r)
        flag = f["flag"]
        if flag & 0x900:
            continue
        L = f["l_seq"]
        if L == 0 or L > mu.MAX_LSEQ:
            return None, (i, 1, f["qname"])
        ops = [(c >> 4, c & 15) for c in f["cigar"]]
        ref_len = sum(n for n, t in ops if t in (0, 2, 3, 7, 8))
        placed = not flag & 4
        if placed:
            if f["rid"] < 0 or f["rid"] >= len(ref.names) or f["pos"] < 0 or f["pos"] + ref_len > ref.lens[f["rid"]]:
                return None, (i, 2, f["qname"])
            if sum(n for n, t in ops if t in (0, 1, 4, 7, 8)) != L:
                return None, (i, 3, f["qname"])
        x["clusters"] += (not flag & 1) or bool(flag & 0x40)
        if not placed:
            continue
        x["aligned"] += 1
        p = f["pos"] + ref_len - W if flag & 0x10 else f["pos"] + 1     # Picard's 1-based start used as a 0-based index
        if not 1 <= p < ref.lens[f["rid"]] - W:
            continue
        b = window_bin(ref, ref.off[f["rid"]] + p)
        if b < 0:
            continue
        seq, g, q, mism = f["seq"], ref.off[f["rid"]] + f["pos"], 0, 0
        for n, t in ops:
            if t in (0, 7, 8):
                mism += sum(seq[q + k] != ref.letter(g + k) for k in range(n))
            if t in (0, 2, 3, 7, 8):
                g += n
            if t in (0, 1, 4, 7, 8):
                q += n
        x["reads"][b] += 1
        x["bases"][b] += L
        x["errors"][b] += mism + sum(n for n, t in ops if t in (1, 2))
    return x, None


# ---- the files ----

def _ratio(a, b):
    return a / b if b else 0.0


def detail_text(windows, x, args):
    o = mu._header(args, "picard.analysis.GcBiasDetailMetrics") + "\t".join(DETAIL_COLS) + "\n"
    m = _ratio(sum(x["reads"]), sum(windows))
    for k in range(BINS):
        r, w, e, b = x["reads"][k], windows[k], x["errors"][k], x["bases"][k]
        q = math.floor(-10.0 * math.log10(e / b) + 0.5) if e > 0 else 0
        v = ["All Reads", "ALL", k, w, r, q, mu._d(_ratio(_ratio(r, w), m)), mu._d(_ratio(_ratio(math.sqrt(r), w), m)), "", "", ""]
        o += "\t".join(str(a) for a in v) + "\n"
    return o


def summary_text(windows, x, args):
    o = mu._header(args, "picard.analysis.GcBiasSummaryMetrics") + "\t".join(SUMMARY_COLS) + "\n"
    tw, tr = sum(windows), sum(x["reads"])
    at = gc = 0.0
    for k in range(BINS):
        if windows[k] < 1e-5 * tw:
            continue
        d = _ratio(100.0 * windows[k], tw) - _ratio(100.0 * x["reads"][k], tr)
        if d > 0 and k <= 50:
            at += d
        if d > 0 and k >= 50:
            gc += d
    m = _ratio(tr, sum(windows))
    v = ["All Reads", "ALL", W, x["clusters"], x["aligned"], mu._d(at), mu._d(gc)]
    for a, b in ((0, 19), (20, 39), (40, 59), (60, 79), (80, 100)):
        ks = [k for k in range(a, b + 1) if x["reads"][k] > 0]
        v.append(mu._d(_ratio(sum(x["reads"][k] for k in ks), sum(windows[k] for k in ks) * m)))
    return o + "\t".join(str(a) for a in v + ["", "", ""]) + "\n"


def files(recs, ref, args="", windows=None):
    windows = list(ref_windows_numpy(ref)) if windows is None else list(windows)
    x, err = reads(recs, ref)
    assert err is None, err
    return detail_text(windows, x, args), summary_text(windows, x, args)


def rows(text):
    lines = text.split("\n")
    cols = lines[4].split("\t")
    return [dict(zip(cols, l.split("\t"))) for l in lines[5:] if l]


# ---- the host emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gc_emul") / "libgcemul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + bq.CSRC, "-I" + os.path.join(bq.ROOT, "include"),
                           os.path.join(bq.ROOT, "tests", "host_emul", "gcbias_emul.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.gce_new.restype = C.c_void_p
    lib.gce_new.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int64]
    lib.gce_add.restype = C.c_int32
    lib.gce_add.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_char_p, C.c_int64]
    lib.gce_counts.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gce_text.restype = C.c_int64
    lib.gce_text.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_char_p, C.c_char_p, C.c_int64]
    lib.gce_word.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.gce_free.argtypes = [C.c_void_p]
    return lib


def emul_texts(lib, bins, totals, args=""):
    """mm_gcbias.h's two files of counts in gce_counts's layout ([4, 101] windows, reads, bases, errors; [clusters, aligned])."""
    b = np.ascontiguousarray(bins, np.int64).reshape(-1)
    t = np.ascontiguousarray(totals, np.int64)
    out = []
    for which in (0, 1):
        n = lib.gce_text(b.ctypes.data, t.ctypes.data, which, args.encode(), None, 0)
        s = C.create_string_buffer(n + 1)
        lib.gce_text(b.ctypes.data, t.ctypes.data, which, args.encode(), s, n + 1)
        out.append(s.value.decode())
    return tuple(out)


def emul_new(lib, ref):
    off = np.array(ref.off, np.int64); ln = np.array(ref.lens, np.int32)
    pac = mu.pac_bytes(ref)
    hb, hc = mu.hole_arrays(ref)
    return lib.gce_new(off.ctypes.data, ln.ctypes.data, len(off), ref.l_pac, pac.ctypes.data, hb.ctypes.data, hc, len(ref.holes))


def emul_run(lib, ref, wins, args=""):
    """The emulation over windows of records -> (detail, summary, bins [4, 101], totals [2], None) or (None, None, None, None, error)."""
    h = emul_new(lib, ref)
    try:
        err = C.create_string_buffer(4096)
        for w in wins:
            data, starts = bq.flatten(w)
            buf = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
            sb = starts if len(starts) else np.zeros(1, np.int64)
            if lib.gce_add(h, buf.ctypes.data, sb.ctypes.data, len(w), err, 4096):
                return None, None, None, None, err.value.decode()
        bins, totals = np.zeros((4, BINS), np.int64), np.zeros(2, np.int64)
        lib.gce_counts(h, bins.ctypes.data, totals.ctypes.data)
        return emul_texts(lib, bins, totals, args) + (bins, totals, None)
    finally:
        lib.gce_free(h)


def random_ref(rng, n_contigs, min_len, max_len, hole_every=300, extra_lens=()):
    """Random contigs (lengths in [min_len, max_len) plus extra_lens, shuffled) with holes of N, n, IUPAC letters and '.' of 1 to 40
    bases, about one per hole_every bases; sorted and disjoint."""
    lens = [int(x) for x in rng.integers(min_len, max_len, n_contigs)] + list(extra_lens)
    rng.shuffle(lens)
    contigs = [("r%d" % k, ln) for k, ln in enumerate(lens)]
    total = sum(lens)
    holes, at = [], 0
    while True:
        at += int(rng.integers(1, 2 * hole_every))
        n = int(rng.choice([1, 2, 3, 4, 5, 6, 10, 40]))
        if at + n > total:
            break
        holes.append((at, n, str(rng.choice(list("NNNnnRYSKM.")))))
        at += n
    return mu.Ref(contigs, holes, rng.integers(0, 4, total).astype(np.uint8))

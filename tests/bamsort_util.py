"""Helpers of the bm2_sort tests: samtools sort -n's name comparison restated literally in Python (strnum_cmp of samtools' bam_sort.c, the
1.9-era form, as bwa-mem2_b200/csrc/bam_sort_device.cuh states it), both orders of bm2_sort over whole records, its header rewrite and @PG rule,
and the host emulation of both orders (tests/host_emul/bamsort_emul.cpp)."""
import ctypes as C
import functools, os, struct, subprocess
import numpy as np
import bam_util as bu
import bam_sort_util as bs

ROOT = bs.ROOT
CSRC = bs.CSRC
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_sort")


def _digit(c):
    return 48 <= c <= 57


def strnum_cmp(a: bytes, b: bytes) -> int:
    """samtools' strnum_cmp over unsigned bytes: < 0, 0 or > 0.  A NUL ends each name, as in C."""
    a = a + b"\0"; b = b + b"\0"
    pa = pb = 0
    while a[pa] and b[pb]:
        if _digit(a[pa]) and _digit(b[pb]):
            while a[pa] == 48:
                pa += 1
            while b[pb] == 48:
                pb += 1
            while _digit(a[pa]) and _digit(b[pb]) and a[pa] == b[pb]:
                pa += 1; pb += 1
            if _digit(a[pa]) and _digit(b[pb]):
                i = 0
                while _digit(a[pa + i]) and _digit(b[pb + i]):
                    i += 1
                return 1 if _digit(a[pa + i]) else -1 if _digit(b[pb + i]) else a[pa] - b[pb]
            elif _digit(a[pa]):
                return 1
            elif _digit(b[pb]):
                return -1
            elif pa != pb:
                return 1 if pa < pb else -1
        else:
            if a[pa] != b[pb]:
                return a[pa] - b[pb]
            pa += 1; pb += 1
    return 1 if a[pa] else -1 if b[pb] else 0


def sign(x):
    return (x > 0) - (x < 0)


def name_of(r: bytes) -> bytes:
    return r[36:36 + r[12] - 1]


def flag_of(r: bytes) -> int:
    return struct.unpack_from("<H", r, 18)[0]


def name_order(recs):
    """bm2_sort -n: the names by strnum_cmp, then flag & 0xc0 ascending, then input order."""
    def cmp(x, y):
        (i, a), (j, b) = x, y
        c = sign(strnum_cmp(name_of(a), name_of(b)))
        if c:
            return c
        fa, fb = flag_of(a) & 0xC0, flag_of(b) & 0xC0
        return sign(fa - fb) or sign(i - j)
    return [r for _, r in sorted(enumerate(recs), key=functools.cmp_to_key(cmp))]


def coordinate_order(recs):
    """bm2_sort: samtools' coordinate key, ties in input order."""
    return sorted(recs, key=lambda r: bs.key(bu.fields(r)))


def expected_records(recs, by_name):
    return name_order(recs) if by_name else coordinate_order(recs)


def header_with_sort_order(text: str, so: str) -> str:
    """The first @HD line moved to the front with SO:<so> in place of its SO field (or appended), its other fields kept; an @HD line added when
    there is none.  Every line ends with a newline."""
    hd, rest = None, ""
    lines = text.split("\n")
    if text.endswith("\n"):
        lines = lines[:-1]
    for line in lines if text else []:
        if hd is None and (line == "@HD" or line.startswith("@HD\t")):
            fs, seen = [], False
            for f in line.split("\t")[1:]:
                if f.startswith("SO:"):
                    if not seen:
                        fs.append("SO:" + so)
                    seen = True
                else:
                    fs.append(f)
            if not seen:
                fs.append("SO:" + so)
            hd = "\t".join(["@HD"] + fs)
        else:
            rest += line + "\n"
    return (hd if hd is not None else "@HD\tVN:1.6\tSO:" + so) + "\n" + rest


def out_header(text: str, by_name: bool, argv) -> str:
    """bm2_sort's header text: the input's, trailing NULs dropped, rewritten for the order, then @PG ID:bm2_sort (.1, .2, ... when taken) with
    PP the input's last @PG.  argv: the command line, program first."""
    text = text.rstrip("\0")
    ids = [bu_tag(l, "ID:") for l in text.split("\n") if l.startswith("@PG\t")]
    pg = "bm2_sort"
    k = 1
    while pg in ids:
        pg = "bm2_sort.%d" % k; k += 1
    out = header_with_sort_order(text, "queryname" if by_name else "coordinate")
    return out + "@PG\tID:%s\tPN:bm2_sort%s\tVN:b200-r2\tCL:%s\n" % (pg, "\tPP:" + ids[-1] if ids else "", " ".join(argv))


def bu_tag(line, t):
    at = line.find("\t" + t)
    if at < 0:
        return ""
    e = line.find("\t", at + 4)
    return line[at + 4:] if e < 0 else line[at + 4:e]


# ---- the host emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bamsort_emul") / "libbamsortemul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "host_emul", "bamsort_emul.cpp"), os.path.join(ROOT, "tests", "host_emul", "bgzf_emul.cpp"),
                           "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.bamsort_emul_cmp.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.bamsort_emul_once.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                      C.c_void_p, C.c_void_p, C.c_void_p]
    lib.bamsort_emul_file.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_char_p, C.c_int, C.c_uint64, C.c_int, C.c_char_p,
                                      C.c_char_p, C.c_void_p, C.c_char_p, C.c_int]
    return lib


def emul_cmp(lib, names, pairs):
    """bam_qname_cmp (flags and ordinals equal) of names[i] against names[j] for each (i, j) of pairs -> list of -1 / 0 / 1."""
    blob = b"".join(n + b"\0" for n in names)
    offs = np.cumsum([0] + [len(n) + 1 for n in names[:-1]]).astype(np.int64)
    p = np.ascontiguousarray(np.array(pairs, np.int64).reshape(-1))
    out = np.zeros(max(len(pairs), 1), np.int32)
    b = np.frombuffer(blob, np.uint8)
    lib.bamsort_emul_cmp(b.ctypes.data, offs.ctypes.data, p.ctypes.data, len(pairs), out.ctypes.data)
    return [int(x) for x in out[:len(pairs)]]


def emul_once(lib, data, starts, carry=b"", last=True, by_name=True):
    starts = np.ascontiguousarray(starts, np.int64)
    cap = len(data) + len(carry) + 64 * (len(data) // 65280 + len(starts) + 4)
    z = np.zeros(cap, np.uint8); co = np.zeros(65536, np.uint8); recs = np.zeros(max(len(starts), 1), bs.SORT_REC_DT); sizes = np.zeros(3, np.int64)
    b, cb = bs._buf(data), bs._buf(carry)
    rc = lib.bamsort_emul_once(int(by_name), b.ctypes.data, starts.ctypes.data, len(starts), cb.ctypes.data, len(carry), int(last), z.ctypes.data,
                               cap, co.ctypes.data, recs.ctypes.data, sizes.ctypes.data)
    assert rc == 0
    return dict(z=z[:sizes[0]].tobytes(), carry=co[:sizes[1]].tobytes(), n_members=int(sizes[2]), recs=recs[:len(starts)])


def emul_file(lib, data, run_bytes, tmp_prefix, out_path, by_name=True, bai_path=None, out_off=0, n_ref=0, chunk=0, threads=2):
    stats = np.zeros(3, np.int64); err = C.create_string_buffer(512)
    b = bs._buf(data)
    rc = lib.bamsort_emul_file(int(by_name), b.ctypes.data, len(data), chunk, run_bytes, tmp_prefix.encode(), threads, out_off, n_ref,
                               out_path.encode(), bai_path.encode() if bai_path else None, stats.ctypes.data, err, 512)
    assert rc == 0, err.value
    return dict(runs=int(stats[0]), spill_bytes=int(stats[1]), windows=int(stats[2]))


def run_tool(argv, stdin=None, env=None, check=True):
    r = subprocess.run([TOOL] + argv, capture_output=True, timeout=900, stdin=stdin, env=env)
    if check:
        assert r.returncode == 0, r.stderr[-3000:]
    return r

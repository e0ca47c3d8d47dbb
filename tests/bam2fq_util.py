"""Helpers of the bm2_bam2fq tests: its rule (bwa-mem2_b200/csrc/bam2fq_device.cuh and bam2fq.h) restated in Python, BAM records built from
names, flags, bases and qualities, and the host emulation tests/host_emul/bam2fq_emul.cpp.

The rule, where it follows `samtools fastq` at its defaults: records with 0x100 or 0x800 are skipped (-F 0x900); a kept record is a READ1
(0x40 without 0x80), a READ2 (0x80 without 0x40) or other; its text is '@' QNAME [/1 | /2], SEQ, '+', QUAL + 33, a 0x10 record written
reverse-complemented (htslib's seq_comp_table) with its qualities reversed; /1 and /2 are on when interleaved and off when split, as samtools'
default is described.  Our choices: a record with QUAL '*' is a FASTA record ('>' QNAME [/1 | /2] and SEQ); a READ1 and READ2 of one name
are a pair wherever they lie, written at the later record, READ1 first; singletons come last; split mode without -0 or -s drops what would
go there; two READ1s or two READ2s of one name are an error."""
import ctypes as C
import os, struct, subprocess
import numpy as np
import markdup_util as mu

ROOT = mu.ROOT
CSRC = mu.CSRC
TOOL = os.path.join(ROOT, "bwa-mem2_b200", "bm2_bam2fq")
LETTERS = "=ACMGRSVTWYHKDBN"
# htslib's seq_comp_table (hts.c), for the 16 4-bit codes
SEQ_COMP_TABLE = [0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15]
SKIP, READ1, READ2, OTHER = 0, 1, 2, 3
REC_DT = np.dtype([("hash", "<u8"), ("text_len", "<i8"), ("kind", "<i4"), ("pad", "<i4")])


class Bam2fqError(Exception):
    pass


def rec(name, flag, seq, qual=None, cigar=None, tags=b""):
    """A BAM record: seq a string of LETTERS, qual a list of Phred values or None for '*'."""
    nm = name.encode() + b"\0"
    codes = [LETTERS.index(c) for c in seq]
    packed = bytes((codes[i] << 4) | (codes[i + 1] if i + 1 < len(codes) else 0) for i in range(0, len(codes), 2))
    q = bytes([0xFF] * len(seq)) if qual is None else bytes(qual)
    cig = b"".join(struct.pack("<I", ln << 4 | op) for ln, op in (cigar if cigar is not None else ([(len(seq), 0)] if seq else [])))
    body = struct.pack("<iiBBHHHiiii", -1, -1, len(nm), 0, 4680, len(cig) // 4, flag, len(seq), -1, -1, 0) + nm + cig + packed + q + tags
    return struct.pack("<i", len(body)) + body


def fields(r):
    l_name, n_cigar, flag, l_seq = r[12], struct.unpack_from("<H", r, 16)[0], struct.unpack_from("<H", r, 18)[0], struct.unpack_from("<i", r, 20)[0]
    name = r[36:36 + l_name - 1]
    at = 36 + l_name + 4 * n_cigar
    codes = [(r[at + i // 2] >> (4 * (1 - i % 2))) & 15 for i in range(l_seq)]
    q = r[at + (l_seq + 1) // 2: at + (l_seq + 1) // 2 + l_seq]
    return name, flag, codes, q


def kind(flag):
    if flag & 0x900:
        return SKIP
    e = flag & 0xC0
    return READ1 if e == 0x40 else READ2 if e == 0x80 else OTHER


def text(r, suffixes):
    name, flag, codes, q = fields(r)
    k = kind(flag)
    if not codes:
        raise Bam2fqError("read %s has no bases (l_seq 0)" % name.decode())
    fasta = q[0] == 0xFF
    if not fasta and max(q) > 93:
        raise Bam2fqError("read %s has a quality above 93" % name.decode())
    if flag & 0x10:
        codes = [SEQ_COMP_TABLE[c] for c in reversed(codes)]
        q = q[::-1]
    head = name + (b"/%d" % k if suffixes and k in (READ1, READ2) else b"")
    seq = "".join(LETTERS[c] for c in codes).encode()
    if fasta:
        return b">" + head + b"\n" + seq + b"\n"
    return b"@" + head + b"\n" + seq + b"\n+\n" + bytes(x + 33 for x in q) + b"\n"


def convert(recs, split=False, suffixes=None, other=True, single=True):
    """The whole rule over the records in input order -> ({stream: text}, stats).  Streams: 'main' (interleaved), or '1', '2', and '0' and
    's' when `other` / `single`."""
    if suffixes is None:
        suffixes = not split
    out = {k: b"" for k in (["1", "2"] + (["0"] if other else []) + (["s"] if single else []))} if split else {"main": b""}
    st = dict(records=len(recs), kept=0, pairs=0, others=0, singletons=0, others_dropped=0, singletons_dropped=0, pending_max=0)
    pend = {}                                      # name -> [(index, kind, record)], unjoined halves in input order
    for i, r in enumerate(recs):
        name, flag, _, _ = fields(r)
        k = kind(flag)
        if k == SKIP:
            continue
        t = text(r, suffixes)
        st["kept"] += 1
        if k == OTHER:
            st["others"] += 1
            if not split:
                out["main"] += t
            elif other:
                out["0"] += t
            else:
                st["others_dropped"] += 1
            continue
        if pend.get(name):
            j, kj, rj = pend[name].pop(0)
            if kj == k:
                raise Bam2fqError("read %s: two %s records" % (name.decode(), "READ1" if k == READ1 else "READ2"))
            t1, t2 = (t, text(rj, suffixes)) if k == READ1 else (text(rj, suffixes), t)
            st["pairs"] += 1
            if split:
                out["1"] += t1
                out["2"] += t2
            else:
                out["main"] += t1 + t2
        else:
            pend.setdefault(name, []).append((i, k, r))
    rest = sorted(x for v in pend.values() for x in v)
    st["singletons"] = len(rest)
    for _, _, r in rest:
        if not split:
            out["main"] += text(r, suffixes)
        elif single:
            out["s"] += text(r, suffixes)
        else:
            st["singletons_dropped"] += 1
    return out, st


def window_pending_max(recs, bounds):
    """pending_max of the windows [bounds[k], bounds[k+1]): the most halves carried after a window"""
    pend, best = {}, 0
    for a, b in zip(bounds[:-1], bounds[1:]):
        for r in recs[a:b]:
            name, flag, _, _ = fields(r)
            k = kind(flag)
            if k in (READ1, READ2):
                if pend.get(name):
                    pend[name].pop(0)
                else:
                    pend.setdefault(name, []).append(k)
        best = max(best, sum(len(v) for v in pend.values()))
    return best


# ---- the emulation ----

def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bam2fq_emul") / "libb2femul.so")
    he = os.path.join(ROOT, "tests", "host_emul")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(he, "bam2fq_emul.cpp"), os.path.join(he, "markdup_bam_emul.cpp"), os.path.join(he, "markdup_metrics_emul.cpp"),
                           os.path.join(he, "markdup_emul.cpp"), os.path.join(he, "bam_sort_emul.cpp"), os.path.join(he, "bgzf_emul.cpp"),
                           "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.b2f_emul_records.restype = C.c_int64
    lib.b2f_emul_records.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
    lib.b2f_emul_text.restype = C.c_int64
    lib.b2f_emul_text.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int64]
    lib.b2f_emul_run.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_char_p, C.c_int]
    return lib


STAT_NAMES = ("records", "kept", "pairs", "others", "singletons", "others_dropped", "singletons_dropped", "pending_max", "pending_bytes_max", "windows")


def _flat(recs):
    data = b"".join(recs)
    starts = np.array(np.cumsum([0] + [len(r) for r in recs[:-1]]), np.int64) if recs else np.zeros(1, np.int64)
    return (data if data else b"\0"), starts


def emul_records(lib, recs, suffixes):
    """-> (structured array of bm2_bam2fq_rec, first error as index << 4 | kind or -1)"""
    data, starts = _flat(recs)
    out = np.zeros(max(len(recs), 1), REC_DT)
    e = lib.b2f_emul_records(data, starts.ctypes.data, len(recs), int(suffixes), out.ctypes.data)
    return out[:len(recs)], int(e)


def emul_text(lib, window, order, extra, suffixes):
    """the text of order (window index i, or ~k for extra[k]) as the format kernel writes it"""
    wd, ws = _flat(window)
    xd, xs = _flat(extra)
    lst = np.ascontiguousarray(list(order) + [0], np.int64)
    n = lib.b2f_emul_text(lst.ctypes.data, len(order), wd, ws.ctypes.data, xd, xs.ctypes.data, int(suffixes), None, 0)
    buf = C.create_string_buffer(max(n, 1))
    lib.b2f_emul_text(lst.ctypes.data, len(order), wd, ws.ctypes.data, xd, xs.ctypes.data, int(suffixes), buf, n)
    return buf.raw[:n]


def emul_run(lib, in_path, paths, split=False, suffixes=None, threads=2, window=256 << 20):
    """paths: [-o] or [-1, -2, -0, -s] with '' for one not given -> (exit code, message or warnings, stats dict)"""
    if suffixes is None:
        suffixes = not split
    st = np.zeros(10, np.int64)
    err = C.create_string_buffer(4096)
    rc = lib.b2f_emul_run(in_path.encode(), "\n".join(paths).encode(), int(split), int(suffixes), threads, window, st.ctypes.data, err, 4096)
    return rc, err.value.decode(), dict(zip(STAT_NAMES, (int(v) for v in st)))

"""Helpers of the coordinate-sort tests: the host emulation of bm2_mem --sort (tests/host_emul/bam_sort_emul.cpp), BAM records built field by
field, samtools' coordinate key and bam_endpos computed from bam_util.fields, and a BAI reader with the region query of SAMv1 §5.3."""
import ctypes as C
import os, struct, subprocess
import numpy as np
import bam_util as bu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bwa-mem2_b200", "csrc")
SORT_REC_DT = np.dtype([("rid", "<i4"), ("pos", "<i4"), ("end", "<i4"), ("bin", "<u2"), ("flag", "<u2"), ("block", "<i8"), ("offset", "<i4"), ("_pad", "<i4")])


def build_emul(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bam_sort_emul") / "libbamsortemul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "host_emul", "bam_sort_emul.cpp"), os.path.join(ROOT, "tests", "host_emul", "bgzf_emul.cpp"),
                           "-o", so, "-lz", "-lpthread"])
    lib = C.CDLL(so)
    lib.bam_sort_emul_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.bam_sort_emul_once.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                       C.c_void_p, C.c_void_p, C.c_void_p]
    lib.bam_sort_emul_file.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_char_p, C.c_int, C.c_uint64, C.c_int, C.c_char_p,
                                       C.c_char_p, C.c_void_p, C.c_char_p, C.c_int]
    return lib


def _buf(data):
    return np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)


def emul_keys(lib, data):
    st = np.array([a for a, _ in bu.records(data)], np.int64)
    keys = np.zeros(max(len(st), 1), np.uint64); info = np.zeros(max(len(st), 1), SORT_REC_DT)
    b = _buf(data)
    lib.bam_sort_emul_keys(b.ctypes.data, st.ctypes.data, len(st), keys.ctypes.data, info.ctypes.data)
    return keys[:len(st)], info[:len(st)]


def emul_once(lib, data, starts, carry=b"", last=True):
    starts = np.ascontiguousarray(starts, np.int64)
    cap = len(data) + len(carry) + 64 * (len(data) // 65280 + len(starts) + 4)
    z = np.zeros(cap, np.uint8); co = np.zeros(65536, np.uint8); recs = np.zeros(max(len(starts), 1), SORT_REC_DT); sizes = np.zeros(3, np.int64)
    b, cb = _buf(data), _buf(carry)
    rc = lib.bam_sort_emul_once(b.ctypes.data, len(data), starts.ctypes.data, len(starts), cb.ctypes.data, len(carry), int(last), z.ctypes.data, cap,
                                co.ctypes.data, recs.ctypes.data, sizes.ctypes.data)
    assert rc == 0
    return dict(z=z[:sizes[0]].tobytes(), carry=co[:sizes[1]].tobytes(), n_members=int(sizes[2]), recs=recs[:len(starts)])


def emul_file(lib, data, run_bytes, tmp_prefix, out_path, bai_path=None, out_off=0, n_ref=0, chunk=0, threads=2):
    stats = np.zeros(3, np.int64); err = C.create_string_buffer(512)
    b = _buf(data)
    rc = lib.bam_sort_emul_file(b.ctypes.data, len(data), chunk, run_bytes, tmp_prefix.encode(), threads, out_off, n_ref, out_path.encode(),
                                bai_path.encode() if bai_path else None, stats.ctypes.data, err, 512)
    assert rc == 0, err.value
    return dict(runs=int(stats[0]), spill_bytes=int(stats[1]), windows=int(stats[2]))


def key(f):
    """samtools' coordinate key of a record's fields."""
    return ((f["rid"] & 0xFFFFFFFF) << 32) | (((f["pos"] + 1) & 0xFFFFFFFF) << 1) | (1 if f["flag"] & 16 else 0)


def end_pos(f):
    """bam_endpos: pos + the CIGAR's reference length; pos + 1 when unmapped or when nothing consumes the reference."""
    rl = 0 if f["flag"] & 4 else bu.ref_len(f["cigar"])
    return f["pos"] + (rl if rl else 1)


def rec_fields_raw(r):
    """refID, pos, flag and the stored CIGAR (not restored from CG) of a record."""
    rid, pos, lrn = struct.unpack("<iiB", r[4:13])
    ncig, flag = struct.unpack("<HH", r[16:20])
    return rid, pos, flag, list(struct.unpack("<%dI" % ncig, r[36 + lrn:36 + lrn + 4 * ncig]))


def make_rec(rid, pos, flag=0, cigar=((50, 0),), name=b"r", l_seq=None, extra=b"", cg=None):
    """One BAM record.  cigar: (length, op) pairs; cg: operations to store in CG:B,I behind the <l_seq>S<ref_len>N placeholder."""
    ops = [(n << 4) | op for n, op in cigar]
    if l_seq is None:
        l_seq = sum(n for n, op in (cg or cigar) if op in (0, 1, 4, 7, 8))
    tags = extra
    if cg is not None:
        cg_ops = [(n << 4) | op for n, op in cg]
        rl = sum(n for n, op in cg if op in (0, 2, 3, 7, 8))
        ops = [(l_seq << 4) | 4, (rl << 4) | 3]
        tags += b"CGBI" + struct.pack("<i", len(cg_ops)) + struct.pack("<%dI" % len(cg_ops), *cg_ops)
    if flag & 4:
        ops = []
    end = pos + (sum(o >> 4 for o in ops if o & 15 in (0, 2, 3, 7, 8)) or 1)
    bin_ = bu.reg2bin(pos, end) if rid >= 0 and pos >= 0 else 4680
    body = struct.pack("<iiBBHHHiiii", rid, pos, len(name) + 1, 60, bin_, len(ops), flag, l_seq, -1, -1, 0)
    body += name + b"\0" + struct.pack("<%dI" % len(ops), *ops) + bytes((l_seq + 1) // 2) + bytes([30]) * l_seq + tags
    return struct.pack("<i", len(body)) + body


# ---- BAI (SAMv1 §5.2) ----

def parse_bai(b: bytes):
    assert b[:4] == b"BAI\x01"
    at = 4
    n_ref = struct.unpack_from("<i", b, at)[0]; at += 4
    refs = []
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", b, at)[0]; at += 4
        bins, pseudo = {}, None
        for _ in range(n_bin):
            bn, nc = struct.unpack_from("<Ii", b, at); at += 8
            ch = [struct.unpack_from("<QQ", b, at + 16 * k) for k in range(nc)]; at += 16 * nc
            if bn == 37450:
                assert nc == 2
                pseudo = dict(beg=ch[0][0], end=ch[0][1], mapped=ch[1][0], unmapped=ch[1][1])
            else:
                assert bn not in bins and bn < 37450
                assert all(s < e for s, e in ch) and all(ch[k][1] <= ch[k + 1][0] for k in range(nc - 1))
                bins[bn] = ch
        n_intv = struct.unpack_from("<i", b, at)[0]; at += 4
        lin = list(struct.unpack_from("<%dQ" % n_intv, b, at)); at += 8 * n_intv
        refs.append(dict(bins=bins, lin=lin, pseudo=pseudo))
    n_no_coor = struct.unpack_from("<Q", b, at)[0] if at < len(b) else None
    at += 8
    assert at == len(b)
    return refs, n_no_coor


def reg2bins(beg, end):
    """SAMv1 §5.3: the bins that may hold records overlapping [beg, end)."""
    end -= 1
    out = [0]
    for shift, base in ((26, 1), (23, 9), (20, 73), (17, 585), (14, 4681)):
        out += list(range(base + (beg >> shift), base + (end >> shift) + 1))
    return out


class BgzfFile:
    """Random access to a BGZF file by virtual offset."""
    def __init__(self, data: bytes):
        self.data = data; self.cache = {}

    def block(self, addr):
        if addr not in self.cache:
            size = struct.unpack_from("<H", self.data, addr + 16)[0] + 1
            m = self.data[addr:addr + size]
            self.cache[addr] = (bu.members(m)[0][1], size)
        return self.cache[addr]

    def _read(self, addr, off, n):
        buf = b""
        while len(buf) < n:
            raw, size = self.block(addr)
            assert raw, "read past the last record"
            take = raw[off:off + n - len(buf)]
            buf += take; off += len(take)
            if off >= len(raw):
                addr, off = addr + size, 0
        return buf, addr, off

    def read_records(self, beg, end):
        """The records that start at virtual offsets in [beg, end), beg being a record start."""
        out, addr, off = [], beg >> 16, beg & 0xFFFF
        while (addr << 16 | off) < end and addr < len(self.data) and self.block(addr)[0]:
            hdr, addr, off = self._read(addr, off, 4)
            body, addr, off = self._read(addr, off, struct.unpack("<i", hdr)[0])
            out.append(hdr + body)
        return out


def query(bai_refs, bgzf, rid, beg, end):
    """Records reached through the index for [beg, end) on rid: the region's bins, chunks clipped by the linear index, decoded, filtered for
    overlap (pos < end and end_pos > beg)."""
    r = bai_refs[rid]
    lin = r["lin"]
    min_off = lin[min(beg >> 14, len(lin) - 1)] if lin and (beg >> 14) < len(lin) else (lin[-1] if lin else 0)
    chunks = sorted(c for bn in reg2bins(beg, end) for c in r["bins"].get(bn, []) if c[1] > min_off)
    got = []
    for s, e in chunks:
        for rec in bgzf.read_records(s, e):
            f = bu.fields(rec)
            if f["rid"] == rid and f["pos"] < end and end_pos(f) > beg:
                got.append(rec)
    return got

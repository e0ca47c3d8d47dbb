"""A small BAM reader for the tests (no samtools / pysam here): BGZF members inflated by Python's zlib with their framing checked, and BAM
records turned back into SAM text lines the way `samtools view` prints them."""
import struct, zlib
import numpy as np

EOF_BLOCK = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def members(data: bytes):
    """Split a BGZF stream into members, checking each: gzip header with the BC subfield, BSIZE, raw DEFLATE that ends where the member
    ends, CRC32, ISIZE, and at most 65536 bytes.  -> list of (member bytes, uncompressed bytes)."""
    out, at = [], 0
    while at < len(data):
        h = data[at:at + 18]
        assert len(h) == 18 and h[:4] == b"\x1f\x8b\x08\x04" and h[10:16] == b"\x06\x00BC\x02\x00", ("bad member header", at)
        size = struct.unpack("<H", h[16:18])[0] + 1
        assert size <= 65536 and at + size <= len(data), ("bad BSIZE", at, size)
        m = data[at:at + size]
        d = zlib.decompressobj(-15)
        raw = d.decompress(m[18:-8]) + d.flush()
        assert d.eof and not d.unused_data, ("DEFLATE data does not end with the member", at)
        crc, isize = struct.unpack("<II", m[-8:])
        assert crc == zlib.crc32(raw) and isize == len(raw), ("bad CRC32 / ISIZE", at)
        out.append((m, raw))
        at += size
    return out


def inflate(data: bytes) -> bytes:
    return b"".join(raw for _, raw in members(data))


def reg2bin(beg, end):
    end -= 1
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return base + (beg >> shift)
    return 0


def records(raw: bytes):
    """Uncompressed BAM records (no header) -> list of (offset, record bytes)."""
    out, at = [], 0
    while at < len(raw):
        n = struct.unpack("<i", raw[at:at + 4])[0]
        out.append((at, raw[at:at + 4 + n]))
        at += 4 + n
    assert at == len(raw)
    return out


def parse_header(raw: bytes):
    """-> (header text, [(name, length)], bytes used)."""
    assert raw[:4] == b"BAM\x01"
    lt = struct.unpack("<i", raw[4:8])[0]
    text = raw[8:8 + lt].decode()
    at = 8 + lt
    n = struct.unpack("<i", raw[at:at + 4])[0]; at += 4
    refs = []
    for _ in range(n):
        ln = struct.unpack("<i", raw[at:at + 4])[0]; at += 4
        name = raw[at:at + ln - 1].decode(); at += ln
        refs.append((name, struct.unpack("<i", raw[at:at + 4])[0])); at += 4
    return text, refs, at


INT_T = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}


def fields(rec: bytes):
    """One BAM record -> dict of its fixed fields, CIGAR (restored from CG when the kSmN placeholder is there), SEQ, QUAL and typed tags."""
    (bs, rid, pos, lrn, mapq, bin_, ncig, flag, lseq, nrid, npos, tlen) = struct.unpack("<iiiBBHHHiiii", rec[:36])
    assert bs == len(rec) - 4
    at = 36
    qname = rec[at:at + lrn - 1].decode(); assert rec[at + lrn - 1] == 0; at += lrn
    cig = list(struct.unpack("<%dI" % ncig, rec[at:at + 4 * ncig])); at += 4 * ncig
    sb = rec[at:at + (lseq + 1) // 2]; at += (lseq + 1) // 2
    seq = "".join("=ACMGRSVTWYHKDBN"[(sb[k // 2] >> (4 * (1 - k % 2))) & 15] for k in range(lseq))
    qual = rec[at:at + lseq]; at += lseq
    tags = []
    while at < len(rec):
        tg, t = rec[at:at + 2].decode(), chr(rec[at + 2]); at += 3
        if t == "A":
            v = chr(rec[at]); at += 1
        elif t in INT_T:
            sz = struct.calcsize(INT_T[t]); v = struct.unpack(INT_T[t], rec[at:at + sz])[0]; at += sz
        elif t == "f":
            v = struct.unpack("<f", rec[at:at + 4])[0]; at += 4
        elif t in "ZH":
            e = rec.index(b"\0", at); v = rec[at:e].decode(); at = e + 1
        elif t == "B":
            sub = chr(rec[at]); n = struct.unpack("<i", rec[at + 1:at + 5])[0]; at += 5
            fmt = INT_T.get(sub, "<f"); sz = struct.calcsize(fmt)
            v = (sub, [struct.unpack(fmt, rec[at + k * sz:at + (k + 1) * sz])[0] for k in range(n)]); at += n * sz
        else:
            raise AssertionError("unknown tag type " + t)
        tags.append((tg, t, v))
    cg = [v for tg, t, v in tags if tg == "CG" and t == "B"]
    if cg and ncig == 2 and cig[0] & 15 == 4 and cig[1] & 15 == 3:
        cig = cg[0][1]
        tags = [x for x in tags if x[0] != "CG"]
    return dict(rid=rid, pos=pos, mapq=mapq, bin=bin_, n_cigar_op=ncig, flag=flag, l_seq=lseq, next_rid=nrid, next_pos=npos, tlen=tlen,
                qname=qname, cigar=cig, seq=seq, qual=qual, tags=tags)


def ref_len(cigar):
    return sum(c >> 4 for c in cigar if c & 15 in (0, 2, 3, 7, 8))


def tag_text(tg, t, v):
    if t in INT_T:
        return "%s:i:%d" % (tg, v)
    if t == "f":
        return "%s:f:%s" % (tg, repr(float(np.float32(v))))
    if t == "B":
        return "%s:B:%s" % (tg, ",".join([v[0]] + [str(x) for x in v[1]]))
    return "%s:%s:%s" % (tg, t, v)


def to_sam(f, names):
    """A record's fields -> its SAM line (without the newline), as samtools view prints it; pa:f: as the float32 value (see norm)."""
    rname = names[f["rid"]] if f["rid"] >= 0 else "*"
    cig = "".join("%d%s" % (c >> 4, "MIDNSHP=X"[c & 15]) for c in f["cigar"]) or "*"
    rnext = "*" if f["next_rid"] < 0 else "=" if f["next_rid"] == f["rid"] else names[f["next_rid"]]
    seq = f["seq"] or "*"
    qual = "*" if f["l_seq"] == 0 or f["qual"][0] == 0xFF else "".join(chr(q + 33) for q in f["qual"])
    cols = [f["qname"], str(f["flag"]), rname, str(f["pos"] + 1), str(f["mapq"]), cig, rnext, str(f["next_pos"] + 1), str(f["tlen"]), seq, qual]
    return "\t".join(cols + [tag_text(*x) for x in f["tags"]])


def norm(line: str) -> str:
    """A SAM line with its float tags written as their float32 value (the text has %.3f, BAM the float of that text)."""
    cols = line.rstrip("\n").split("\t")
    for k in range(11, len(cols)):
        if cols[k][2:5] == ":f:":
            cols[k] = cols[k][:5] + repr(float(np.float32(float(cols[k][5:]))))
    return "\t".join(cols)


def bam_to_sam_lines(raw: bytes, names):
    return [to_sam(fields(r), names) for _, r in records(raw)]


def read_bam_file(data: bytes):
    """A whole BAM file -> (header text, refs, SAM lines, member list); checks the EOF block and that the header ends a member."""
    assert data.endswith(EOF_BLOCK), "no BGZF EOF block at the end"
    ms = members(data)
    raw = b"".join(r for _, r in ms)
    text, refs, used = parse_header(raw)
    ends = np.cumsum([len(r) for _, r in ms])
    assert used in ends.tolist(), "the header does not end a member"
    return text, refs, bam_to_sam_lines(raw[used:], [n for n, _ in refs]), ms


def htslib_cuts(n, starts):
    """The block starts htslib's writer makes of records starting at `starts` (bam_write1 -> bgzf_flush_try, bgzf_write)."""
    BLK = 0xff00
    bounds = [0] + [s for s in starts if s > 0] + [n]
    out, off, b0 = [], 0, 0
    for s, e in zip(bounds[:-1], bounds[1:]):
        if e <= s:
            continue
        if off and off + (e - s) > BLK:
            out.append(b0); b0, off = s, 0
        p = s
        while p < e:
            take = min(BLK - off, e - p); off += take; p += take
            if off == BLK:
                out.append(b0); b0, off = p, 0
    if off:
        out.append(b0)
    return out + [n]

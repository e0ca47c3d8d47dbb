"""BAM out without a GPU: bm2_bam_format_ex (csrc/sam_text.cpp) decoded back to SAM equals bm2_sam_format_ex's text on the same records,
its encoding rules (integer tag types, bin, CG for long CIGARs, errors), and the BGZF compressor's per-block logic (csrc/bgzf_device.cuh) run
by the host emulation tests/host_emul/bgzf_emul.cpp on an adversarial corpus: every member inflates with zlib to its input, with the right
CRC32 / ISIZE / BSIZE, and the blocks are cut where htslib's writer cuts them."""
import ctypes as C
import os, struct, subprocess, zlib
import numpy as np
import pytest
import bam_util as bu
import test_sam_text_cpu as st
import test_sam_text_extra_cpu as sx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bwa-mem2_b200", "csrc")


@pytest.fixture(scope="module")
def c0(pkg, golden_dir):
    """The golden C0 reads' records as test_sam_text_cpu builds them (the SAM stage's device logic run by the host emulation)."""
    capi = pkg.capi
    import oracle_lib as ol
    idx = capi.Index(golden_dir + "/c0_index/ref.fa")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    codes = reads.reshape(-1); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    names = [l.split()[1] for i, l in enumerate(open(golden_dir + "/c0_index/ref.fa.ann")) if i % 2 == 1]
    opt = capi.default_opt(); opt.flag |= 0x2 | 0x100
    regs, ro, _, rc = ol.seed_chain_extend(idx, opt, codes, offs)
    assert rc == 0
    pes = capi.pestat(opt, idx.desc.l_pac, regs, ro)
    lh = np.array([v for d in range(4) for v in (pes[d]["low"], pes[d]["high"], pes[d]["failed"])], np.int32)
    as_ = np.array([v for d in range(4) for v in (pes[d]["avg"], pes[d]["std"])], np.float64)
    e_recs, e_cig, e_md, aux, xas, xops = st._emul_full(capi, idx, opt, codes, offs, regs, ro, lh, as_)
    recs, xa, cig = st._to_product_records(capi, e_recs, e_cig, aux, xas, xops)
    idx.close()
    rng = np.random.default_rng(3)
    quals = rng.integers(35, 74, len(codes)).astype(np.uint8)
    return dict(recs=recs, xa=xa, cig=cig, md=e_md, codes=codes, offs=offs, names=names, reads=reads, quals=quals)


def _both(capi, c, **kw):
    args = (c["recs"], c["xa"], c["cig"], c["md"], c["codes"], c["offs"], c["names"])
    text = capi.sam_format(*args, **kw).decode()
    bam, ro = capi.bam_format(*args, **kw)
    return text, bam, ro


def _check_equal(c, text, bam, ro):
    want = [bu.norm(l) for l in text.split("\n") if l]
    got = [bu.norm(l) for l in bu.bam_to_sam_lines(bam, c["names"])]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g == w
    # read_off: where each read's records start
    starts = [at for at, _ in bu.records(bam)]
    per_read = np.bincount(c["recs"]["read"], minlength=len(ro) - 1)
    assert ro[0] == 0 and ro[-1] == len(bam)
    assert list(ro[:-1][per_read > 0]) == [starts[k] for k in np.concatenate([[0], np.cumsum(per_read)])[:-1][per_read > 0]]


@pytest.mark.parametrize("threads", [1, 4])
def test_bam_records_decode_to_the_sam_text(pkg, c0, threads):
    text, bam, ro = _both(pkg.capi, c0, read_names=["p%d" % (i // 2) for i in range(len(c0["reads"]))], quals=c0["quals"], n_threads=threads)
    assert text.count("\n") == len(c0["recs"]) and ("\tXA:Z:" in text or "\tSA:Z:" in text)
    _check_equal(c0, text, bam, ro)


@pytest.mark.parametrize("threads", [1, 4])
def test_bam_with_rg_comments_xr_and_no_qualities(pkg, c0, threads):
    """-R, -C with comments that are SAM tags, -V annotations (one with a tab), and reads without qualities (FASTA): QUAL 0xFF."""
    reads = c0["reads"]
    b1, s1 = sx._fastq(reads, 0); b2, s2 = sx._fastq(reads, 1)
    spans = [s for pair in zip(s1, s2) for s in pair]
    bufs = (b1, b2)
    # only the BX:Z:...\tCB:Z:... comments; a 'plain comment' is the error case below
    keep = [s[3] > 0 and bufs[r % 2][s[2]:s[2] + s[3]].startswith(b"BX:Z:") for r, s in enumerate(spans)]
    nb = np.array([s[0] for s in spans], np.int64); nl = np.array([s[1] for s in spans], np.int32)
    cb = np.array([s[2] for s in spans], np.int64); cl = np.array([s[3] if k else 0 for s, k in zip(spans, keep)], np.int32)
    assert cl.astype(bool).sum() > 10
    qp = (np.arange(len(reads)) % 3 != 0).astype(np.uint8)
    anno = ["first contig description", "", "has\ta tab", ""]
    text, bam, ro = _both(pkg.capi, c0, quals=c0["quals"], n_threads=threads, name_spans=(b1, b2, nb, nl), rg_id="grp.1", comments=(cb, cl),
                          contig_anno=anno, ref_hdr=True, qual_present=qp)
    assert "\tRG:Z:grp.1" in text and "\tBX:Z:" in text and "\tXR:Z:has a tab" in text and "\t*\tNM:i:" in text
    _check_equal(c0, text, bam, ro)
    raw = [bu.fields(r) for _, r in bu.records(bam)]
    assert any(f["l_seq"] and f["qual"] == b"\xff" * f["l_seq"] for f in raw)
    assert all(dict((t, ty) for t, ty, _ in f["tags"]).get("BX", "Z") == "Z" for f in raw)


def _one_read(capi, n_cig=1, name="q1", flag=0, rid=0, pos=100, rnext=-1, pnext=0, score=-1, sub=-1, cigar=None, l_seq=10):
    recs = np.zeros(1, capi.SAM_REC_DT)
    cig = np.array(cigar if cigar is not None else [l_seq << 4], np.uint32)
    md = np.frombuffer(b"%d\0" % l_seq, np.uint8)
    recs[0] = 0
    for k, v in dict(read=0, flag=flag, rid=rid, rnext=rnext, mapq=60, nm=0, score=score, sub=sub, reg=-1, n_cigar=len(cig) if rid >= 0 else 0,
                     n_md=len(md), pos=pos, pnext=pnext, tlen=0, cigar_off=0, md_off=0).items():
        recs[k] = v
    codes = (np.arange(l_seq) % 4).astype(np.uint8)
    return dict(recs=recs, xa=np.zeros(0, capi.SAM_XA_DT), cig=cig, md=md, codes=codes, offs=np.array([0, l_seq], np.int64), names=["c1", "c2"]), name


def _tags(bam):
    return [(t, ty, v) for _, r in bu.records(bam) for t, ty, v in bu.fields(r)["tags"]]


@pytest.mark.parametrize("v,ty", [(0, "C"), (127, "C"), (128, "C"), (255, "C"), (256, "S"), (65535, "S"), (65536, "I"), (2**31 - 1, "I")])
def test_integer_tags_take_htslibs_smallest_type(pkg, v, ty):
    c, name = _one_read(pkg.capi, score=v, sub=v)
    bam, _ = pkg.capi.bam_format(c["recs"], c["xa"], c["cig"], c["md"], c["codes"], c["offs"], c["names"], read_names=[name])
    t = dict((tg, (tt, vv)) for tg, tt, vv in _tags(bam))
    assert t["AS"] == (ty, v) and t["XS"] == (ty, v) and t["NM"] == ("C", 0)


def test_comment_tags_are_typed_as_sam_parse1_types_them(pkg):
    cmt = b"X1:i:-1\tX2:i:-128\tX3:i:-129\tX4:i:-32768\tX5:i:-32769\tX6:i:127\tX7:i:128\tX8:i:65536\tXf:f:1.5\tXa:A:q\tXh:H:1AE3\tXb:B:s,-2,300\tXz:Z:a b"
    c, name = _one_read(pkg.capi)
    buf = b"@q1 " + cmt + b"\n"
    bam, _ = pkg.capi.bam_format(c["recs"], c["xa"], c["cig"], c["md"], c["codes"], c["offs"], c["names"],
                                 name_spans=(buf, None, np.array([1], np.int64), np.array([2], np.int32)),
                                 comments=(np.array([4], np.int64), np.array([len(cmt)], np.int32)))
    t = dict((tg, (tt, vv)) for tg, tt, vv in _tags(bam))
    assert t["X1"] == ("c", -1) and t["X2"] == ("c", -128) and t["X3"] == ("s", -129) and t["X4"] == ("s", -32768) and t["X5"] == ("i", -32769)
    assert t["X6"] == ("C", 127) and t["X7"] == ("C", 128) and t["X8"] == ("I", 65536)
    assert t["Xf"] == ("f", 1.5) and t["Xa"] == ("A", "q") and t["Xh"] == ("H", "1AE3") and t["Xb"] == ("B", ("s", [-2, 300])) and t["Xz"] == ("Z", "a b")


@pytest.mark.parametrize("case", ["mapped", "unmapped_placed_mate", "unplaced", "deletion_span"])
def test_bin_is_reg2bin(pkg, case):
    capi = pkg.capi
    if case == "mapped":
        c, name = _one_read(capi, pos=16380, l_seq=10)                       # spans the 16 kbp bin boundary
    elif case == "unmapped_placed_mate":
        c, name = _one_read(capi, flag=0x4 | 0x1, pos=5000, rnext=0, pnext=5000, cigar=[])
        c["recs"]["n_cigar"] = 0
    elif case == "unplaced":
        c, name = _one_read(capi, flag=0x4, rid=-1, pos=0, cigar=[])
    else:
        c, name = _one_read(capi, pos=1 << 20, cigar=[5 << 4, (100000 << 4) | 2, 5 << 4])
    bam, _ = capi.bam_format(c["recs"], c["xa"], c["cig"], c["md"], c["codes"], c["offs"], c["names"], read_names=[name])
    f = bu.fields(bu.records(bam)[0][1])
    if case == "unplaced":
        assert f["pos"] == -1 and f["rid"] == -1 and f["bin"] == 4680
    else:
        rl = bu.ref_len(f["cigar"])
        assert f["bin"] == bu.reg2bin(f["pos"], f["pos"] + (rl if rl else 1))
    assert f["pos"] == int(c["recs"]["pos"][0]) - 1 or case == "unplaced"


def test_more_than_65535_cigar_operations_go_to_cg(pkg):
    capi = pkg.capi
    n_pairs = 35000
    cig = [1 << 4 | 0, 1 << 4 | 2] * n_pairs + [1 << 4 | 0]             # 70001 operations: M D M D ... M
    c, name = _one_read(capi, cigar=cig, l_seq=n_pairs + 1)
    args = (c["recs"], c["xa"], c["cig"], c["md"], c["codes"], c["offs"], c["names"])
    text = capi.sam_format(*args, read_names=[name]).decode()
    bam, _ = capi.bam_format(*args, read_names=[name])
    rec = bu.records(bam)[0][1]
    assert struct.unpack("<H", rec[16:18])[0] == 2                         # n_cigar_op: the kSmN placeholder
    ph = struct.unpack("<II", rec[36 + 3:36 + 3 + 8])
    assert ph == ((n_pairs + 1) << 4 | 4, (2 * n_pairs + 1) << 4 | 3)
    assert bu.bam_to_sam_lines(bam, c["names"]) == [text.rstrip("\n")]


def test_long_qname_and_unparseable_comment_are_errors(pkg):
    capi = pkg.capi
    c, _ = _one_read(capi)
    args = (c["recs"], c["xa"], c["cig"], c["md"], c["codes"], c["offs"], c["names"])
    with pytest.raises(capi.Bm2Error, match="x" * 255):
        capi.bam_format(*args, read_names=["x" * 255])
    capi.bam_format(*args, read_names=["x" * 254])
    buf = b"@frag7 1:N:0:ACGT\n"
    with pytest.raises(capi.Bm2Error, match="frag7"):
        capi.bam_format(*args, name_spans=(buf, None, np.array([1], np.int64), np.array([5], np.int32)),
                        comments=(np.array([7], np.int64), np.array([10], np.int32)))


# ---- the compressor's per-block logic, emulated on the host ----

def build_emul(tmp_path_factory):
    """tests/host_emul/bgzf_emul.cpp compiled with g++ and loaded."""
    so = str(tmp_path_factory.mktemp("bgzf_emul") / "libbgzfemul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + CSRC, os.path.join(ROOT, "tests", "host_emul", "bgzf_emul.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.bgzf_emul.restype = C.c_int64
    lib.bgzf_emul.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
    lib.bgzf_emul_cuts.restype = C.c_int64
    lib.bgzf_emul_cuts.argtypes = [C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
    lib.bgzf_emul_block.restype = C.c_int
    lib.bgzf_emul_block.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return build_emul(tmp_path_factory)


def emul_stream(lib, data: bytes, cut):
    cut = np.ascontiguousarray(cut, np.int64)
    buf = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
    cap = len(data) + 64 * (len(data) // 65280 + len(cut) + 2) + 64
    out = np.zeros(cap, np.uint8)
    k = lib.bgzf_emul(buf.ctypes.data, len(data), cut.ctypes.data, len(cut), out.ctypes.data, cap)
    assert k >= 0
    starts = np.zeros(len(data) // 1 + len(cut) + 4 if len(data) < 10**6 else len(data) // 100 + len(cut) + 4, np.int64)
    nb = lib.bgzf_emul_cuts(len(data), cut.ctypes.data, len(cut), starts.ctypes.data, len(starts))
    return out[:k].tobytes(), starts[:nb + 1].tolist()


def emul_block(lib, data: bytes) -> bytes:
    buf = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
    out = np.zeros(65536, np.uint8)
    k = lib.bgzf_emul_block(buf.ctypes.data, len(data), out.ctypes.data)
    assert k > 0
    return out[:k].tobytes()


def realistic_bam(n_reads=3000, seed=7):
    """Uncompressed BAM records of paired 151 bp reads with Illumina-like qualities (a position-dependent Markov walk) -> (bytes, record starts)."""
    import bam_inputs
    return bam_inputs.bam_records(n_reads, seed)


def corpus():
    rng = np.random.default_rng(11)
    rnd = rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes()
    r32 = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    no_match = bytes(range(256)) + bytes(reversed(range(256)))
    one_dist = (b"ab" + bytes(rng.integers(99, 123, 998, dtype=np.uint8))) * 2             # one match, at distance 1000
    runs3 = b"".join(b"%c%cz" % (65 + k % 26, 97 + (k * 7) % 26) + rng.integers(0, 256, 5, dtype=np.uint8).tobytes() for k in range(6000))
    return {
        "empty": (b"", []), "one_byte": (b"A", []), "exact_block": (rnd[:65280], []), "zeros": (bytes(300_000), []),
        "repeated_symbol": (b"q" * 131_000, []), "random": (rnd, []), "len3": (runs3, []), "len258": (b"xy" * 40_000, []),
        "dist32768": (r32 + r32[:4000] + rnd[:20000], []), "no_match": (no_match, []), "one_distance_code": (one_dist, []),
        "records": (rnd[:100_000], [0, 10, 65270, 65290, 70000, 99_999]),
        "big_record": (bytes(200_000), [0, 5, 150_000]),
    }


@pytest.mark.parametrize("name", list(corpus().keys()))
def test_emulated_members_inflate_and_are_cut_as_htslib_cuts(emul, name):
    data, cut = corpus()[name]
    z, starts = emul_stream(emul, data, cut)
    ms = bu.members(z)
    assert b"".join(raw for _, raw in ms) == data
    assert starts == bu.htslib_cuts(len(data), cut)
    assert [len(raw) for _, raw in ms] == list(np.diff(starts))
    if name == "random":
        assert all(m[18] & 7 == 1 for m, _ in ms)                                      # BFINAL, BTYPE 00: stored
    if name in ("zeros", "repeated_symbol", "len258"):
        assert all(m[18] & 6 == 4 for m, _ in ms) and len(z) < len(data) // 50       # dynamic Huffman


@pytest.mark.parametrize("n", [0, 1, 2, 3, 255, 256, 257, 65279, 65280])
def test_emulated_block_sizes(emul, n):
    rng = np.random.default_rng(n)
    for data in (bytes(rng.integers(65, 69, n, dtype=np.uint8)), bytes(rng.integers(0, 256, n, dtype=np.uint8))):
        ms = bu.members(emul_block(emul, data))
        assert len(ms) == 1 and ms[0][1] == data


def test_emulated_bam_stream_and_ratio_against_zlib(emul):
    data, cut = realistic_bam()
    z, starts = emul_stream(emul, data, cut)
    assert bu.inflate(z) == data and starts == bu.htslib_cuts(len(data), cut)
    zl1 = sum(len(zlib.compress(data[a:b], 1)) - 6 + 26 for a, b in zip(starts[:-1], starts[1:]))
    assert len(z) < 1.10 * zl1, (len(z), zl1)

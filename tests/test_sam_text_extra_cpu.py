"""bm2_sam_format_ex (csrc/sam_text.cpp): the -R / -C / -V additions of mem_aln2sam (src/bwamem.cpp:1693, :1720-1728) on the records of the SAM
stage's device logic (host emulation) for the golden C0 reads, against the unmodified reference run live with `-R ... -C -V` on the same reads
written as FASTQ with comments, on a copy of the C0 index whose contigs carry annotations (one of them with a tab)."""
import os, shutil, subprocess
import numpy as np
import pytest
import test_sam_text_cpu as st

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANNOS = ["first contig description", "", "has\ta tab", "(null)"]          # the last one is the reference's spelling of "none"


def _fastq(reads, which, eol=b"\n"):
    recs, spans = [], []
    at = 0
    for i in range(which, len(reads), 2):
        name = b"p%d/%d" % (i // 2, which + 1)
        cmt = b"" if i % 7 == 0 else (b"BX:Z:AC%d\tCB:Z:%d" % (i, i % 5) if i % 3 else b"plain comment %d" % i)
        head = b"@" + name + ((b" " + cmt) if cmt else b"")
        seq = bytes(b"ACGTN"[c] for c in reads[i])
        rec = head + eol + seq + eol + b"+" + eol + b"I" * len(seq) + eol
        nb = at + 1; nl = len(name) - 2                                       # trim_readno
        cb = at + 1 + len(name) + 1 if cmt else 0
        spans.append((nb, nl, cb, len(cmt)))
        recs.append(rec); at += len(rec)
    return b"".join(recs), spans


@pytest.mark.parametrize("eol", [b"\n", b"\r\n"], ids=["lf", "crlf"])
def test_rg_comment_and_xr_equal_the_reference(pkg, golden_dir, tmp_path, eol):
    isa = "avx512bw" if "avx512bw" in open("/proc/cpuinfo").read() else "avx2"
    drv = os.path.join(ROOT, "oracle", "_ref", isa, "ref_driver")
    if not os.path.exists(drv):
        pytest.skip("oracle/_ref not built")
    capi = pkg.capi
    import oracle_lib as ol
    d = tmp_path / "idx"; d.mkdir()
    for f in os.listdir(golden_dir + "/c0_index"):
        shutil.copy(os.path.join(golden_dir, "c0_index", f), d / f)
    lines = open(d / "ref.fa.ann").read().split("\n")
    for k in range(4):                                                      # "gi name anno" lines (src/bntseq.cpp:86-90)
        gi, name = lines[1 + 2 * k].split()[:2]
        lines[1 + 2 * k] = "%s %s %s" % (gi, name, ANNOS[k]) if ANNOS[k] else "%s %s" % (gi, name)
    (d / "ref.fa.ann").write_text("\n".join(lines))
    prefix = str(d / "ref.fa")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    b1, s1 = _fastq(reads, 0, eol); b2, s2 = _fastq(reads, 1, eol)
    (tmp_path / "r1.fq").write_bytes(b1); (tmp_path / "r2.fq").write_bytes(b2)
    rg = r"@RG\tID:grp.1\tSM:s1"
    ref = subprocess.run([drv, "mem", "-K", "100000000", "-R", rg, "-C", "-V", prefix, str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")],
                         env=dict(os.environ, BM2_MODE="ref"), capture_output=True, timeout=600)
    assert ref.returncode == 0, ref.stderr[-2000:]
    want = [ln + "\n" for ln in ref.stdout.decode().split("\n") if ln and not ln.startswith("@")]
    assert sum("\tXR:Z:has a tab" in ln for ln in want) > 0 and sum("\tXR:Z:first contig description" in ln for ln in want) > 0
    assert sum("\tBX:Z:" in ln for ln in want) > 0 and all("\tRG:Z:grp.1" in ln for ln in want)

    idx = capi.Index(prefix)
    codes = reads.reshape(-1); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    opt = capi.default_opt(); opt.flag |= 0x2 | 0x100
    regs, ro, _, rc = ol.seed_chain_extend(idx, opt, codes, offs)
    assert rc == 0
    pes = capi.pestat(opt, idx.desc.l_pac, regs, ro)
    lh = np.array([v for dd in range(4) for v in (pes[dd]["low"], pes[dd]["high"], pes[dd]["failed"])], np.int32)
    as_ = np.array([v for dd in range(4) for v in (pes[dd]["avg"], pes[dd]["std"])], np.float64)
    e_recs, e_cig, e_md, aux, xas, xops = st._emul_full(capi, idx, opt, codes, offs, regs, ro, lh, as_)
    recs, xa, cig = st._to_product_records(capi, e_recs, e_cig, aux, xas, xops)
    spans = [s for pair in zip(s1, s2) for s in pair]                        # reads 2i / 2i+1 from buffers 1 / 2
    nb = np.array([s[0] for s in spans], np.int64); nl = np.array([s[1] for s in spans], np.int32)
    cb = np.array([s[2] for s in spans], np.int64); cl = np.array([s[3] for s in spans], np.int32)
    names = [l.split()[1] for i, l in enumerate(open(golden_dir + "/c0_index/ref.fa.ann")) if i % 2 == 1]
    anno = [a if a != "(null)" else "" for a in ANNOS]
    quals = np.full(len(codes), ord("I"), np.uint8)
    for threads in (1, 3):
        got = capi.sam_format(recs, xa, cig, e_md, codes, offs, names, quals=quals, n_threads=threads, name_spans=(b1, b2, nb, nl),
                              rg_id="grp.1", comments=(cb, cl), contig_anno=anno, ref_hdr=True).decode()
        assert got == "".join(want)
    # without the additions, bm2_sam_format_ex is bm2_sam_format
    plain = capi.sam_format(recs, xa, cig, e_md, codes, offs, names, quals=quals, name_spans=(b1, b2, nb, nl))
    none = capi.sam_format(recs, xa, cig, e_md, codes, offs, names, quals=quals, name_spans=(b1, b2, nb, nl), rg_id="", ref_hdr=False,
                           comments=(cb, np.zeros_like(cl)))
    assert plain == none
    idx.close()

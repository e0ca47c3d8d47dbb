"""GPU parity of seam 4 (bm2_sam_pe: mate rescue, pairing, MAPQ, CIGAR / NM / MD, SAM records, XA entries) through the C ABI: every
SAM column and the NM MD AS XS XA pa tags of every line of the UNMODIFIED reference's output on C0 (tests/golden/c0.sam), and the
oracle on flag variants and on the tandem-repeat reads (hundreds of regions per read).
The per-pair logic the kernel launches is also checked on the host
(tests/test_oracle_sam_pe.py)."""
import numpy as np
import pytest
import oracle_lib as ol
import test_oracle_sam_pe as tp

pytestmark = pytest.mark.gpu


def _xa_strings(recs, xa, cigar, names):
    by_key = {}
    for e in xa:
        ops = cigar[e["cigar_off"]:e["cigar_off"] + e["n_cigar"]]
        txt = f"{names[e['rid']]},{'+-'[e['is_rev']]}{e['pos'] + 1}," + "".join(f"{v >> 4}{'MIDSHN'[v & 15]}" for v in ops) + f",{e['nm']};"
        by_key.setdefault((int(e["read"]), int(e["reg"])), []).append(txt)
    return ["".join(by_key.get((int(r["read"]), int(r["reg"])), [])) if r["reg"] >= 0 else "" for r in recs]


@pytest.fixture(scope="module")
def c0(pkg, golden_dir):
    capi = pkg.capi
    idx = capi.Index(golden_dir + "/c0_index/ref.fa")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    codes = reads.reshape(-1); offs = (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    names = [l.split()[1] for i, l in enumerate(open(golden_dir + "/c0_index/ref.fa.ann")) if i % 2 == 1]
    yield capi, idx, reads, codes, offs, names
    idx.close()


def test_sam_records_match_reference_golden(c0, golden_dir):
    capi, idx, reads, codes, offs, names = c0
    opt = capi.default_opt(); opt.flag |= 0x2
    ctx = capi.Context(0, index=idx, opt=opt)
    try:
        regs, ro = ctx.seed_chain_extend(codes, offs)
        pes = capi.pestat(opt, idx.desc.l_pac, regs, ro)
        recs, xa, cig, md = ctx.sam_pe(codes, offs, regs, ro, pes)
    finally:
        ctx.close()
    lines = [ln.rstrip("\n") for ln in open(golden_dir + "/c0.sam") if not ln.startswith("@")]
    tp._compare(tp.fields(recs, cig, md, names), tp.parse_sam(lines))
    assert _xa_strings(recs, xa, cig, names) == tp.xa_of_lines(lines)
    import sam_text                                                  # the whole text (SEQ / QUAL, MC, SA ...) from the records
    txt = sam_text.format_lines(recs, cig, md, _xa_strings(recs, xa, cig, names), names, codes, offs)
    want = [ln.split("\t", 1)[1] for ln in lines]
    bad = [i for i in range(len(want)) if txt[i] != want[i]]
    assert not bad, (len(bad), [(txt[i], want[i]) for i in bad[:2]])
    pa_want = [([f for f in w.split("\t") if f.startswith("pa:f:")] or [""])[0] for w in lines]
    pa_got = [("pa:f:%.3f" % (float(r["score"]) / float(r["alt_sc"]))) if r["alt_sc"] > 0 and not (r["flag"] & 0x100) else "" for r in recs]
    assert pa_got == pa_want


@pytest.mark.parametrize("flags", [0x8, 0x10, 0x4, 0x20, 0x200, 0x1800], ids=["all", "no_multi", "no_pairing", "no_rescue", "softclip", "primary5"])
def test_sam_records_match_oracle_with_flags(c0, flags):
    capi, idx, reads, codes, offs, names = c0
    opt = capi.default_opt(); opt.flag |= 0x2 | flags
    ctx = capi.Context(0, index=idx, opt=opt)
    try:
        regs, ro = ctx.seed_chain_extend(codes, offs)
        pes = capi.pestat(opt, idx.desc.l_pac, regs, ro)
        recs, xa, cig, md = ctx.sam_pe(codes, offs, regs, ro, pes)
    finally:
        ctx.close()
    lh = np.array([v for d in range(4) for v in (pes[d]["low"], pes[d]["high"], pes[d]["failed"])], np.int32)
    as_ = np.array([v for d in range(4) for v in (pes[d]["avg"], pes[d]["std"])], np.float64)
    want = tp.oracle_sam_pe(capi, idx, opt, codes, offs, regs, ro, lh, as_)
    tp._compare(tp.fields(recs, cig, md, names), tp.fields(*want, names))


def test_tandem_repeat_pairs_match_oracle(pkg, golden_dir):
    """Hundreds of regions per read: large arenas, several waves' worth of scratch per pair."""
    capi = pkg.capi
    idx = capi.Index(golden_dir + "/tandem_index/ref.fa")
    rd = np.load(golden_dir + "/tandem_reads.npz"); codes, offs = rd["codes"], rd["offs"]
    opt = capi.default_opt(); opt.flag |= 0x2
    ctx = capi.Context(0, index=idx, opt=opt)
    try:
        regs, ro = ctx.seed_chain_extend(codes, offs)
        pes = np.zeros(4, capi.PESTAT_DT)                              # -I style statistics: FR pairs of 100..700 bp
        pes["failed"] = 1
        pes[1] = (100, 700, 0, 0, 400.0, 80.0)
        recs, xa, cig, md = ctx.sam_pe(codes, offs, regs, ro, pes)
    finally:
        ctx.close()
    lh = np.array([v for d in range(4) for v in (pes[d]["low"], pes[d]["high"], pes[d]["failed"])], np.int32)
    as_ = np.array([v for d in range(4) for v in (pes[d]["avg"], pes[d]["std"])], np.float64)
    want = tp.oracle_sam_pe(capi, idx, opt, codes, offs, regs, ro, lh, as_)
    names = ["tr1", "tr2"]
    tp._compare(tp.fields(recs, cig, md, names), tp.fields(*want, names))
    idx.close()


@pytest.mark.parametrize("flags", [0, 0x8, 0x1800], ids=["default", "all", "primary5"])
def test_single_end_records_match_oracle(c0, flags):
    """bm2_sam_se: the r1 reads of C0 as single-end reads, against the oracle's single-end SAM stage (pinned to the live reference by
    tests/test_oracle_sam_se.py)."""
    import test_oracle_sam_se as ts
    capi, idx, reads, codes, offs, names = c0
    r1 = reads[0::2]; codes1 = np.ascontiguousarray(r1.reshape(-1)); offs1 = (np.arange(len(r1) + 1) * r1.shape[1]).astype(np.int64)
    opt = capi.default_opt(); opt.flag |= flags
    ctx = capi.Context(0, index=idx, opt=opt)
    try:
        regs, ro = ctx.seed_chain_extend(codes1, offs1)
        recs, xa, cig, md = ctx.sam_se(codes1, offs1, regs, ro)
    finally:
        ctx.close()
    alns, ocig, omd = ts.oracle_sam_se(capi, idx, opt, codes1, offs1, regs, ro)
    want = ts.sam_fields(alns, ocig, omd, names, soft_clip_all=False)
    assert ts.rec_fields(recs, cig, md, names) == want


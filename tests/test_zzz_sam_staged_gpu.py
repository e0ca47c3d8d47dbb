"""GPU parity of the STAGED mate rescue of bm2_sam_pe (bm2_set_sam_staged: sam_jobs_kernel lists the windows, sam_ksw_jobs_kernel aligns
them one window per warp - or, mode 2, sam_ksw_jobs_thread_kernel one window per thread -, the per-pair kernel looks them up): the same records as the unmodified reference's SAM on C0, as the default
mode on the flag variants, and as the oracle on the tandem-repeat pairs.  Written after the round's GPU minutes were spent: non-strict xfail until it
has run once (the same split is checked on the host: tests/test_oracle_sam_pe.py::test_staged_rescue_equals_the_per_pair_block).
Named to run after every other file - a fault in kernels that have never run must not take later tests with it."""
import numpy as np
import pytest
import test_oracle_sam_pe as tp
from test_zz_sam_gpu import c0, _xa_strings          # noqa: F401  (fixture)

pytestmark = [pytest.mark.gpu]


def _run(capi, idx, opt, codes, offs, staged, pes=None):
    ctx = capi.Context(0, index=idx, opt=opt)
    try:
        ctx.set_sam_staged(staged)
        regs, ro = ctx.seed_chain_extend(codes, offs)
        if pes is None:
            pes = capi.pestat(opt, idx.desc.l_pac, regs, ro)
        out = ctx.sam_pe(codes, offs, regs, ro, pes)
        st = ctx.last_sam_stats()
    finally:
        ctx.close()
    return out, st, (regs, ro, pes)


MODES = pytest.mark.parametrize("mode", [1, 2], ids=["warp_per_window", "thread_per_window"])


@MODES
def test_staged_records_match_reference_golden(c0, golden_dir, mode):
    capi, idx, reads, codes, offs, names = c0
    opt = capi.default_opt(); opt.flag |= 0x2
    (recs, xa, cig, md), st, _ = _run(capi, idx, opt, codes, offs, mode)
    lines = [ln.rstrip("\n") for ln in open(golden_dir + "/c0.sam") if not ln.startswith("@")]
    tp._compare(tp.fields(recs, cig, md, names), tp.parse_sam(lines))
    assert _xa_strings(recs, xa, cig, names) == tp.xa_of_lines(lines)
    # the batch held what the pairs asked for (the host emulation of the same split: 0 in place on C0)
    assert st["staged"] == mode and st["jobs"] > 50 and st["looked_up"] > 50 and st["looked_up"] <= st["jobs"], st
    assert st["in_place"] == 0 and st["window_moved"] == 0, st


@MODES
@pytest.mark.parametrize("flags", [0x8, 0x10, 0x4, 0x200, 0x1800], ids=["all", "no_multi", "no_pairing", "softclip", "primary5"])
def test_staged_equals_default_mode_with_flags(c0, flags, mode):
    capi, idx, reads, codes, offs, names = c0
    opt = capi.default_opt(); opt.flag |= 0x2 | flags
    a, st_a, _ = _run(capi, idx, opt, codes, offs, 0)
    b, st_b, _ = _run(capi, idx, opt, codes, offs, mode)
    assert st_a["staged"] == 0 and st_a["jobs"] == 0 and st_b["staged"] == mode and st_b["jobs"] > 0
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


def test_staged_no_rescue_flag_lists_nothing(c0):
    capi, idx, reads, codes, offs, names = c0
    opt = capi.default_opt(); opt.flag |= 0x2 | 0x20
    a, st_a, _ = _run(capi, idx, opt, codes, offs, 0)
    b, st_b, _ = _run(capi, idx, opt, codes, offs, 1)
    assert st_b["staged"] == 0 and st_b["jobs"] == 0
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


@MODES
def test_staged_tandem_repeat_pairs_match_oracle(pkg, golden_dir, mode):
    """Hundreds of regions per read, up to max_matesw anchors per read: long job lists per pair, windows that move after earlier rescues."""
    capi = pkg.capi
    idx = capi.Index(golden_dir + "/tandem_index/ref.fa")
    try:
        rd = np.load(golden_dir + "/tandem_reads.npz"); codes, offs = rd["codes"], rd["offs"]
        opt = capi.default_opt(); opt.flag |= 0x2
        pes = np.zeros(4, capi.PESTAT_DT)
        pes["failed"] = 1
        pes[1] = (100, 700, 0, 0, 400.0, 80.0)
        (recs, xa, cig, md), st, (regs, ro, _) = _run(capi, idx, opt, codes, offs, mode, pes=pes)
        lh = np.array([v for d in range(4) for v in (pes[d]["low"], pes[d]["high"], pes[d]["failed"])], np.int32)
        as_ = np.array([v for d in range(4) for v in (pes[d]["avg"], pes[d]["std"])], np.float64)
        want = tp.oracle_sam_pe(capi, idx, opt, codes, offs, regs, ro, lh, as_)
        names = ["tr1", "tr2"]
        tp._compare(tp.fields(recs, cig, md, names), tp.fields(*want, names))
        assert st["staged"] == mode
    finally:
        idx.close()

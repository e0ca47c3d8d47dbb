"""GPU parity of bm2_ksw_align2 (the local alignment of mate rescue, one window per warp: ksw.cu / ksw_warp.cuh) through the C ABI: the
golden vectors made by the UNMODIFIED reference's ksw_align2 (tests/golden/ksw_c0.npz) and the oracle on fresh requests with other
scoring.  ksw.cu was written after the round's GPU minutes were spent: non-strict xfail until it has run once (its arithmetic is
checked on the host, tests/test_oracle_ksw.py[warp_scan]).  Named to run after every other file (a fault in a kernel that has never run must not take later tests with it)."""
import numpy as np
import pytest
import ksw_util as ku
import test_oracle_ksw as tk

pytestmark = [pytest.mark.gpu]


def test_golden_vectors_of_the_reference(pkg, golden_dir):
    reqs, want = tk._golden(golden_dir)
    ctx = pkg.capi.Context(0)
    try:
        got = ctx.ksw_align2(reqs)
    finally:
        ctx.close()
    bad = np.nonzero((got != want).any(1))[0]
    assert len(bad) == 0, (bad[:5], got[bad[:5]], want[bad[:5]])


@pytest.mark.parametrize("seed,qlens,sc", [(31, (151, 100, 36, 17), {}), (32, (249, 250, 300, 497), {}),
                                           (33, (151, 76), dict(o_del=1, e_del=1, o_ins=1, e_ins=1, b=1)),
                                           (34, (120, 260), dict(o_del=4, e_del=2, o_ins=5, e_ins=1, a=2, b=3))])
def test_fresh_requests_against_oracle(pkg, seed, qlens, sc):
    o = pkg.capi.default_opt()
    for k, v in sc.items():
        setattr(o, k, v)
    k = 0
    for i in range(4):
        for j in range(4):
            o.mat[k] = o.a if i == j else -o.b; k += 1
        o.mat[k] = -1; k += 1
    reqs = ku.make_requests(np.random.default_rng(seed), 1500, qlens=qlens)
    reqs = [(q, t, ku.mate_xtra(len(q), a=o.a, min_seed_len=o.min_seed_len)) for q, t, _ in reqs]
    want = ku.oracle_ksw(reqs, o)
    ctx = pkg.capi.Context(0, opt=o)
    try:
        got = ctx.ksw_align2(reqs)
    finally:
        ctx.close()
    bad = np.nonzero((got != want).any(1))[0]
    assert len(bad) == 0, (bad[:5], got[bad[:5]], want[bad[:5]])

"""GPU parity on reads inside short tandem repeats (tests/golden/tandem_*, see tests/test_chain_tree_cpu.py): hundreds of chains per
read, chains with equal positions (the kernels keep the shape of the reference's chain B-tree, chain_tree_put_d), up to a thousand
alignment regions per read, 16-bit extension jobs of 251-bp reads.  Through the C ABI, against the UNMODIFIED reference's regs
(golden) and the oracle.  The same device logic is checked on the host by
tests/test_chain_tree_cpu.py."""
import numpy as np
import pytest
import oracle_lib as ol

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tandem(pkg, golden_dir):
    idx = pkg.capi.Index(golden_dir + "/tandem_index/ref.fa")
    rd = np.load(golden_dir + "/tandem_reads.npz"); gd = np.load(golden_dir + "/tandem_regs.npz")
    ctx = pkg.capi.Context(0, index=idx)
    yield idx, ctx, rd["codes"], rd["offs"], gd["regs"], gd["offs"]
    ctx.close(); idx.close()


def test_chains_match_oracle(pkg, tandem):
    idx, ctx, codes, offs, _, _ = tandem
    ch, sd, co = ctx.seed_chain(codes, offs)
    och, osd, oco = ol.seed_chain(idx, pkg.capi.default_opt(), codes, offs)
    assert np.array_equal(co, oco)
    for f in ("pos", "rid", "n_seeds", "w", "kept", "first", "frac_rep", "seed_off"):
        assert np.array_equal(ch[f], och[f]), f
    for f in ("rbeg", "qbeg", "len", "score"):
        assert np.array_equal(sd[f], osd[f]), f
    assert int(np.diff(co).max()) > 1000


def test_regs_match_reference_and_oracle(pkg, tandem):
    idx, ctx, codes, offs, gregs, goffs = tandem
    regs, ro = ctx.seed_chain_extend(codes, offs)
    assert ol.regs_equal_to_dump(regs, ro, gregs, goffs) == []
    oregs, oro, cells, rc = ol.seed_chain_extend(idx, pkg.capi.default_opt(), codes, offs)
    assert rc == 0 and np.array_equal(ro, oro) and regs.tobytes() == oregs.tobytes()

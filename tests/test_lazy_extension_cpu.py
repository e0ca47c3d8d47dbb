"""Lazy extension (BM2_EXT_LAZY, ext_walk_read_d in bwa-mem2_b200/csrc/ext_device.cuh): the extension runs in waves and the seeds
that the post-filter purges before any of them is extended are never extended.  The device logic compiled for the host, with the
kernels' waves (tests/host_emul/lazy_emul.cpp), must give the same regs, byte for byte, as the eager host emulation (which the other CPU
tests pin to the oracle and the reference) with laziness on and off, must actually skip jobs, and every reg the final post-filter keeps
must have been extended."""
import numpy as np
import pytest
import emul_lib as el
import lazy_emul_lib as ll
import longread_util as lu
import oracle_lib as ol
from test_option_surface_cpu import CASES, opt_from_cli


@pytest.fixture(scope="module")
def c0(pkg, golden_dir):
    idx = pkg.capi.Index(golden_dir + "/c0_index/ref.fa")
    reads = np.load(golden_dir + "/c0_reads.npz")["reads"]
    yield idx, reads.reshape(-1), (np.arange(len(reads) + 1) * reads.shape[1]).astype(np.int64)
    idx.close()


@pytest.fixture(scope="module")
def tandem(pkg, golden_dir):
    idx = pkg.capi.Index(golden_dir + "/tandem_index/ref.fa")
    rd = np.load(golden_dir + "/tandem_reads.npz")
    yield idx, rd["codes"], rd["offs"]
    idx.close()


def _check(monkeypatch, idx, opt, codes, offs, env=None, min_regs=1000):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    want, wo = el.seed_chain_extend(idx, opt, codes, offs)
    monkeypatch.setenv("BM2_EXT_LAZY", "0")
    eregs, eo, eager = ll.seed_chain_extend(idx, opt, codes, offs)
    monkeypatch.setenv("BM2_EXT_LAZY", "1")
    got, go, lazy = ll.seed_chain_extend(idx, opt, codes, offs)
    assert len(want) > min_regs
    assert np.array_equal(eo, wo) and eregs.tobytes() == want.tobytes()
    assert np.array_equal(go, wo) and got.tobytes() == want.tobytes()
    assert eager["skipped"] == 0 and eager["jobs"] == lazy["jobs"] and eager["kept_not_extended"] == 0
    assert lazy["skipped"] > 0 and lazy["kept_not_extended"] == 0
    print(f"{lazy['skipped']} of {lazy['jobs']} jobs skipped ({lazy['skipped'] / lazy['jobs']:.1%}), "
          f"{lazy['done_wave1']} reads decided after wave 1")
    return got, go


def test_c0_default(pkg, golden_dir, monkeypatch, c0):
    idx, codes, offs = c0
    got, go = _check(monkeypatch, idx, pkg.capi.default_opt(), codes, offs)
    st = np.load(golden_dir + "/c0_stages.npz")
    assert ol.regs_equal_to_dump(got, go, st["regs"], st["reg_off"]) == []       # the reference's own regs


@pytest.mark.parametrize("waves", ["3", "4", "8"])
def test_c0_more_waves(pkg, monkeypatch, c0, waves):
    idx, codes, offs = c0
    _check(monkeypatch, idx, pkg.capi.default_opt(), codes, offs, {"BM2_EXT_WAVES": waves})


@pytest.mark.parametrize("name,args", CASES, ids=[c[0] for c in CASES])
def test_c0_option_sets(pkg, monkeypatch, c0, name, args):
    idx, codes, offs = c0
    _check(monkeypatch, idx, opt_from_cli(pkg.capi, args), codes, offs)


@pytest.mark.parametrize("env", [{}, {"BM2_EXT_WALK_HEAVY": "1000000", "BM2_EXT_WAVES": "3"}], ids=["default", "all_walked"])
def test_tandem(pkg, monkeypatch, tandem, env):
    """Reads inside short tandem repeats: many regs per read; 'all_walked' walks the heavy reads too."""
    idx, codes, offs = tandem
    _check(monkeypatch, idx, pkg.capi.default_opt(), codes, offs, env)


def test_long_reads(pkg, monkeypatch):
    ds = lu.make_dataset(n3k=4, n8k=1, ref_bp=500_000)
    if ds is None:
        pytest.skip("oracle/_ref not built")
    prefix, codes, offs = ds
    idx = pkg.capi.Index(prefix)
    _check(monkeypatch, idx, lu.ont2d_opt(pkg.capi), codes, offs, min_regs=5)
    idx.close()

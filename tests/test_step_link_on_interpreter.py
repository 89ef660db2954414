"""The kernels of a tmd_md_steps step hand work to each other -- the fused prepare, the bonded sums folded into the
kernel after the force call, the bonded terms deferred into the second half-kick -- only inside that step.  So after a
tmd_md_steps call a standalone tmd_forces and tmd_vv_second launch the kernels they launch on a context that never ran
one, and tmd_forces leaves no bonded fold for tmd_vv_second to pick up.  On the host SIMT-interpreter build with the
product's defaults (tests/simt, tag "_cl": captured step graphs, fused prepare and step boundary, cluster lists)."""
import ctypes as C

import numpy as np
import pytest

import test_simt_kernels as T
from conftest import load_golden
from torchmd_b200._lib import PAIR_CLUSTER


@pytest.fixture(scope="module")
def simt_cl():
    return T.load(T.build_simt("_cl", T.VARIANTS["_cl"]))


def setup(L):
    from torchmd_b200 import _lib

    c = T.Ctx(L, load_golden("ala2_nobox_rf"))  # two replicas of a protein without a box: the cluster path
    c.posw = c.pos.copy()
    c.vel = np.random.default_rng(7).normal(scale=0.01, size=c.pos.shape).astype(np.float32)
    c.F, _ = c.forces(pos=c.posw)
    c.masses = np.ascontiguousarray(c.g["par_masses"].astype(np.float32))
    c.dt = 1.0 / T.TIMEFACTOR
    c.ene = np.zeros((c.nrep, _lib.NUM_ENERGIES))
    c.ke = np.zeros(c.nrep)
    return c


def launches(L, c):
    from torchmd_b200 import _lib

    st = _lib.Stats()
    L.tmd_get_stats(c.h, C.byref(st), None)  # (only the launch counter is read here)
    return st.kernel_launches


def standalone_calls(L, c, pos, vel, F0):
    """tmd_forces at pos, then tmd_vv_second of vel with the forces F0: the launches of each and the results."""
    F = np.zeros_like(pos)
    E = np.zeros_like(c.ene)
    ke = np.zeros_like(c.ke)
    l0 = launches(L, c)
    c.check(L.tmd_forces(c.h, pos.ctypes.data, F.ctypes.data, E.ctypes.data, None))
    l1 = launches(L, c)
    c.check(L.tmd_vv_second(c.h, vel.ctypes.data, F0.ctypes.data, c.masses.ctypes.data, c.dt, -1.0, None, None, 1, 0,
                            ke.ctypes.data, None))
    return (l1 - l0, launches(L, c) - l1), F, E, vel, ke


@pytest.mark.parametrize("graph", ["1", "0"], ids=["captured", "stream"])
@pytest.mark.parametrize("overlap", ["1", "0"], ids=["fold", "deferred"])
def test_standalone_calls_after_md_steps_are_those_of_a_fresh_context(simt_cl, monkeypatch, overlap, graph):
    # TMD_B200_OVERLAP=1: the bonded kernels run on the side stream, and the step boundary or the second half-kick adds
    # their sums; =0: the second half-kick evaluates the bonded terms itself (k_bonded_vv_second)
    monkeypatch.setenv("TMD_B200_OVERLAP", overlap)
    monkeypatch.setenv("TMD_B200_GRAPH", graph)
    ran, fresh = setup(simt_cl), setup(simt_cl)
    T.md_steps(simt_cl, ran, 3)
    assert simt_cl.tmd_pair_kernel(ran.h) == PAIR_CLUSTER
    pos, vel, F0 = ran.posw.copy(), ran.vel.copy(), ran.F.copy()
    got = standalone_calls(simt_cl, ran, pos, vel.copy(), F0)
    want = standalone_calls(simt_cl, fresh, pos, vel.copy(), F0)
    assert got[0] == want[0]
    # the forces carry the bonded terms and are in atom order, as on the fresh context (whose lists were built at other
    # positions: the pair sums may differ in their last bits)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-6, atol=1e-4)
    # the plain second half-kick: nothing is added to the forces it was given
    assert np.array_equal(got[3], want[3]) and np.array_equal(got[4], want[4])
    assert not np.array_equal(got[3], vel)
    ran.close()
    fresh.close()

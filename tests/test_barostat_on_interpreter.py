"""The Monte Carlo barostat on the CPU: the molecule move (k_scale_molecules) and the box rescale (tmd_rescale_box) on
the host SIMT-interpreter build of the library (tests/simt), k_pme_influence against the host formula, and the
acceptance rule, the dV_max adaptation and the refusals as host code."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_mirrors_on_interpreter import _install, hostsim  # noqa: F401
from test_simt_kernels import CSRC, SIMT_DIR


def _params(natoms, bonds, charges=None, sigma=3.0, eps=0.1):
    from torchmd_b200.parameters import TopologyParameters

    kw = {}
    if bonds is not None and len(bonds):
        b = np.asarray(bonds, np.int64)
        kw["bonds"] = (b, np.stack([np.arange(len(b)), np.zeros(len(b), np.int64)], 1), np.array([[100.0, 1.5]]))
    q = np.zeros(natoms) if charges is None else charges
    return lambda precision: TopologyParameters(atom_types=np.zeros(natoms, np.int64), type_sigma=[sigma], type_epsilon=[eps],
                                                charges=q, masses=np.full(natoms, 12.0), precision=precision, **kw)


def _finalised(make, pos, L, dtype, cutoff=3.0):
    """A Forces context finalised on positions pos (R,N,3) in boxes L (R,3) (CPU tensors: the interpreter's memory)."""
    from torchmd_b200 import Forces

    f = Forces(make(dtype), terms=["lj"], cutoff=cutoff)
    p = torch.tensor(pos, dtype=dtype)
    box = torch.diag_embed(torch.tensor(L, dtype=dtype))
    f.compute(p, box, torch.zeros_like(p))
    return f


def _graph_system(rng, L):
    """Molecules of every kind the move must get right, as (natoms, bonds, positions (N,3)):
    random trees with extra ring bonds, waters split across the box, a chain longer than half the box, atoms several
    boxes away, and lone atoms."""
    atoms, bonds, xyz = 0, [], []

    def add(coords, edges):
        nonlocal atoms
        xyz.extend(coords)
        bonds.extend([(atoms + i, atoms + j) for i, j in edges])
        atoms += len(coords)

    for _ in range(6):  # random bond graphs: a random tree plus a few ring closures, atoms scattered anywhere
        n = int(rng.integers(2, 9))
        edges = [(int(rng.integers(0, k)), k) for k in range(1, n)]
        edges += [(0, n - 1)] if n > 3 else []
        c = rng.uniform(0, L)
        pts = [c]
        for k in range(1, n):
            pts.append(pts[edges[k - 1][0]] + rng.normal(0, 1.0, 3))
        pts = np.array(pts) + L * rng.integers(-3, 4, (n, 1))  # every atom in its own image, up to 3 boxes away
        add(list(pts), edges)
    for _ in range(4):  # waters split across a face of the box
        o = np.array([L[0] - 0.3, rng.uniform(0, L[1]), rng.uniform(0, L[2])])
        h1 = o + [0.9, 0.2, 0.0]
        h2 = o + [-0.3, 0.9, 0.0]
        h1[0] -= L[0]  # wrapped to the other side
        add([o, h1, h2], [(0, 1), (0, 2)])
    n = int(0.8 * L[0] / 1.2)  # a chain longer than half the box, wrapped atom by atom
    chain = np.array([[1.2 * k, 0.5 * math.sin(k), 0.3 * k] for k in range(n)]) + rng.uniform(0, L)
    add(list(chain - L * np.floor(chain / L)), [(k, k + 1) for k in range(n - 1)])
    for _ in range(5):  # lone atoms, some far away
        add([rng.uniform(0, L) + L * rng.integers(-5, 6, 3)], [])
    return atoms, np.array(bonds, np.int64), np.array(xyz)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_molecule_move_matches_the_oracle(hostsim, dtype):  # noqa: F811
    from oracle import barostat as ob
    from torchmd_b200 import _lib
    from torchmd_b200.barostat import molecule_trees

    rng = np.random.default_rng(11)
    L0 = np.array([21.0, 23.0, 25.0])
    natoms, bonds, xyz = _graph_system(rng, L0)
    make = _params(natoms, bonds)
    Ls = np.stack([L0, L0 * 1.1])
    pos = np.stack([xyz, xyz * 1.1 + 0.37])  # replica 1: other coordinates in its own box
    f = _finalised(make, pos, Ls, dtype)
    ptr, atoms, parent = molecule_trees(natoms, bonds)
    L = _lib.lib()
    _lib.check(L.tmd_set_molecules(f._ctx, len(ptr) - 1, ptr.ctypes.data, atoms.ctypes.data, parent.ctypes.data))
    s = np.array([[1.013] * 3, [0.987] * 3])
    p = torch.tensor(pos, dtype=dtype)
    x0 = p.double().numpy().copy()
    scale = torch.tensor(s, dtype=torch.float64)
    sfx = "_f64" if dtype == torch.float64 else ""
    _lib.check(getattr(L, "tmd_scale_molecules" + sfx)(f._ctx, p.data_ptr(), scale.data_ptr(), None))
    want = ob.scale_molecules(x0, Ls.astype(np.dtype(str(dtype).split(".")[1])).astype(np.float64), s, ptr, atoms, parent)
    npd = np.float64 if dtype == torch.float64 else np.float32
    want_r = want.astype(npd)
    got = p.numpy()
    assert np.all(np.abs(got.astype(np.float64) - want_r.astype(np.float64)) <= np.spacing(np.abs(want_r)).astype(np.float64)), \
        np.abs(got - want_r).max()
    # intra-molecular minimum-image vectors in the scaled box equal those before, to the coordinates' rounding
    Lw = Ls.astype(npd).astype(np.float64)
    for r in range(2):
        for i, j in bonds:
            d0 = ob.image(x0[r, j] - x0[r, i], Lw[r])
            d1 = ob.image(got[r, j].astype(np.float64) - got[r, i].astype(np.float64), Lw[r] * s[r])
            tol = 4 * np.spacing(np.abs(got[r, [i, j]]).max().astype(npd)).astype(np.float64)
            assert np.all(np.abs(d1 - d0) <= tol), (r, i, j, d0, d1)


def test_molecule_move_under_a_random_thread_order():
    env = dict(os.environ, SIMT_SCHEDULE="random:5")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", __file__, "-k", "matches_the_oracle"],
                       cwd=os.path.dirname(os.path.abspath(__file__)), env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_acceptance_rule_and_adaptation():
    from torchmd_b200.barostat import BAR_TO_KCAL_PER_MOL_A3, accept, acceptance_work, adapt_dv_max

    assert abs(BAR_TO_KCAL_PER_MOL_A3 - 1.43933e-5) < 1e-10
    kT = 0.6
    # w = dE + P dV - N kT ln(V'/V): 1 + 1e5 bar * 1.4393262e-5 * 10 - 2 * 0.6 * ln(1010/1000)
    w = acceptance_work(1.0, 10.0, 1000.0, 1e5, 2, kT)
    assert abs(w - (1.0 + 14.393262 - 1.2 * math.log(1.01))) < 1e-6
    assert accept(-0.5, kT, 0.999999)  # downhill: always
    assert accept(0.6, kT, math.exp(-1.0) - 1e-12) and not accept(0.6, kT, math.exp(-1.0) + 1e-12)
    assert not accept(-1.0, kT, math.inf)  # u = inf rejects any move
    assert adapt_dv_max(100.0, 10, 2, 1e4) == pytest.approx(90.0)
    assert adapt_dv_max(100.0, 10, 8, 1e4) == pytest.approx(110.0)
    assert adapt_dv_max(100.0, 10, 5, 1e4) == 100.0
    assert adapt_dv_max(2900.0, 10, 10, 1e4) == pytest.approx(3000.0)  # capped at 0.3 V


def test_molecule_trees():
    from torchmd_b200.barostat import molecule_trees

    ptr, atoms, parent = molecule_trees(7, np.array([[0, 2], [2, 4], [4, 0], [5, 6]]))
    assert ptr.tolist() == [0, 3, 5, 6, 7]
    assert atoms.tolist() == [0, 2, 4, 5, 6, 1, 3]
    assert parent.tolist() == [0, 0, 0, 5, 5, 1, 3]


@pytest.fixture(scope="module")
def infl_lib():
    src = os.path.join(SIMT_DIR, "pme_influence.cpp")
    out = os.path.join(SIMT_DIR, "libpme_influence.so")
    deps = [src, os.path.join(CSRC, "pme.cuh"), os.path.join(SIMT_DIR, "simt.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        cmd = ["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-U_FORTIFY_SOURCE", "-I",
               os.path.join(SIMT_DIR, "stub"), "-I", CSRC, "-o", out + ".tmp", src]
        subprocess.run(cmd, check=True)
        os.replace(out + ".tmp", out)
    h = C.CDLL(out)
    h.simt_pme_influence.restype = C.c_int
    h.simt_pme_influence.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p]
    return h


def _host_influence(L, alpha, K, mods):
    """The host triple loop k_pme_influence replaced, operation for operation."""
    V = L[0] * L[1] * L[2]
    G = np.zeros(K)
    for x in range(K[0]):
        mx = (x - K[0] if x > K[0] // 2 else x) / L[0]
        for y in range(K[1]):
            my = (y - K[1] if y > K[1] // 2 else y) / L[1]
            for z in range(K[2]):
                mz = (z - K[2] if z > K[2] // 2 else z) / L[2]
                m2 = mx * mx + my * my + mz * mz
                if m2 > 0.0:
                    G[x, y, z] = math.exp(-math.pi * math.pi * m2 / (alpha * alpha)) / (math.pi * V * m2 * mods[0][x] * mods[1][y] * mods[2][z])
    return G


@pytest.mark.parametrize("bits", [64, 32])
def test_pme_influence_kernel_against_the_host_formula(infl_lib, bits):
    from oracle.pme import bspline_moduli

    K = np.array([10, 12, 15], np.int32)
    L = np.array([[20.0, 22.5, 27.1], [20.2, 22.7, 27.3]])
    alpha = 0.35
    mods = [bspline_moduli(int(k)) for k in K]
    flat = np.ascontiguousarray(np.concatenate(mods))
    G = np.zeros((2,) + tuple(K))
    assert infl_lib.simt_pme_influence(2, K.ctypes.data, L.ctypes.data, alpha, flat.ctypes.data, bits, G.ctypes.data) == 0
    for r in range(2):
        want = _host_influence(L[r], alpha, tuple(K), mods)
        if bits == 32:
            want = want.astype(np.float32).astype(np.float64)
            ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        else:
            ulp = np.spacing(np.abs(want))
        assert np.all(np.abs(G[r] - want) <= 2 * ulp), np.max(np.abs(G[r] - want) / np.maximum(ulp, 1e-300))


def _water(nw, dtype, L_scale=1.0, seed=0):
    from torchmd_b200 import testsystems

    sysd = testsystems.water_box(nw, seed=seed)
    par = testsystems.water_parameters(sysd, precision=dtype)
    return sysd, par


def _rescale(f, box, new_diag):
    """tmd_rescale_box on the Forces context, and the box tensor written in place with the Forces key moved along."""
    from torchmd_b200 import _lib

    f64 = box.dtype == torch.float64
    host = np.ascontiguousarray(new_diag, dtype=np.float64 if f64 else np.float32)
    rc = (_lib.lib().tmd_rescale_box_f64 if f64 else _lib.lib().tmd_rescale_box)(f._ctx, host.ctypes.data, None)
    if rc == 0:
        idx = torch.arange(3)
        box[:, idx, idx] = torch.as_tensor(host)
        f._box_key = (box.data_ptr(), box._version, tuple(box.shape), tuple(box.stride()), box.dtype)
        f._box_ref = box
    return rc


def _fast_vs_fresh(dtype, nw, cutoff, pme, s, constraints=False):
    """Energies and forces after a fast rescale against a context finalised at the scaled box."""
    from torchmd_b200 import Forces
    from torchmd_b200.barostat import molecule_trees
    from torchmd_b200 import _lib

    sysd, par = _water(nw, dtype)
    terms = ["lj", "electrostatics", "bonds", "angles"]
    cfg = dict(cutoff=cutoff, switch_dist=cutoff - 1.0, pme=pme, rfa=not pme)
    f = Forces(par, terms=terms, **cfg)
    pos = torch.tensor(np.asarray(sysd["coords"])[None], dtype=dtype).contiguous()
    L0 = np.asarray(sysd["box"], np.float64).reshape(1, 3)
    box = torch.diag_embed(torch.tensor(L0, dtype=dtype))
    F = torch.zeros_like(pos)
    f.compute(pos, box, F)
    natoms = pos.shape[1]
    ptr, atoms, parent = molecule_trees(natoms, par.bond_params["idx"].numpy())
    L = _lib.lib()
    _lib.check(L.tmd_set_molecules(f._ctx, len(ptr) - 1, ptr.ctypes.data, atoms.ctypes.data, parent.ctypes.data))
    new = (L0 * s).astype(np.float64 if dtype == torch.float64 else np.float32).astype(np.float64)
    scale = torch.tensor(new / L0, dtype=torch.float64)
    sfx = "_f64" if dtype == torch.float64 else ""
    _lib.check(getattr(L, "tmd_scale_molecules" + sfx)(f._ctx, pos.data_ptr(), scale.data_ptr(), None))
    assert _rescale(f, box, new) == 0
    E1 = f.compute(pos, box, F, returnDetails=True)[0]
    g = Forces(par, terms=terms, **cfg)
    F2 = torch.zeros_like(pos)
    E2 = g.compute(pos, box.clone(), F2, returnDetails=True)[0]
    if pme:
        assert f.pme_parameters()[1] == g.pme_parameters()[1]
    return E1, E2, F, F2


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("pme", [True, False])
def test_rescale_equals_a_fresh_context_full_rows(hostsim, dtype, pme):  # noqa: F811
    E1, E2, F1, F2 = _fast_vs_fresh(dtype, 100, 5.0, pme, 1.004)
    rel = 1e-12 if dtype == torch.float64 else 2e-6
    for k in E1:
        assert abs(E1[k] - E2[k]) <= rel * max(1.0, abs(E2[k])), (k, E1[k], E2[k])
    fa = 1e-9 if dtype == torch.float64 else 5e-4
    assert (F1.double() - F2.double()).abs().max().item() <= fa


def test_rescale_equals_a_fresh_context_cluster_path(monkeypatch):
    handle = _install(monkeypatch, "_cl")
    from torchmd_b200 import _lib

    monkeypatch.setenv("TMD_B200_CLUSTER", "1")
    for pme in (True, False):
        E1, E2, F1, F2 = _fast_vs_fresh(torch.float32, 1200, 5.0, pme, 0.997)
        for k in E1:
            assert abs(E1[k] - E2[k]) <= 2e-6 * max(1.0, abs(E2[k])), (k, E1[k], E2[k])
        assert (F1 - F2).abs().max().item() <= 5e-4
    assert handle is _lib.lib()


def test_rescale_refusals_change_nothing(hostsim):  # noqa: F811
    from torchmd_b200 import Forces
    from torchmd_b200 import _lib

    sysd, par = _water(100, torch.float64)
    f = Forces(par, terms=["lj", "electrostatics"], cutoff=5.0, pme=True)
    pos = torch.tensor(np.asarray(sysd["coords"])[None], dtype=torch.float64).contiguous()
    L0 = np.asarray(sysd["box"], np.float64).reshape(1, 3)
    box = torch.diag_embed(torch.tensor(L0))
    F = torch.zeros_like(pos)
    E0 = f.compute(pos, box, F)[0]
    L = _lib.lib()
    for bad in (L0 * 0.1, L0 * [[1.0, 1.0, 0.2]]):  # PME's cutoff <= L/2, and the cell grid below 2 nsub + 1
        h = np.ascontiguousarray(bad)
        assert L.tmd_rescale_box_f64(f._ctx, h.ctypes.data, None) == _lib.ERR_UNSUPPORTED
    big = np.ascontiguousarray(L0 * 300.0)
    assert L.tmd_rescale_box_f64(f._ctx, big.ctypes.data, None) == _lib.ERR_UNSUPPORTED  # fp64 limit
    assert L.tmd_rescale_box(f._ctx, np.ascontiguousarray(L0, np.float32).ctypes.data, None) != 0  # precision
    assert f.compute(pos, box, F)[0] == E0  # nothing changed
    _lib.check(L.tmd_set_force_convention(f._ctx, 1))  # a setter: no rescale until finalised again
    _lib.check(L.tmd_set_force_convention(f._ctx, 0))


def test_refusals(hostsim):  # noqa: F811
    from torchmd_b200 import Forces, Integrator, MonteCarloBarostat, System
    from torchmd_b200.domain import DecomposedIntegrator

    for kw in (dict(pressure=0.0), dict(pressure=-1.0), dict(temperature=0.0), dict(frequency=0)):
        with pytest.raises(ValueError):
            MonteCarloBarostat(**kw)
    sysd, par = _water(20, torch.float32)
    n = len(sysd["coords"])
    system = System(n, 1, torch.float32, "cpu")
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    f = Forces(par, terms=["lj"], cutoff=3.0)
    with pytest.raises(RuntimeError, match="thermostat"):
        Integrator(system, f, 1.0, "cpu", barostat=MonteCarloBarostat())

    class Ext:
        def calculate(self, pos, box):
            return torch.zeros(1), torch.zeros_like(pos)

    with pytest.raises(RuntimeError, match="native"):
        Integrator(system, Forces(par, terms=["lj"], cutoff=3.0, external=Ext()), 1.0, "cpu", gamma=1.0, T=300.0,
                   barostat=MonteCarloBarostat())
    open_sys = System(n, 1, torch.float32, "cpu")
    open_sys.set_positions(sysd["coords"])
    with pytest.raises(RuntimeError, match="periodic"):
        Integrator(open_sys, f, 1.0, "cpu", gamma=1.0, T=300.0, barostat=MonteCarloBarostat())
    with pytest.raises(NotImplementedError, match="barostat"):
        DecomposedIntegrator(system, f, 1.0, "cpu", gamma=1.0, T=300.0, barostat=MonteCarloBarostat())


def test_npt_steps_on_the_interpreter(hostsim):  # noqa: F811
    """A few moves through Integrator.step: chunks end where a move is due, the box lands in systems.box, the stats
    count every attempt, and the returned energy is the state's."""
    from torchmd_b200 import Forces, Integrator, MonteCarloBarostat, System, maxwell_boltzmann

    torch.manual_seed(0)
    sysd, par = _water(100, torch.float64)
    n = len(sysd["coords"])
    system = System(n, 1, torch.float64, "cpu")
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    f = Forces(par, terms=["lj", "electrostatics", "bonds", "angles"], cutoff=5.0, pme=True)
    bar = MonteCarloBarostat(pressure=1.0, frequency=3)
    integ = Integrator(system, f, 1.0, "cpu", gamma=1.0, T=300.0, barostat=bar)
    box0 = system.box.clone()
    _, pot, _ = integ.step(7)  # moves after steps 3 and 6
    st = bar.stats()[0]
    assert st["attempted"] == 2 and st["fast_box_changes"] + st["full_box_changes"] >= 2
    _, pot2, _ = integ.step(2)  # step 9: a move closes the call
    assert bar.stats()[0]["attempted"] == 3
    e = f.compute(system.pos, system.box, torch.zeros_like(system.pos))[0]
    assert abs(e - pot2[0]) <= 1e-9 * max(1.0, abs(e))
    if bar.stats()[0]["accepted"]:
        assert not torch.equal(system.box, box0)

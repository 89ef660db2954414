"""Generalized Born implicit solvent (OBC2, Forces(..., implicit_solvent="obc2")) on the GPU: the GB part of the
energies and forces against the fp64 oracle (oracle/gbsa.py) on ligand, benzamidine and thrombin, bitwise
reproducibility, the autograd path, the captured MD step with and without constraints, replica exchange, energy
conservation, and every refusal.  tests/test_gbsa_on_interpreter.py runs the small cases on the CPU interpreter."""
import numpy as np
import pytest
import torch

from conftest import load_golden, params_from_golden
from oracle import gbsa

DEV = "cuda"
F32, F64 = torch.float32, torch.float64
TERMS = ["bonds", "angles", "dihedrals", "impropers", "1-4", "lj", "electrostatics"]
EPS = 78.5


def _golden(name):
    return load_golden("thrombin_nobox_rf" if name == "thrombin" else name + "_amber_nocut")


def _params(name, dtype):
    g, gb = _golden(name), load_golden("gb_radii")
    par = params_from_golden(g, precision=dtype, device=DEV)
    par.gb_params = {"radius": torch.tensor(gb[name + "_radii"]), "screen": torch.tensor(gb[name + "_screen"])}
    return g, par


def _positions(g, dtype, nrep=2, seed=5):
    """Replica 0: the fixture's coordinates; every other replica deformed by N(0, 0.05 A)."""
    x = np.asarray(g["coords"], np.float64)
    rng = np.random.default_rng(seed)
    pos = np.stack([x] + [x + rng.normal(0.0, 0.05, x.shape) for _ in range(nrep - 1)])
    return torch.tensor(pos, dtype=dtype, device=DEV).contiguous(), torch.zeros(nrep, 3, 3, dtype=dtype, device=DEV)


def _forces(par, gb=True, sigma=0.0, **kw):
    from torchmd_b200 import Forces

    if gb:
        kw.update(implicit_solvent="obc2", surface_tension=sigma)
    return Forces(par, terms=TERMS, cutoff=None, rfa=False, solventDielectric=EPS, **kw)


def _gb_part(name, dtype, sigma, nrep=2):
    """(positions, GB energies (R,), GB forces (R,N,3)) as the kernels give them: with GB minus without."""
    g, par = _params(name, dtype)
    pos, box = _positions(g, dtype, nrep)
    out = []
    for gb in (True, False):
        fr = _forces(par, gb, sigma)
        F = torch.empty_like(pos)
        E = fr.compute(pos, box, F, returnDetails=True)
        out.append((np.array([e["electrostatics"] for e in E]), F.double().cpu().numpy()))
    return pos, g, out[0][0] - out[1][0], out[0][1] - out[1][1]


def _magnitude(pos, charges, radius, screen, Enp):
    """1/2 k (1 - 1/eps) sum_ij |qi qj| / f_ij + E_np: the scale of the GB energy's rounding error."""
    B, _, _ = gbsa.born_radii(pos, radius, screen)
    q = np.abs(np.asarray(charges, np.float64))
    r2 = ((pos[:, None, :] - pos[None, :, :]) ** 2).sum(-1)
    D = B[:, None] * B[None, :]
    f = np.sqrt(r2 + D * np.exp(-r2 / (4 * D)))
    return 0.5 * gbsa.COULOMB * (1 - 1 / EPS) * (q[:, None] * q[None, :] / f).sum() + Enp


@pytest.mark.gpu
@pytest.mark.parametrize("sigma", [0.0, 0.0054])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", ["ligand", "benzamidine", "thrombin"])
def test_against_the_oracle(name, dtype, sigma):
    pos, g, dE, dF = _gb_part(name, dtype, sigma)
    gb = load_golden("gb_radii")
    for r in range(pos.shape[0]):
        E, Enp, F = gbsa.energy_forces(pos[r].double().cpu().numpy(), g["par_charges"], gb[name + "_radii"], gb[name + "_screen"],
                                       EPS, sigma)
        want = E + Enp
        # relative to the magnitudes summed: a neutral molecule's polar energy is a small difference of large pair terms
        err_e = abs(dE[r] - want) / _magnitude(pos[r].double().cpu().numpy(), g["par_charges"], gb[name + "_radii"],
                                               gb[name + "_screen"], Enp)
        err_f = np.abs(dF[r] - F).max()
        if dtype == F64:
            assert err_e <= 1e-10, (r, dE[r], want)
            assert err_f <= 1e-9 * np.abs(F).max(), (r, err_f, np.abs(F).max())
        else:
            assert err_e <= 1e-6, (r, dE[r], want)
            assert err_f <= 5e-4, (r, err_f)
        print(f"[gbsa] {name} {dtype} sigma={sigma} replica {r}: E {want:.6f} rel dE {err_e:.2e} max|dF| {err_f:.2e} "
              f"max|F| {np.abs(F).max():.2f}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_gb_forces_are_bitwise_reproducible(dtype, name="thrombin"):
    g, par = _params(name, dtype)
    pos, box = _positions(g, dtype)
    fr = _forces(par, True, 0.0054)
    F1, F2 = torch.empty_like(pos), torch.empty_like(pos)
    fr.compute(pos, box, F1)
    fr.compute(pos, box, F2)
    assert torch.equal(F1, F2)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_autograd_and_vmap(dtype, name="ligand"):
    g, par = _params(name, dtype)
    pos, box = _positions(g, dtype)
    fr = _forces(par, True, 0.0054)
    F = torch.empty_like(pos)
    fr.compute(pos, box, F)
    p = pos.clone().requires_grad_(True)
    Fa = torch.empty_like(pos)
    E = fr.compute(p, box, Fa, explicit_forces=False, toNumpy=False)
    E.sum().backward()
    tol = 1e-12 if dtype == F64 else 1e-5
    scale = F.abs().max().item()
    assert (p.grad + F).abs().max().item() <= tol * scale
    assert (Fa - F).abs().max().item() <= tol * scale
    Ev = torch.vmap(lambda x: fr.compute(x, box, None, toNumpy=False, calculateForces=False))(pos[None])
    assert torch.allclose(Ev[0], E.detach(), rtol=1e-12 if dtype == F64 else 1e-6)


def _integrator(name, dtype, nrep=2, constraints=None, T=300.0, gamma=1.0, rex=None, dt=1.0):
    from torchmd_b200 import Constraints, Integrator, System, maxwell_boltzmann

    g, par = _params(name, dtype)
    pos, box = _positions(g, dtype, nrep)
    system = System(pos.shape[1], nrep, dtype, DEV)
    system.pos[:] = pos
    system.box[:] = box
    torch.manual_seed(4)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, nrep))
    fr = _forces(par, True, 0.0054)
    fr.compute(system.pos, system.box, system.forces)
    con = Constraints(par, constraints) if constraints else None
    integ = Integrator(system, fr, dt, DEV, gamma=gamma, T=T, constraints=con, replica_exchange=rex)
    return system, fr, integ


@pytest.mark.gpu
@pytest.mark.parametrize("constraints", [None, "hbonds"])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_native_steps_report_a_fresh_energy(dtype, constraints, name="thrombin", nsteps=20):
    system, fr, integ = _integrator(name, dtype, constraints=constraints, dt=2.0 if constraints else 1.0)
    for _ in range(2):
        _, pot, _ = integ.step(nsteps)
        fresh = fr.compute(system.pos.clone(), system.box, torch.empty_like(system.pos))
        tol = 1e-9 if dtype == F64 else 2e-6
        for r in range(len(pot)):
            assert abs(pot[r] - fresh[r]) <= tol * abs(fresh[r]), (r, pot[r], fresh[r])
    assert np.isfinite(system.pos.cpu().numpy()).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F64, F32], ids=["fp64", "fp32"])
def test_replica_exchange_exchanges_on_the_gb_energy(dtype, name="ligand"):
    from torchmd_b200 import ReplicaExchange

    rex = ReplicaExchange(frequency=5, seed=11)
    seen = []
    inner = rex.attempt

    def attempt(ctx, energies, stride, nterms):
        seen.append(energies.cpu().numpy().copy())
        inner(ctx, energies, stride, nterms)

    rex.attempt = attempt
    system, fr, integ = _integrator(name, dtype, nrep=4, T=[300.0, 330.0, 363.0, 400.0], gamma=5.0, rex=rex)
    integ.step(20)
    assert len(seen) == 4 and rex.attempts == 4
    # the last attempt saw the potential energies of the state the step returned, GB included
    fresh = fr.compute(system.pos.clone(), system.box, torch.empty_like(system.pos))
    vacuum = _forces(fr.par, False).compute(system.pos.clone(), system.box, torch.empty_like(system.pos))
    got = seen[-1].reshape(4, -1).sum(1)
    tol = 1e-9 if dtype == F64 else 2e-6
    for r in range(4):
        assert abs(got[r] - fresh[r]) <= tol * abs(fresh[r]), (r, got[r], fresh[r])
        assert abs(got[r] - vacuum[r]) > 1e3 * tol * abs(fresh[r]), (r, got[r], vacuum[r])  # (GB resolved)


@pytest.mark.gpu
def test_energy_conservation_nve_fp64(name="ligand", nsteps=20000):
    system, fr, integ = _integrator(name, F64, nrep=1, T=None, gamma=None, dt=0.5)
    ek, et = [], []
    for _ in range(nsteps // 100):
        k, p, _ = integ.step(100)
        ek.append(k[0])
        et.append(k[0] + p[0])
    ek, et = np.array(ek), np.array(et)
    print(f"[gbsa] NVE ligand 0.5 fs x {nsteps}: std(E_tot) {et.std():.3e} std(E_kin) {ek.std():.3e}")
    assert et.std() <= 0.01 * ek.std(), (et.std(), ek.std())


@pytest.mark.gpu
def test_minimizer_and_external_plugin(dtype=F32, name="ligand"):
    from torchmd_b200 import System
    from torchmd_b200.minimizers import minimize_cg, minimize_pytorch_bfgs

    g, par = _params(name, dtype)
    pos, box = _positions(g, dtype, 1)

    class Spring:  # a harmonic pull on atom 0, to check the plugin's energy and force are added
        def calculate(self, pos, box):
            e = 0.5 * (pos[:, 0] ** 2).sum(-1)
            f = torch.zeros_like(pos)
            f[:, 0] = -pos[:, 0]
            return e, f

    fr = _forces(par, True, 0.0054)
    fe = _forces(par, True, 0.0054, external=Spring())
    F, Fe = torch.empty_like(pos), torch.empty_like(pos)
    e0, e1 = fr.compute(pos, box, F)[0], fe.compute(pos, box, Fe)[0]
    assert abs(e1 - e0 - 0.5 * float((pos[0, 0].double() ** 2).sum())) <= 1e-3
    assert torch.allclose(Fe[0, 0] - F[0, 0], -pos[0, 0], atol=1e-3)
    for minimize in (minimize_cg, minimize_pytorch_bfgs):
        system = System(pos.shape[1], 1, dtype, DEV)
        system.pos[:] = pos
        system.box[:] = box
        before = fr.compute(system.pos, system.box, system.forces)[0]
        if minimize is minimize_cg:
            minimize(system, fr, steps=5, update_system=True)
        else:
            minimize(system, fr, steps=5)
        after = fr.compute(system.pos, system.box, system.forces)[0]
        assert np.isfinite(after) and after < before, (minimize.__name__, before, after)


@pytest.mark.gpu
def test_refusals(name="benzamidine"):
    from torchmd_b200 import Forces, Integrator, MonteCarloBarostat, System, _lib
    from torchmd_b200.domain import DecomposedIntegrator

    g, par = _params(name, F32)
    pos, box = _positions(g, F32, 1)
    for kw in (dict(cutoff=9.0), dict(cutoff=9.0, rfa=True), dict(cutoff=9.0, pme=True)):
        with pytest.raises(RuntimeError):
            Forces(par, terms=TERMS, implicit_solvent="obc2", **kw)
    with pytest.raises(RuntimeError, match="electrostatics"):
        Forces(par, terms=["bonds", "lj"], implicit_solvent="obc2")
    with pytest.raises(ValueError):
        Forces(par, terms=TERMS, implicit_solvent="hct")
    good = dict(par.gb_params)
    n = len(good["radius"])
    for bad in ({"radius": good["radius"].clone().fill_(0.09), "screen": good["screen"]},
                {"radius": good["radius"], "screen": -good["screen"]},
                {"radius": good["radius"].clone().fill_(float("nan")), "screen": good["screen"]},
                {"radius": good["radius"][:-1], "screen": good["screen"][:-1]}, None):
        par.gb_params = bad
        with pytest.raises(RuntimeError, match="gb_params"):
            _forces(par)
    par.gb_params = good
    fr = _forces(par)
    with pytest.raises(RuntimeError, match="box"):
        fr.compute(pos, torch.eye(3, device=DEV)[None] * 30.0, torch.empty_like(pos))
    # the library refuses the same configurations on its own
    L = _lib.lib()
    import ctypes as C

    def ctx():
        h = C.c_void_p()
        _lib.check(L.tmd_create(C.byref(h), 0, n, 1))
        return h

    radius = np.ascontiguousarray(good["radius"].cpu().numpy())
    screen = np.ascontiguousarray(good["screen"].cpu().numpy())
    h = ctx()
    try:
        _lib.check(L.tmd_set_nonbonded(h, 1 << 5, 9.0, -1.0, 0, EPS, 332.0, 1.0))
        assert L.tmd_set_gb(h, n, _lib.ptr(radius), _lib.ptr(screen), EPS, 0.0) == _lib.ERR_UNSUPPORTED
        _lib.check(L.tmd_set_nonbonded(h, 1 << 6, -1.0, -1.0, 0, EPS, 332.0, 1.0))
        assert L.tmd_set_gb(h, n, _lib.ptr(radius), _lib.ptr(screen), EPS, 0.0) == _lib.ERR_UNSUPPORTED
        _lib.check(L.tmd_set_nonbonded(h, 1 << 5, -1.0, -1.0, 0, EPS, 332.0, 1.0))
        assert L.tmd_set_gb(h, n - 1, _lib.ptr(radius), _lib.ptr(screen), EPS, 0.0) == -1
        small = radius.copy()
        small[3] = 0.05
        assert L.tmd_set_gb(h, n, _lib.ptr(small), _lib.ptr(screen), EPS, 0.0) == -1
        neg = -screen
        assert L.tmd_set_gb(h, n, _lib.ptr(radius), _lib.ptr(neg), EPS, 0.0) == -1
        inf = radius.copy()
        inf[0] = np.inf
        assert L.tmd_set_gb(h, n, _lib.ptr(inf), _lib.ptr(screen), EPS, 0.0) == -1
        _lib.check(L.tmd_set_gb(h, n, _lib.ptr(radius), _lib.ptr(screen), EPS, 0.0))
        assert L.tmd_set_owned_atoms(h, 0, n // 2) == _lib.ERR_UNSUPPORTED
        assert L.tmd_dd_create(h, 0, 1, (C.c_ubyte * 64)()) == _lib.ERR_UNSUPPORTED
        assert L.tmd_dd_connect(h, (C.c_ubyte * 64)()) == _lib.ERR_UNSUPPORTED
        assert L.tmd_set_pme(h, 5e-4) == _lib.ERR_UNSUPPORTED
        b = np.full(3, 30.0, np.float32)
        _lib.check(L.tmd_set_box(h, _lib.ptr(b)))
        q = np.zeros(n, np.float32)
        t = np.zeros(n, np.int32)
        _lib.check(L.tmd_set_atoms(h, _lib.ptr(q), _lib.ptr(t), 1, None, None))
        out = torch.empty(1, n, 3, device=DEV)
        x = torch.zeros(1, n, 3, device=DEV)
        assert L.tmd_forces(h, x.data_ptr(), out.data_ptr(), None, torch.cuda.current_stream().cuda_stream) == _lib.ERR_UNSUPPORTED
    finally:
        L.tmd_destroy(h)
    h = ctx()
    try:
        _lib.check(L.tmd_set_nonbonded(h, 1 << 5, -1.0, -1.0, 0, EPS, 332.0, 1.0))
        _lib.check(L.tmd_set_owned_atoms(h, 0, n // 2))
        assert L.tmd_set_gb(h, n, _lib.ptr(radius), _lib.ptr(screen), EPS, 0.0) == _lib.ERR_UNSUPPORTED
    finally:
        L.tmd_destroy(h)
    # integrators: the barostat and decomposed runs
    system = System(n, 1, F32, DEV)
    system.pos[:] = pos
    system.box[:] = torch.eye(3, device=DEV) * 40.0  # (a box the barostat takes: the refusal is about the solvent)
    with pytest.raises(RuntimeError, match="implicit solvent"):
        Integrator(system, fr, 1.0, DEV, gamma=1.0, T=300.0, barostat=MonteCarloBarostat(1.0))
    with pytest.raises(NotImplementedError, match="implicit solvent"):
        DecomposedIntegrator(system, fr, 1.0, DEV, gamma=1.0, T=300.0)

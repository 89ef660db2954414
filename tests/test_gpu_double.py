"""'precision: double' on the GPU: fp64 state through Forces / Integrator / Wrapper, checked against the reference's
own fp64 answers stored in the goldens and against the fp64 CPU oracle.

Tolerances: the stored fp64 answers and the kernels differ only in summation order and in the last ulps of pow and
sqrt (~1e-13 relative), so forces must agree to 1e-9 * max(1, max|F|) and every energy term to 1e-10 |E| + 1e-9.
Neighbour pairs are the reference's fp64 decisions bit for bit."""
import hashlib

import numpy as np
import pytest
import torch

from conftest import golden_cfg, golden_system_tensors, load_golden, params_from_golden
from oracle import refmd

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = torch.float64

# fixtures whose goldens the reference produced in fp64 with fp64 decisions
CASES = ["water291_rf_switch", "water291_plain", "argon100_nocut", "argon100_cut", "argon100_lj_rep_mix",
         "argon100_lj_rep_nocut", "water999_eq", "chain_amber_vacuum", "chain_amber_periodic", "chain_charmm_periodic",
         "adversarial_cutoff"]
CASES += ["charmm_" + n for n in ("1water", "2ions", "3ions", "1dihedral", "singledihedral", "4dihedrals", "benzamidine",
                                  "2watersperiodic", "sodiumperiodic", "waterbox")]
# the fp32 pair-set test skips water291_plain; so does this one
PAIR_CASES = [c for c in CASES if c not in ("water291_plain", "argon100_lj_rep_mix", "argon100_lj_rep_nocut")]
# goldens generated with fp32 decisions: compared with the fp64 oracle deciding in fp64
AMBER_CASES = ["ala2_nobox_rf", "ala2_xsc_rf", "benzamidine_amber_nocut", "ligand_amber_nocut", "thrombin_nobox_rf"]


def ftol(F):
    return 1e-9 * max(1.0, float(np.abs(F).max()))


def run64(g, skin=None, **kw):
    from torchmd_b200 import Forces

    par = params_from_golden(g, precision=F64, device=DEV)
    f = Forces(par, terms=[str(t) for t in g["terms"]], skin=skin, **golden_cfg(g), **kw)
    pos, box = golden_system_tensors(g, F64, DEV)
    F = torch.full_like(pos, 7.0)
    E = f.compute(pos, box, F, returnDetails=True)
    return f, pos, box, F, E


def sha(pairs):
    return hashlib.sha256(np.ascontiguousarray(pairs.astype(np.int32)).tobytes()).hexdigest()


@pytest.mark.parametrize("name", CASES)
def test_golden_forces_energies_f64(name):
    g = load_golden(name)
    f, pos, box, F, E = run64(g)
    ref = g["forces_f64"]
    err = np.abs(F.cpu().numpy() - ref).max()
    print(f"{name}: max|dF| vs reference fp64 {err:.3e} (max|F| {np.abs(ref).max():.1f})")
    assert err <= ftol(ref), err
    for r in range(len(E)):
        for c, k in enumerate(str(x) for x in g["energy_keys"]):
            e_ref = g["energies_f64"][r, c]
            assert abs(E[r][k] - e_ref) <= 1e-10 * abs(e_ref) + 1e-9, (k, E[r][k], e_ref)


@pytest.mark.parametrize("name", PAIR_CASES)
def test_golden_neighbour_pairs_f64_bit_exact(name):
    g = load_golden(name)
    if "npairs_f64" not in g:
        pytest.skip("no pair term")
    f, pos, box, F, E = run64(g)
    pairs = f.neighbour_pairs(pos, box).cpu().numpy()
    assert len(pairs) == int(g["npairs_f64"])
    assert sha(pairs) == str(g["pairs_sha256_f64"])


@pytest.mark.parametrize("name", AMBER_CASES)
def test_amber_fixtures_against_fp64_oracle(name):
    g = load_golden(name)
    f, pos, box, F, E = run64(g)
    terms = [str(t) for t in g["terms"]]
    o = refmd.OracleForces(params_from_golden(g, precision=F64), terms, decision_dtype=None, **golden_cfg(g))
    Fo = torch.zeros(pos.shape, dtype=F64)
    Eo = o.compute(pos.cpu(), box.cpu(), Fo)
    assert float((F.cpu() - Fo).abs().max()) <= ftol(Fo.numpy())
    for r in range(len(E)):
        for k in terms:
            want = float(Eo[r][k])
            assert abs(E[r][k] - want) <= 1e-10 * abs(want) + 1e-9, (k, E[r][k], want)
    if f.require_distances and golden_cfg(g)["cutoff"] is not None:
        want = o.neighbour_pairs(pos[0].cpu(), torch.diagonal(box[0]).cpu()).numpy().astype(np.int32)
        assert np.array_equal(f.neighbour_pairs(pos, box).cpu().numpy(), want)


def _argon(n, dtype, device="cpu"):
    from test_gpu_forces import _lj_coulomb_parameters

    return _lj_coulomb_parameters(n, dtype, device)


@pytest.mark.parametrize("periodic", [False, True])
def test_cutoff_adversaries_at_fp64_resolution(periodic):
    """Pairs planted at r_c (1 + k 2^-52), k = -4..4, along random directions; in the box the partners of the sites at
    x, y or z = 1 A that point the other way straddle the boundary."""
    from torchmd_b200 import Forces

    rc = 9.0
    rng = np.random.default_rng(5 + periodic)
    ks = np.arange(-4, 5)
    npairs = 4 * len(ks)
    L = 18 * rc  # 3 x 3 x 4 sites, 4 rc apart (and 6 rc across the boundary): only the planted partners interact
    coords = []
    for p in range(npairs):
        a = np.array([p % 3, (p // 3) % 3, p // 9], dtype=np.float64) * 4 * rc + 1.0
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        d = rc * (1.0 + ks[p % len(ks)] * 2.0**-52)
        coords += [a, a + d * u]
    coords = torch.tensor(np.array(coords))[None]
    n = coords.shape[1]
    box = (torch.eye(3, dtype=F64) * (L if periodic else 0.0))[None]
    cfg = dict(cutoff=rc, rfa=True)
    o = refmd.OracleForces(_argon(n, F64), ["lj", "electrostatics"], decision_dtype=None, **cfg)
    want = o.neighbour_pairs(coords[0], torch.diagonal(box[0])).numpy().astype(np.int32)
    f = Forces(_argon(n, F64, DEV), terms=["lj", "electrostatics"], **cfg)
    got = f.neighbour_pairs(coords.to(DEV), box.to(DEV)).cpu().numpy()
    assert 0 < len(want) < npairs
    assert np.array_equal(got, want)


def test_molecules_boxes_away_and_far_positions():
    """Waters moved one to three boxes away: the fp64 pair set bit for bit.  A molecule 10^5 A away is beyond the
    coordinates the fp32 shadow of the list build covers: the call reports it instead of returning."""
    from torchmd_b200 import Forces, testsystems
    from torchmd_b200._lib import TmdError

    sysd = testsystems.water_box(1000, seed=4)
    coords = np.asarray(sysd["coords"], dtype=np.float64).copy()
    L = np.asarray(sysd["box"], dtype=np.float64).reshape(-1)[:3]
    rng = np.random.default_rng(9)
    nmol = len(coords) // 3
    shift = rng.integers(-3, 4, size=(nmol, 3)) * (rng.random((nmol, 1)) < 0.4)
    coords += np.repeat(shift, 3, axis=0) * L
    terms, cfg = ["lj", "electrostatics", "bonds", "angles"], dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    pos = torch.tensor(coords)[None]
    box = torch.tensor(np.diag(L))[None]
    f = Forces(testsystems.water_parameters(sysd, precision=F64, device=DEV), terms=terms, **cfg)
    got = f.neighbour_pairs(pos.to(DEV), box.to(DEV)).cpu().numpy()
    o = refmd.OracleForces(testsystems.water_parameters(sysd, precision=F64), terms, decision_dtype=None, **cfg)
    want = o.neighbour_pairs(pos[0], torch.diagonal(box[0])).numpy().astype(np.int32)
    assert np.array_equal(got, want)
    Fo = torch.zeros_like(pos)
    o.compute(pos, box, Fo)
    F = torch.zeros_like(pos, device=DEV)
    f.compute(pos.to(DEV), box.to(DEV), F)
    assert float((F.cpu() - Fo).abs().max()) <= ftol(Fo.numpy())

    far = pos.clone()
    far[0, :3, 0] += 1.0e5
    with pytest.raises(TmdError, match="8192"):
        f.compute(far.to(DEV), box.to(DEV), F)


@pytest.mark.parametrize("periodic", [True, False])
def test_molecules_5000_to_8100_A_from_the_origin(periodic):
    """Coordinates where an fp32 ulp is 2^-10 to 2^-11 A, just inside the 8192 A limit: the range in which the shadow term
    of the list margin (tmd_b200.cu, finalize) matters.  Pairs bit for bit and forces against the fp64 oracle."""
    from torchmd_b200 import Forces, testsystems

    sysd = testsystems.water_box(1000, seed=6)
    coords = np.asarray(sysd["coords"], dtype=np.float64).copy()
    L = np.asarray(sysd["box"], dtype=np.float64).reshape(-1)[:3]
    rng = np.random.default_rng(10)
    nmol = len(coords) // 3
    if periodic:  # whole boxes: the same system, its molecules spread over 5000-8100 A
        shift = np.floor(rng.uniform(5000.0 + L, 8050.0 - L, size=(nmol, 3)) / L) * L
    else:  # one rigid translation
        shift = np.broadcast_to(rng.uniform(5000.0, 8100.0 - L, size=3), (nmol, 3))
    coords += np.repeat(shift, 3, axis=0)
    assert 5000.0 < coords.min() and coords.max() < 8192.0
    terms, cfg = ["lj", "electrostatics", "bonds", "angles"], dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    pos = torch.tensor(coords)[None]
    box = torch.tensor(np.diag(L) * (1.0 if periodic else 0.0))[None]
    f = Forces(testsystems.water_parameters(sysd, precision=F64, device=DEV), terms=terms, **cfg)
    got = f.neighbour_pairs(pos.to(DEV), box.to(DEV)).cpu().numpy()
    o = refmd.OracleForces(testsystems.water_parameters(sysd, precision=F64), terms, decision_dtype=None, **cfg)
    want = o.neighbour_pairs(pos[0], torch.diagonal(box[0])).numpy().astype(np.int32)
    assert len(want) > 0 and np.array_equal(got, want)
    Fo = torch.zeros_like(pos)
    o.compute(pos, box, Fo)
    F = torch.zeros_like(pos, device=DEV)
    f.compute(pos.to(DEV), box.to(DEV), F)
    assert float((F.cpu() - Fo).abs().max()) <= ftol(Fo.numpy())


def _water_setup64(g, t):
    from torchmd_b200 import Forces, System

    par = params_from_golden(g, precision=F64, device=DEV)
    forces = Forces(par, terms=[str(x) for x in g["terms"]], **golden_cfg(g))
    system = System(len(g["coords"]), int(g["cfg_nrep"]), F64, DEV)
    system.set_positions(g["coords"])
    system.set_box(g["box"])
    system.set_velocities(torch.tensor(t["vel0_f64"]))
    forces.compute(system.pos, system.box, system.forces)
    return forces, system


def test_nve_trajectory_f64():
    from torchmd_b200 import Integrator

    g, t = load_golden("water291_rf_switch"), load_golden("water291_traj")
    forces, system = _water_setup64(g, t)
    integ = Integrator(system, forces, 1.0, DEV)
    ek, ep, T = integ.step(niter=1)
    assert np.abs(system.pos.cpu().numpy() - t["nve_pos1_f64"]).max() < 1e-9
    assert np.abs(system.vel.cpu().numpy() - t["nve_vel1_f64"]).max() < 1e-9
    ek, ep, T = integ.step(niter=9)
    dp = np.abs(system.pos.cpu().numpy() - t["nve_pos10_f64"]).max()
    dv = np.abs(system.vel.cpu().numpy() - t["nve_vel10_f64"]).max()
    print(f"NVE fp64 10 steps: dpos {dp:.2e} dvel {dv:.2e}")
    assert dp < 1e-9 and dv < 1e-9
    assert ek.dtype == np.float64
    np.testing.assert_allclose(ek, t["nve_ekin10_f64"], rtol=1e-9)
    np.testing.assert_allclose(ep, t["nve_epot10_f64"], rtol=1e-9, atol=1e-9)


def test_langevin_injected_noise_f64():
    from torchmd_b200 import Integrator

    g, t = load_golden("water291_rf_switch"), load_golden("water291_traj")
    forces, system = _water_setup64(g, t)
    integ = Integrator(system, forces, 1.0, DEV, gamma=0.1, T=300.0)
    ek, ep, T = integ.step(niter=4, noise=torch.tensor(t["lan_noise_f64"]))
    assert np.abs(system.pos.cpu().numpy() - t["lan_pos4_f64"]).max() < 1e-9
    assert np.abs(system.vel.cpu().numpy() - t["lan_vel4_f64"]).max() < 1e-9
    np.testing.assert_allclose(T, t["lan_T4_f64"], rtol=1e-9)


def test_inkernel_fp64_langevin_noise_statistics():
    from test_gpu_integrator import ConstantForces
    from torchmd_b200 import Integrator, System

    n, nrep = 20000, 2
    system = System(n, nrep, F64, DEV)
    system.set_masses(torch.full((n,), 4.0))
    torch.manual_seed(3)
    integ = Integrator(system, ConstantForces(torch.zeros(nrep, n, 3, dtype=F64)), 1.0, DEV, gamma=0.0, T=300.0)
    integ.vcoeff = torch.full((n, 1), 0.5, device=DEV, dtype=F64)
    v_prev = system.vel.clone()
    draws = []
    for _ in range(3):
        integ.step(niter=1)
        draws.append(((system.vel - v_prev) / 0.5).cpu().numpy())
        v_prev = system.vel.clone()
    x = np.stack(draws)
    assert abs(x.mean()) < 0.01 and abs(x.std() - 1.0) < 0.01
    assert abs(np.mean(x**4) - 3.0) < 0.1
    flat = x.reshape(3, -1)
    assert abs(np.corrcoef(flat[0], flat[1])[0, 1]) < 0.01
    assert abs(np.corrcoef(x[0, 0, :, 0], x[0, 0, :, 2])[0, 1]) < 0.02


def test_autograd_and_vmap_f64():
    from torchmd_b200 import Forces

    g = load_golden("water291_rf_switch")
    want = load_golden("water291_autograd")["forces_autograd_f64"]
    f = Forces(params_from_golden(g, precision=F64, device=DEV), terms=[str(t) for t in g["terms"]], **golden_cfg(g))
    pos, box = golden_system_tensors(g, F64, DEV)
    q = pos.clone().requires_grad_(True)
    F = torch.zeros_like(pos)
    f.compute(q, box, F, explicit_forces=False)
    assert float(np.abs(F.cpu().numpy() - want).max()) <= ftol(want)
    e = f.compute(q, box, None, toNumpy=False, calculateForces=False)
    assert e.dtype == F64
    e.sum().backward()
    assert float(np.abs(-q.grad.cpu().numpy() - want).max()) <= ftol(want)
    batch = torch.stack([pos, pos])
    ev = torch.vmap(lambda p: f.compute(p, box, None, toNumpy=False, calculateForces=False))(batch)
    # (energies are block sums combined with atomics: equal to ~1e-13, not bitwise; forces are bitwise, below)
    assert ev.dtype == F64 and torch.allclose(ev[0], ev[1], rtol=1e-12, atol=1e-9)
    assert torch.allclose(ev[0], e.detach(), rtol=1e-12, atol=1e-9)


def test_determinism_and_equal_replicas():
    g = load_golden("water999_eq")
    f, pos, box, F, E = run64(g)
    F2 = torch.empty_like(F)
    f.compute(pos, box, F2)
    assert torch.equal(F, F2)
    pos3 = pos[:1].repeat(3, 1, 1).contiguous()
    box3 = box[:1].repeat(3, 1, 1).contiguous()
    F3 = torch.empty_like(pos3)
    f.compute(pos3, box3, F3)
    assert torch.equal(F3[0], F3[1]) and torch.equal(F3[0], F3[2])
    assert torch.equal(F3[0], F[0])


def test_overflow_regrowth_box_change_and_errors():
    """240 atoms in a 12 A blob of a 90 A box overflow the rows sized from the mean density: regrown inside compute()
    and inside Integrator.step; a changed box is picked up; mixed dtypes and decomposed runs are refused."""
    from test_gpu_forces import _lj_coulomb_parameters
    from torchmd_b200 import Forces, Integrator, System
    from torchmd_b200.domain import DecomposedIntegrator

    n = 240
    rng = np.random.default_rng(11)
    gr = np.stack(np.meshgrid(*[np.arange(7)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n] * 1.7 + 40.0
    coords = torch.tensor((gr + rng.normal(0, 0.05, gr.shape))[None], dtype=F64)
    box = (torch.eye(3, dtype=F64) * 90.0)[None]
    terms, cfg = ["lj", "electrostatics"], dict(cutoff=9.0, rfa=True)
    o = refmd.OracleForces(_lj_coulomb_parameters(n, F64, "cpu"), terms, decision_dtype=None, **cfg)
    Fo = torch.zeros(1, n, 3, dtype=F64)
    o.compute(coords, box, Fo)
    f = Forces(_lj_coulomb_parameters(n, F64, DEV), terms=terms, **cfg)
    p, b = coords.to(DEV), box.to(DEV)
    F = torch.zeros_like(p)
    f.compute(p, b, F)
    assert not f.stats()["overflow"]
    assert float((F.cpu() - Fo).abs().max()) <= ftol(Fo.numpy())

    b2 = (torch.eye(3, dtype=F64) * 60.0)[None]
    Fo2 = torch.zeros_like(Fo)
    o.compute(coords, b2, Fo2)
    f.compute(p, b2.to(DEV), F)
    assert float((F.cpu() - Fo2).abs().max()) <= ftol(Fo2.numpy())

    f2 = Forces(_lj_coulomb_parameters(n, F64, DEV), terms=terms, **cfg)
    system = System(n, 1, F64, DEV)
    system.set_positions(coords[0].numpy())
    system.set_box(np.array([90.0, 90.0, 90.0]))
    integ = Integrator(system, f2, 0.1, DEV)
    integ.step(niter=2)  # the first force call inside the fused call overflows: restored and rerun
    assert not f2.stats()["overflow"] and torch.isfinite(system.pos).all()

    with pytest.raises(RuntimeError, match="one precision"):
        f.compute(p, b.float(), F)
    with pytest.raises(RuntimeError, match="one precision"):
        f.compute(p, b, F.float())
    with pytest.raises(NotImplementedError):
        DecomposedIntegrator(system, f2, 1.0, DEV)


@pytest.mark.parametrize("case", ["water", "mixed", "nobonds", "zerobox"])
def test_wrap_f64_bit_exact(case):
    from torchmd_b200 import Wrapper

    z = load_golden("wrap_cases")
    natoms, bonds = int(z[case + "_natoms"]), z[case + "_bonds"]
    pos = torch.tensor(z[case + "_pos"], dtype=F64)
    box = torch.tensor(z[case + "_box"], dtype=F64)
    # move some atoms by whole and fractional boxes so that the fp64 offsets matter
    rng = np.random.default_rng(2)
    pos = pos + torch.tensor(rng.integers(-3, 4, size=pos.shape)) * torch.diagonal(box, dim1=1, dim2=2)[:, None, :]
    pos = pos + torch.tensor(rng.random(pos.shape) * 1e-3)
    want = pos.clone()
    groups, single = refmd.molecule_groups(natoms, bonds)
    refmd.wrap_positions(want, box, groups, single)
    w = Wrapper(natoms, bonds, DEV)
    got = pos.to(DEV).contiguous()
    w.wrap(got, box.to(DEV).contiguous())
    assert torch.equal(got.cpu(), want)


def test_minimize_bfgs_f64():
    from torchmd_b200 import Forces, System, testsystems
    from torchmd_b200.minimizers import minimize_bfgs

    sysd = testsystems.water_box(100, seed=1)
    terms, cfg = ["lj", "electrostatics", "bonds", "angles"], dict(cutoff=7.0, rfa=True)
    f = Forces(testsystems.water_parameters(sysd, precision=F64, device=DEV), terms=terms, **cfg)
    system = System(len(sysd["coords"]), 1, F64, DEV)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    e0 = f.compute(system.pos, system.box, system.forces)[0]
    minimize_bfgs(system, f, steps=50)
    e1 = f.compute(system.pos, system.box, system.forces)[0]
    assert system.pos.dtype == F64 and torch.isfinite(system.pos).all()
    assert e1 < e0

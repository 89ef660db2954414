"""Particle-mesh Ewald (Forces(..., pme=True)) on the GPU, against the numpy fp64 oracle (oracle/pme.py).

The fixtures run with PME in place of their reaction field and an 8 A cutoff, below half of their 16.6-19.8 A boxes.
Bounds:
* fp64: the library and the oracle evaluate the same formulas on the same pair set in fp64; the reciprocal part
  differs by the rounding of the FFTs and by the fixed-point charge grid (resolution 2^-40 of the total |charge| or
  finer), so 1e-9 of the largest force component and 1e-9 relative on energies hold with a wide margin.
* fp32: real space in fp32 (erfcf / expf within 4 / 2 ulp), an fp32 FFT grid; 5e-4 kcal/mol/A against the fp64 oracle
  on the fp32 pair set, as for the reference's own fp32 path.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIXTURES = ["water291_rf_switch", "charmm_2watersperiodic", "charmm_sodiumperiodic", "ala2_xsc_rf"]
EXCLUSIONS = ("bonds", "angles", "1-4")


def _fixture(name, dtype, cutoff=8.0):
    from torchmd_b200 import testsystems

    par, coords, box, terms, cfg = testsystems.golden_system(name, precision=dtype, device=DEV)
    par64 = testsystems.golden_system(name, precision=torch.float64)[0]
    sw = cfg["switch_dist"] if cfg["switch_dist"] is not None and cfg["switch_dist"] < cutoff else None
    return par, par64, coords, box, terms, dict(cutoff=cutoff, switch_dist=sw)


def _water(nw, dtype, nrep=1, cutoff=6.0, seed=0, jitter=0.0):
    """testsystems.water_box; ``jitter``: every molecule moved rigidly by up to that many A along each axis (the
    cluster lists do not take the exact lattice start)."""
    from torchmd_b200 import testsystems

    sysd = testsystems.water_box(nw, seed=seed)
    if jitter:
        shift = np.random.default_rng(seed + 1).uniform(-jitter, jitter, (nw, 1, 3))
        sysd["coords"] = (np.asarray(sysd["coords"]).reshape(nw, 3, 3) + shift).reshape(-1, 3).astype(np.float32)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    par64 = testsystems.water_parameters(sysd, precision=torch.float64)
    return sysd, par, par64, ["lj", "electrostatics", "bonds", "angles"], dict(cutoff=cutoff, switch_dist=cutoff - 1.0)


def _run(par, coords, boxes, terms, cfg, dtype, tol=5e-4, **kw):
    """Forces and per-term energies of Forces(pme=True) for replicas (R,N,3) in boxes (R,3)."""
    from torchmd_b200 import Forces

    pos = torch.tensor(np.asarray(coords), dtype=dtype, device=DEV)
    box = torch.diag_embed(torch.tensor(np.asarray(boxes), dtype=dtype, device=DEV))
    forces = Forces(par, terms=terms, pme=True, ewald_tolerance=tol, **cfg, **kw)
    F = torch.zeros_like(pos)
    E = forces.compute(pos, box, F, returnDetails=True)
    return forces, pos, box, F, E


def _oracle(par64, terms, cfg, pos, boxes, alpha, grid, decision_dtype):
    """fp64 oracle: oracle/refmd.py for every term, with its plain-Coulomb pair sum replaced by oracle/pme.py on the
    reference's pair set decided in ``decision_dtype`` (the scaled 1-4 Coulomb stays in the electrostatics)."""
    from oracle import pme as P
    from oracle import refmd
    from torchmd_b200.forces import ELEC_FACTOR

    pos = np.asarray(pos, np.float64)
    boxes = np.asarray(boxes, np.float64)
    pos_t = torch.tensor(pos)
    box_t = torch.diag_embed(torch.tensor(boxes))
    F = torch.zeros_like(pos_t)
    E = refmd.OracleForces(par64, terms, decision_dtype=decision_dtype, **cfg).compute(pos_t, box_t, F)
    Fc = torch.zeros_like(pos_t)
    Ec = refmd.OracleForces(par64, ["electrostatics"], decision_dtype=decision_dtype, **cfg).compute(pos_t, box_t, Fc)
    F = (F - Fc).numpy()
    other = [t for t in terms if t != "electrostatics"]
    ofe = refmd.OracleForces(par64, ["electrostatics"], cutoff=cfg["cutoff"])
    excl = np.asarray(par64.get_exclusions(EXCLUSIONS), np.int64).reshape(-1, 2)
    q = par64.charges.cpu().numpy().reshape(-1)
    out = []
    for r in range(len(pos)):
        pairs = ofe.neighbour_pairs(torch.tensor(pos[r]).to(decision_dtype), torch.tensor(boxes[r]).to(decision_dtype)).numpy()
        ee, fe = P.pme(pos[r], q, boxes[r], alpha, grid, pairs, excl, ELEC_FACTOR)
        F[r] += fe
        d = {t: float(E[r][t]) for t in other}
        d["electrostatics"] = float(E[r]["electrostatics"]) - float(Ec[r]["electrostatics"]) + ee
        out.append(d)
    return out, F


def _compare(dtype, par, par64, coords, boxes, terms, cfg):
    forces, pos, box, F, E = _run(par, coords, boxes, terms, cfg, dtype)
    alpha, grid = forces.pme_parameters()
    Eo, Fo = _oracle(par64, terms, cfg, pos.cpu().double().numpy(), boxes, alpha, grid, dtype)
    dF = np.abs(F.cpu().double().numpy() - Fo).max()
    fmax = np.abs(Fo).max()
    dE = max(abs(E[r][t] - Eo[r][t]) / max(1.0, abs(Eo[r][t])) for r in range(len(Eo)) for t in terms)
    return forces, dF, fmax, dE, F, Fo


@pytest.mark.parametrize("name", FIXTURES)
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_fixtures_against_the_oracle(name, dtype):
    par, par64, coords, box, terms, cfg = _fixture(name, dtype)
    _, dF, fmax, dE, _, _ = _compare(dtype, par, par64, coords[None], box[None], terms, cfg)
    print(f"{name} {dtype}: max |dF| {dF:.3e} (max |F| {fmax:.2f}), energy {dE:.3e}")
    if dtype == torch.float64:
        assert dF <= 1e-9 * fmax and dE <= 1e-9, (dF, fmax, dE)
    else:
        assert dF <= 5e-4 and dE <= 2e-5, (dF, dE)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_replicas_in_different_boxes(dtype, nw=60):
    sysd, par, par64, terms, cfg = _water(nw, dtype)
    L0 = np.asarray(sysd["box"], np.float64)
    scale = np.array([1.0, 1.04, 1.09])
    coords = np.stack([sysd["coords"] * s for s in scale]).astype(np.float32)
    boxes = np.stack([L0 * s for s in scale]).astype(np.float32)
    forces, dF, fmax, dE, _, _ = _compare(dtype, par, par64, coords, boxes, terms, cfg)
    print(f"{dtype}: 3 boxes, grid {forces.pme_parameters()}: max |dF| {dF:.3e}, energy {dE:.3e}")
    if dtype == torch.float64:
        assert dF <= 1e-9 * fmax and dE <= 1e-9, (dF, dE)
    else:
        assert dF <= 5e-4 and dE <= 2e-5, (dF, dE)


def _big_oracle(pos, q, L, cutoff, alpha, grid, excl, decision_dtype, atoms=None):
    """Electrostatics-only PME oracle for boxes too large for the all-pairs table of oracle/refmd.py: candidate pairs
    from a periodic k-d tree, then the reference's own predicate (refmd.pair_geometry, ``dist <= cutoff`` in
    ``decision_dtype``).  ``atoms``: the forces are exact only on these atoms (their pairs and exclusions only; the
    reciprocal part is always the whole box).  Returns (energy or None, forces (N,3))."""
    from scipy.spatial import cKDTree

    from oracle import pme as P
    from oracle import refmd
    from torchmd_b200.forces import ELEC_FACTOR

    N = len(pos)
    w = pos - L * np.floor(pos / L)
    w = np.where(w >= L, w - L, w)
    tree = cKDTree(w, boxsize=L)
    if atoms is None:
        cand = tree.query_pairs(cutoff + 0.01, output_type="ndarray")
    else:
        lists = tree.query_ball_point(w[atoms], cutoff + 0.01)
        cand = np.array([(a, j) for a, js in zip(atoms, lists) for j in js if j != a], np.int64)
    cand = np.unique(np.sort(cand, axis=1), axis=0)
    ex = np.unique(np.sort(np.asarray(excl, np.int64).reshape(-1, 2), axis=1), axis=0)
    cand = cand[~np.isin(cand[:, 0] * N + cand[:, 1], ex[:, 0] * N + ex[:, 1])]
    dist, _, _ = refmd.pair_geometry(torch.tensor(pos).to(decision_dtype), torch.tensor(cand),
                                     torch.tensor(L).to(decision_dtype))
    pairs = cand[(dist <= cutoff).numpy()]
    if atoms is not None:
        ex = ex[np.isin(ex[:, 0], atoms) | np.isin(ex[:, 1], atoms)]
    er, fr = P.real_space(pos, q, L, alpha, pairs, ELEC_FACTOR)
    ek, fk = P.reciprocal(pos, q, L, alpha, grid, ELEC_FACTOR)
    ex_e, fx = P.exclusion_correction(pos, q, L, alpha, ex, ELEC_FACTOR)
    e = er + ek + ex_e + P.self_and_background(q, L, alpha, ELEC_FACTOR) if atoms is None else None
    return e, fr + fk + fx


def _water_big(nw, dtype, nsample=None, seed=0, cutoff=9.0):
    from torchmd_b200 import _lib

    sysd, par, par64, _, _ = _water(nw, dtype, jitter=0.7)
    cfg = dict(cutoff=cutoff)
    forces, pos, box, F, E = _run(par, sysd["coords"][None], sysd["box"][None], ["electrostatics"], cfg, dtype)
    kernel = _lib.lib().tmd_pair_kernel(forces._ctx)
    alpha, grid = forces.pme_parameters()
    p64 = pos.cpu().double().numpy()[0]
    L = np.asarray(sysd["box"], np.float64)
    q = par64.charges.numpy().reshape(-1)
    atoms = None if nsample is None else np.sort(np.random.default_rng(seed).choice(len(q), nsample, replace=False))
    eo, Fo = _big_oracle(p64, q, L, cutoff, alpha, grid, par64.get_exclusions(EXCLUSIONS), dtype, atoms)
    Fg = F.cpu().double().numpy()[0]
    sel = slice(None) if atoms is None else atoms
    dF = np.abs(Fg[sel] - Fo[sel]).max()
    fmax = np.abs(Fo[sel]).max()
    dE = None if eo is None else abs(E[0]["electrostatics"] - eo) / abs(eo)
    print(f"water {3 * nw} atoms {dtype}: kernel {kernel}, alpha {alpha:.4f}, grid {grid}, max |dF| {dF:.3e} "
          f"(max |F| {fmax:.2f}{'' if atoms is None else f', {len(atoms)} sampled atoms'}), energy {dE}")
    return kernel, grid, dF, fmax, dE


def test_water10k_f64_against_the_oracle():
    kernel, grid, dF, fmax, dE = _water_big(3333, torch.float64)
    assert kernel == 8 and grid == (45, 45, 45)
    assert dF <= 1e-9 * fmax and dE <= 1e-9, (dF, fmax, dE)


@pytest.mark.parametrize("nw,want_kernel,grid", [(3333, None, 45), (33333, 10, 90)])
def test_water_f32_sampled_atoms_against_the_oracle(nw, want_kernel, grid):
    """fp32 default path (water100k: the Ewald cluster kernel) against the fp64 oracle on 2000 sampled atoms."""
    kernel, g, dF, fmax, _ = _water_big(nw, torch.float32, nsample=2000)
    assert g == (grid,) * 3 and (want_kernel is None or kernel == want_kernel), (kernel, g)
    assert dF <= 5e-4, dF


def test_fp32_error_is_far_below_the_method_error():
    """water291_rf_switch's box, electrostatics only: the RMS force deviation of the fp32 path from the fp64 oracle is
    at least 10x below the RMS error of smooth PME itself (default tolerance) against the exact Ewald sum."""
    from oracle import pme as P
    from torchmd_b200.forces import ELEC_FACTOR

    par, par64, coords, box, _, cfg = _fixture("water291_rf_switch", torch.float32)
    terms = ["electrostatics"]
    forces, pos, b, F, E = _run(par, coords[None], box[None], terms, cfg, torch.float32)
    alpha, grid = forces.pme_parameters()
    p64 = pos.cpu().double().numpy()
    _, Fo = _oracle(par64, terms, cfg, p64, box[None], alpha, grid, torch.float32)
    q = par64.charges.numpy().reshape(-1)
    L = box.astype(np.float64)
    _, Fx = P.ewald_exact(p64[0], q, L, k=ELEC_FACTOR)
    excl = np.unique(np.sort(np.asarray(par64.get_exclusions(EXCLUSIONS)).reshape(-1, 2), axis=1), axis=0)
    for i, j in excl:  # the excluded pairs carry no Coulomb energy at all
        d = p64[0, i] - p64[0, j]
        d -= L * np.rint(d / L)
        f = ELEC_FACTOR * q[i] * q[j] * d / np.linalg.norm(d) ** 3
        Fx[i] -= f
        Fx[j] += f
    rms32 = float(np.sqrt(np.mean((F.cpu().double().numpy()[0] - Fo[0]) ** 2)))
    rms_method = float(np.sqrt(np.mean((Fo[0] - Fx) ** 2)))
    print(f"water291 box, alpha {alpha:.4f}, grid {grid}: RMS |F32 - F64 oracle| {rms32:.3e}, RMS |SPME - exact Ewald| {rms_method:.3e} kcal/mol/A")
    assert rms32 * 10 <= rms_method, (rms32, rms_method)


def test_pme_kernels_only_with_pme(monkeypatch, nw_cluster=1200):
    """Every pair path a periodic PME context can take runs a real-space Ewald kernel: tmd_pair_kernel 6 k_pair<MODE 2>,
    7 k_pair_fx<MODE 2>, 8 k_ewpair64, 9 k_pair_fx2_ew, 10 k_cpair_ew -- and each one where its path applies."""
    from torchmd_b200 import _lib

    ewald32 = (6, 7, 9, 10)
    for env in ({"TMD_B200_FX": "0"}, {"TMD_B200_FX": "1"}, {"TMD_B200_FX": "2"}, {"TMD_B200_CLUSTER": "1"}, {"TMD_B200_CLUSTER": "0"}):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        for dtype, want in ((torch.float32, ewald32), (torch.float64, (8,))):
            sysd, par, _, terms, cfg = _water(200, dtype)  # (L = 18.2 A: the guard-free image holds at skin 0.5)
            for skin in (0.5, 3.0):  # 3 A: not the guard-free image (k_pair<SAFE = false>)
                forces, *_ = _run(par, sysd["coords"][None], sysd["box"][None], terms, cfg, dtype, skin=skin)
                got = _lib.lib().tmd_pair_kernel(forces._ctx)
                assert got in want, (env, dtype, skin, got)
                if dtype == torch.float32 and skin == 0.5:  # the guard-free image: the fixed-point kernels
                    assert got == {"0": 6, "1": 7, "2": 9}.get(env.get("TMD_B200_FX"), got), (env, got)
                if dtype == torch.float32 and skin == 3.0:
                    assert got == 6, (env, got)
        for k in env:
            monkeypatch.delenv(k)
    # a box the cluster lists take (L > 2 (rl + 8 A + skin)): the Ewald cluster kernel
    monkeypatch.setenv("TMD_B200_CLUSTER", "1")
    sysd, par, _, terms, cfg = _water(nw_cluster, torch.float32, jitter=0.7)
    forces, *_ = _run(par, sysd["coords"][None], sysd["box"][None], ["electrostatics"], dict(cutoff=6.0), torch.float32)
    assert _lib.lib().tmd_pair_kernel(forces._ctx) == 10


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_pair_set_is_the_same_with_pme(dtype):
    from torchmd_b200 import Forces

    par, _, coords, box, terms, cfg = _fixture("water291_rf_switch", dtype)
    pos = torch.tensor(coords[None], dtype=dtype, device=DEV)
    b = torch.diag_embed(torch.tensor(box[None], dtype=dtype, device=DEV))
    with_pme = Forces(par, terms=terms, pme=True, **cfg).neighbour_pairs(pos, b).cpu().numpy()
    without = Forces(par, terms=terms, **cfg).neighbour_pairs(pos, b).cpu().numpy()
    assert np.array_equal(with_pme, without)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_explicit_and_autograd_paths_agree(dtype):
    from torchmd_b200 import Forces

    par, _, coords, box, terms, cfg = _fixture("ala2_xsc_rf", dtype)
    cfg["switch_dist"] = None  # (the explicit switched-LJ formula is not a gradient; PME itself is one either way)
    forces = Forces(par, terms=terms, pme=True, **cfg)
    pos = torch.tensor(coords[None], dtype=dtype, device=DEV)
    b = torch.diag_embed(torch.tensor(box[None], dtype=dtype, device=DEV))
    F1 = torch.zeros_like(pos)
    E1 = forces.compute(pos, b, F1)
    p = pos.clone().requires_grad_(True)
    F2 = torch.zeros_like(pos)
    E2 = forces.compute(p, b, F2, explicit_forces=False)
    assert torch.equal(F1, F2) and abs(E1[0] - E2[0]) <= 1e-12 * abs(E1[0])  # (energies: block sums added atomically)
    p = pos.clone().requires_grad_(True)
    E3 = forces.compute(p, b, None, toNumpy=False, calculateForces=False)
    E3.sum().backward()
    assert torch.equal(-p.grad, F1)
    assert abs(float(E3.sum().detach()) - E1[0]) <= 1e-6 * abs(E1[0])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_forces_are_bitwise_reproducible(dtype):
    par, _, coords, box, terms, cfg = _fixture("ala2_xsc_rf", dtype)
    forces, pos, b, F1, E1 = _run(par, coords[None], box[None], terms, cfg, dtype)
    for _ in range(2):
        F2 = torch.zeros_like(F1)
        forces.compute(pos, b, F2)
        assert torch.equal(F1, F2)


def _md(dtype, nw, nsteps, chunk, dt=2.0, gamma=1.0, seed=0, tol=5e-4):
    from torchmd_b200 import Constraints, Forces, Integrator, System, maxwell_boltzmann, testsystems

    sysd = testsystems.water_box(nw, seed=seed)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    system = System(len(sysd["coords"]), 1, dtype, DEV)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    cut = min(9.0, 0.5 * float(np.min(sysd["box"])))
    forces = Forces(par, terms=["lj", "electrostatics", "bonds", "angles"], cutoff=cut, switch_dist=cut - 1.5, pme=True,
                    ewald_tolerance=tol)
    torch.manual_seed(seed)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    integ = Integrator(system, forces, dt, DEV, gamma=gamma, T=300.0 if gamma else None, constraints=Constraints(par, "water"))
    out = []
    for _ in range(nsteps // chunk):
        ekin, pot, _ = integ.step(chunk)
        out.append((float(ekin[0]), float(pot[0])))
    return system, forces, np.array(out)


def test_captured_steps_match_step_by_step(monkeypatch, nw=300, nsteps=20):
    """Rigid water at 2 fs with Langevin: the captured step (one graph launch) and the stream path give the same bits."""
    monkeypatch.setenv("TMD_B200_GRAPH", "1")
    s1, _, e1 = _md(torch.float32, nw, nsteps, nsteps // 2)
    monkeypatch.setenv("TMD_B200_GRAPH", "0")
    s2, _, e2 = _md(torch.float32, nw, nsteps, nsteps // 2)
    assert torch.equal(s1.pos, s2.pos) and torch.equal(s1.vel, s2.vel)
    np.testing.assert_allclose(e1, e2, rtol=1e-12)  # (energies: block sums added atomically)


def test_launches_per_step_are_fixed(nw=300):
    """The kernels of one PME step are a fixed number: 7 more than the same step on the same pair path without PME
    (k_pme_spread, five k_pme_fft line passes, k_pme_gather); the rebuild kernels run inside the conditional node and are
    not counted."""
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann, testsystems

    def per_step(pme):
        sysd = testsystems.water_box(nw, seed=0)
        par = testsystems.water_parameters(sysd, device=DEV)
        system = System(len(sysd["coords"]), 1, torch.float32, DEV)
        system.set_positions(sysd["coords"])
        system.set_box(sysd["box"])
        cut = min(9.0, 0.5 * float(np.min(sysd["box"])))
        extra = dict(pme=True) if pme else {}
        forces = Forces(par, terms=["lj", "electrostatics", "bonds", "angles"], cutoff=cut, switch_dist=cut - 1.5, **extra)
        torch.manual_seed(0)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        integ = Integrator(system, forces, 1.0, DEV, gamma=1.0, T=300.0)
        integ.step(3)
        counts = []
        for n in (5, 9):
            l0 = forces.stats()["kernel_launches"]
            integ.step(n)
            counts.append((forces.stats()["kernel_launches"] - l0) / n)
        return counts

    with_pme = per_step(True)
    print("launches per step with PME:", with_pme)
    assert with_pme[0] == with_pme[1]
    without = per_step(False)
    assert with_pme[0] == without[0] + 7, (with_pme, without)


def test_madelung_energy_f64():
    """Rock salt, 4 x 4 x 4 conventional cells (512 ions, d = 2.8 A), electrostatics only, tolerance 1e-6."""
    from oracle import pme as P
    from torchmd_b200 import Forces, TopologyParameters
    from torchmd_b200.forces import ELEC_FACTOR

    pos, q, L = P.madelung_rocksalt(4, 2.8)
    n = len(q)
    par = TopologyParameters(atom_types=np.zeros(n, np.int64), type_sigma=[1.0], type_epsilon=[0.0], charges=q,
                             masses=np.full(n, 23.0), precision=torch.float64, device=DEV)
    forces = Forces(par, terms=["electrostatics"], cutoff=9.0, pme=True, ewald_tolerance=1e-6)
    p = torch.tensor(pos[None], dtype=torch.float64, device=DEV)
    box = torch.diag_embed(torch.tensor(L[None], dtype=torch.float64, device=DEV))
    F = torch.zeros_like(p)
    E = forces.compute(p, box, F)[0]
    want = -n * P.MADELUNG_NACL * ELEC_FACTOR / (2 * 2.8)
    print(f"Madelung: {E:.10f} vs {want:.10f} ({abs(E / want - 1):.2e}), max |F| {F.abs().max().item():.2e}")
    assert abs(E / want - 1) <= 1e-5
    assert F.abs().max().item() <= 1e-3


def test_refusals():
    from torchmd_b200 import Forces, _lib
    from torchmd_b200.domain import DecomposedIntegrator

    sysd, par, _, terms, cfg = _water(60, torch.float32)
    with pytest.raises(RuntimeError, match="cutoff"):
        Forces(par, terms=terms, pme=True)
    with pytest.raises(RuntimeError, match="exclude each other"):
        Forces(par, terms=terms, pme=True, rfa=True, cutoff=6.0)
    with pytest.raises(RuntimeError, match="electrostatics"):
        Forces(par, terms=["lj", "bonds"], pme=True, cutoff=6.0)
    L = sysd["box"]
    for bad, what in ((np.zeros(3, np.float32), "periodic"), (np.array([L[0], 11.0, L[2]], np.float32), "half")):
        with pytest.raises(RuntimeError, match=what):
            _run(par, sysd["coords"][None], bad[None], terms, cfg, torch.float32)
    forces, pos, box, F, E = _run(par, sysd["coords"][None], L[None], terms, cfg, torch.float32)
    from torchmd_b200 import System

    system = System(len(sysd["coords"]), 1, torch.float32, DEV)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    with pytest.raises(NotImplementedError, match="one GPU"):
        DecomposedIntegrator(system, forces, 1.0, DEV)
    assert _lib.lib().tmd_set_owned_atoms(forces._ctx, 0, 10) == -5
    import ctypes as C

    assert _lib.lib().tmd_dd_create(forces._ctx, 0, 1, (C.c_ubyte * 64)()) == -5
    # the exclusion correction needs the rows as a set: each pair in both rows, once
    n = len(sysd["coords"])
    for rows in ([[1], []], [[1, 1], [0, 0]]):  # one direction only; a pair listed twice
        row_ptr = np.zeros(n + 1, np.int64)
        row_ptr[1:3] = np.cumsum([len(r) for r in rows])
        row_ptr[3:] = row_ptr[2]
        cols = np.array([c for r in rows for c in r], np.int32)
        _lib.check(_lib.lib().tmd_set_exclusions(forces._ctx, row_ptr.ctypes.data, cols.ctypes.data))
        with pytest.raises(RuntimeError, match="both rows, once"):
            forces.compute(pos, box, F)


def test_nve_rigid_water_energy_conservation_f64(nw=1000, nsteps=5000, tol=1e-5):
    """fp64 NVE, 1000 rigid TIP3P waters, 2 fs: E_tot fluctuates by less than 2 % of E_kin's fluctuation; prints the
    drift in kcal/mol/ns.  The real-space term is cut at rc without a shift, so every pair that crosses the cutoff
    changes the energy by k qi qj erfc(alpha rc) / rc; at the default tolerance (erfc(alpha rc) = 2e-4) that alone
    gives a fluctuation ratio of about 2.6 % (DESIGN 5b); at 1e-5 the jump is 60 times smaller."""
    system, forces, e = _md(torch.float64, nw, nsteps, 10, gamma=None, tol=tol)
    ekin, pot = e[:, 0], e[:, 1]
    etot = ekin + pot
    t_ns = np.arange(len(etot)) * 10 * 2e-6
    drift = np.polyfit(t_ns, etot, 1)[0]
    ratio = etot.std() / ekin.std()
    print(f"NVE PME fp64: std E_tot {etot.std():.4f}, std E_kin {ekin.std():.4f}, ratio {ratio:.4f}, drift {drift:.2f} kcal/mol/ns, "
          f"alpha/grid {forces.pme_parameters()}")
    assert ratio < 0.02, ratio

"""Parity of the CUDA force path (through the C ABI, via torchmd_b200.Forces) with the
golden vectors of the unmodified reference and with the CPU oracle.

Tolerances (stated here, used below):
  * neighbour pairs: bit-exact -- identical (i<j) index set as ava_idx[dist<=cutoff].
  * forces: max |dF| component < 1e-4 kcal/mol/A against the reference evaluated in
    fp64 on the reference's own fp32 pair set (same fp32 inputs, same in/out decisions,
    exact values) on configurations whose largest force is O(100).  The reference's own
    fp32 result is 0.8e-4 (291 atoms) to 4e-4 (10k atoms) away from that yardstick --
    it loses bits in fl(p_i - p_j) across the periodic boundary, which the kernels
    restore (physics.cuh sub_err) -- so against the fp32 reference the bound is
    1e-4 + that deviation (triangle inequality).  For cases with larger forces the
    bounds scale with max|F|/100 (fp32 relative precision).
  * energies: |dE| <= 2e-6 * sum|pair terms| scale, i.e. relative 1e-5 of the term
    magnitude plus 2e-3 absolute.
"""
import os

import numpy as np
import pytest
import torch

from conftest import golden_cfg, golden_system_tensors, load_golden, params_from_golden
from oracle import refmd
from torchmd_b200._lib import PAIR_CLUSTER

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

CASES = [
    "water291_rf_switch",
    "water291_plain",
    "argon100_nocut",
    "argon100_cut",
    "water999_eq",
    "chain_amber_vacuum",
    "chain_amber_periodic",
    "chain_charmm_periodic",
    "adversarial_cutoff",
    "ala2_nobox_rf",  # BASELINE.json config 3 (all AMBER terms), 2 replicas, no box
    "ala2_xsc_rf",  # same system in its periodic box (the tutorial's run)
    "thrombin_nobox_rf",  # config 5: 4676-atom protein + ligand in vacuum, cutoff 7.3, 2 replicas
]
# The two small
# AMBER fixtures of the reference's own test matrix (tests/data), configured as test_torchmd.py:363-365 does without a
# box -- no cutoff, plain Coulomb, all terms; the two replicas are different configurations.
NEW_CASES = ["benzamidine_amber_nocut", "ligand_amber_nocut"]
# ... and its small CHARMM fixtures (PSF + PDB + .prm; goldens from the reference's own Parameters + Forces.compute,
# tests/golden/make_golden_charmm.py)
NEW_CASES += ["charmm_" + n for n in ("1water", "2ions", "3ions", "1dihedral", "singledihedral", "4dihedrals", "benzamidine", "2watersperiodic", "sodiumperiodic", "waterbox")]


def force_tol(ref_F, ref_dev=0.0):
    """1e-4 (scaled with the force magnitude) + the reference's own fp32-vs-fp64 deviation."""
    return 1e-4 * max(1.0, float(np.abs(ref_F).max()) / 100.0) + ref_dev


def run_gpu(g, skin=None, **kw):
    from torchmd_b200 import Forces

    par = params_from_golden(g, precision=torch.float32, device=DEV)
    terms = [str(t) for t in g["terms"]]
    f = Forces(par, terms=terms, skin=skin, **golden_cfg(g), **kw)
    pos, box = golden_system_tensors(g, torch.float32, DEV)
    F = torch.full_like(pos, 7.0)  # must be overwritten, not accumulated into
    E = f.compute(pos, box, F, returnDetails=True)
    return f, pos, box, F, E


@pytest.mark.parametrize("name", CASES)
def test_golden_forces_energies(name):
    g = load_golden(name)
    f, pos, box, F, E = run_gpu(g)
    ref = g["forces_f64"]
    err = np.abs(F.cpu().numpy().astype(np.float64) - ref).max()
    err32 = np.abs(F.cpu().numpy() - g["forces_f32"]).max()
    print(f"{name}: max|dF| vs ref fp32 {err32:.3e}, vs ref fp64 {err:.3e}, max|F| {np.abs(ref).max():.1f}")
    dev = np.abs(g["forces_f32"].astype(np.float64) - ref).max()
    # bonded-heavy fixtures (strained chains, |F| ~ 1000): acos/atan2 in fp32 dominate; there the
    # yardstick is the reference's own fp32 deviation
    assert err < max(force_tol(ref), 1.2 * dev), f"max |dF| vs fp64 reference {err:.3e} (max |F| {np.abs(ref).max():.1f})"
    assert err32 < force_tol(ref, dev), f"max |dF| vs fp32 reference {err32:.3e} (reference fp32 vs fp64: {dev:.3e})"
    keys = [str(k) for k in g["energy_keys"]]
    for r in range(len(E)):
        for c, k in enumerate(keys):
            e_ref = g["energies_f64"][r, c]
            assert abs(E[r][k] - e_ref) <= 1e-5 * abs(e_ref) + 2e-3, (k, E[r][k], e_ref)
        assert E[r]["external"] == 0.0
    # default return format: list of total energies per replica
    tot = f.compute(pos, box, F)
    assert isinstance(tot, list) and len(tot) == pos.shape[0]
    assert abs(tot[0] - g["energies_f64"][0].sum()) <= 1e-5 * np.abs(g["energies_f64"][0]).sum() + 2e-3


@pytest.mark.parametrize("name", [c for c in CASES if not c.startswith("water291_plain")])
def test_golden_neighbour_pairs_bit_exact(name):
    g = load_golden(name)
    if "npairs_f32" not in g:
        pytest.skip("no pair term")
    f, pos, box, F, E = run_gpu(g)
    pairs = f.neighbour_pairs(pos, box).cpu().numpy()
    assert len(pairs) == int(g["npairs_f32"])
    if "pairs_f32" in g:
        assert np.array_equal(pairs, g["pairs_f32"])
    import hashlib

    assert hashlib.sha256(np.ascontiguousarray(pairs.astype(np.int32)).tobytes()).hexdigest() == str(g["pairs_sha256_f32"])


@pytest.mark.parametrize("name", NEW_CASES)
def test_new_reference_fixtures(name):
    test_golden_forces_energies(name)
    test_golden_neighbour_pairs_bit_exact(name)


def test_molecules_several_boxes_away_meet_the_plain_yardstick():
    """Whole waters moved up to seven box lengths away (image counts for which fl(L * count) is inexact): the same pair set
    as the fp32 reference, and forces within the plain 1e-4 yardstick of the fp64 values on that pair set -- the float
    kernel's force values use the unrounded image shift (physics.cuh straddle_value), the reference's fp32 path does not."""
    from torchmd_b200 import Forces

    g = load_golden("water999_eq")
    rng = np.random.default_rng(7)
    coords = g["coords"].astype(np.float64).copy()
    L = g["box"].astype(np.float64).reshape(-1)[:3]
    shift = rng.integers(-7, 8, size=(len(coords) // 3, 3)) * (rng.random((len(coords) // 3, 1)) < 0.3)
    coords += np.repeat(shift, 3, axis=0) * L
    terms = [str(t) for t in g["terms"]]
    cfg = golden_cfg(g)
    f = Forces(params_from_golden(g, precision=torch.float32, device=DEV), terms=terms, **cfg)
    pos = torch.tensor(coords, dtype=torch.float32, device=DEV)[None].contiguous()
    box = torch.zeros(1, 3, 3, dtype=torch.float32, device=DEV)
    for k in range(3):
        box[0, k, k] = float(L[k])
    F = torch.zeros_like(pos)
    f.compute(pos, box, F)
    p32 = pos.cpu()
    o64 = refmd.OracleForces(params_from_golden(g, precision=torch.float64), terms, decision_dtype=torch.float32, **cfg)
    F64 = torch.zeros(1, len(coords), 3, dtype=torch.float64)
    o64.compute(p32.double(), box.cpu().double(), F64)
    o32 = refmd.OracleForces(params_from_golden(g, precision=torch.float32), terms, **cfg)
    F32 = torch.zeros(1, len(coords), 3)
    o32.compute(p32, box.cpu(), F32)
    want = o32.neighbour_pairs(p32[0], torch.diagonal(box[0].cpu())).numpy().astype(np.int32)
    assert np.array_equal(f.neighbour_pairs(pos, box).cpu().numpy(), want)
    err = float((F.cpu().double() - F64).abs().max())
    dev = float((F32.double() - F64).abs().max())
    print(f"far images: max|dF| vs fp64 {err:.3e}; the reference's fp32 path is {dev:.3e} away")
    assert err < force_tol(F64.numpy())


@pytest.mark.parametrize("skin", [0.0, 0.3, 2.5])
def test_results_do_not_depend_on_skin(skin):
    g = load_golden("water999_eq")
    f, pos, box, F, E = run_gpu(g, skin=skin)
    pairs = f.neighbour_pairs(pos, box).cpu().numpy()
    assert np.array_equal(pairs, g["pairs_f32"])
    assert np.abs(F.cpu().numpy().astype(np.float64) - g["forces_f64"]).max() < force_tol(g["forces_f64"])


def test_forces_deterministic_and_replicas_identical():
    g = load_golden("water291_rf_switch")  # 2 replicas of the same coordinates
    f, pos, box, F, E = run_gpu(g)
    F1 = F.clone()
    f.compute(pos, box, F)
    assert torch.equal(F, F1), "two evaluations of the same positions must agree bitwise"
    # no atomics anywhere in the force path: replicas of the same coordinates agree bitwise too
    assert torch.equal(F[0], F[1])
    assert abs(E[0]["lj"] - E[1]["lj"]) < 1e-9


@pytest.mark.parametrize("nwat,seed", [(1000, 1), (3333, 2)])
def test_synthetic_water_vs_oracle(nwat, seed):
    """Sizes the all-pairs oracle finishes in seconds; configuration relaxed on the GPU first."""
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann, testsystems

    sysd = testsystems.water_box(nwat, seed=seed)
    terms = ["lj", "electrostatics", "bonds", "angles"]
    cfg = dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    par = testsystems.water_parameters(sysd, device=DEV)
    n = len(sysd["coords"])
    system = System(n, 1, torch.float32, DEV)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    torch.manual_seed(seed)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    forces = Forces(par, terms=terms, **cfg)
    forces.compute(system.pos, system.box, system.forces)
    integ = Integrator(system, forces, 1.0, DEV, gamma=50.0, T=300.0)
    integ.step(niter=1500)  # lattice start -> liquid near 300 K
    st = forces.stats()
    assert st["rebuilds"] >= 2 and not st["overflow"]

    E = forces.compute(system.pos, system.box, system.forces, returnDetails=True)[0]
    pairs = forces.neighbour_pairs(system.pos, system.box).cpu().numpy()

    pos32 = system.pos.cpu()
    box32 = system.box.cpu()
    of32 = refmd.OracleForces(testsystems.water_parameters(sysd), terms, **cfg)
    ref_pairs = of32.neighbour_pairs(pos32[0], torch.diagonal(box32[0])).numpy().astype(np.int32)
    assert pairs.shape == ref_pairs.shape and np.array_equal(pairs, ref_pairs)

    F32 = torch.zeros(1, n, 3)
    of32.compute(pos32, box32, F32)
    # yardstick: fp64 values on the reference's fp32 in/out decisions
    of64 = refmd.OracleForces(testsystems.water_parameters(sysd, precision=torch.float64), terms,
                              decision_dtype=torch.float32, **cfg)
    F64 = torch.zeros(1, n, 3, dtype=torch.float64)
    E64 = of64.compute(pos32.double(), box32.double(), F64)[0]
    err32 = (system.forces.cpu() - F32).abs().max().item()
    err = (system.forces.cpu().double() - F64).abs().max().item()
    dev = (F32.double() - F64).abs().max().item()
    print(f"water{n}: max|dF| vs oracle fp64(fp32 decisions) {err:.3e}, vs oracle fp32 {err32:.3e}; "
          f"oracle fp32 vs fp64 {dev:.3e}; max|F| {F64.abs().max().item():.1f}")
    rms = (system.forces.cpu().double() - F64).pow(2).mean().sqrt().item()
    print(f"water{n}: rms dF {rms:.3e}")
    assert err < force_tol(F64.numpy()), err
    assert err32 < force_tol(F64.numpy(), dev), err32
    assert rms < 2e-5
    for k in terms:
        assert abs(E[k] - E64[k]) <= 1e-5 * abs(E64[k]) + 2e-3, (k, E[k], E64[k])


def test_large_box_properties():
    """BASELINE size (99,999 atoms): properties that need no O(N^2) oracle."""
    from torchmd_b200 import Forces, System, testsystems

    sysd = testsystems.water_box(33333, seed=0)
    par = testsystems.water_parameters(sysd, device=DEV)
    n = len(sysd["coords"])
    system = System(n, 1, torch.float32, DEV)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    cfg = dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    fa = Forces(par, terms=["lj", "electrostatics"], skin=0.5, **cfg)
    fb = Forces(par, terms=["lj", "electrostatics"], skin=2.0, **cfg)
    Fa, Fb = torch.empty_like(system.pos), torch.empty_like(system.pos)
    Ea = fa.compute(system.pos, system.box, Fa, returnDetails=True)[0]
    Eb = fb.compute(system.pos, system.box, Fb, returnDetails=True)[0]
    # identical pair set and summation order irrespective of the list radius? order may differ: compare to rounding
    assert (Fa - Fb).abs().max().item() < 2e-3 * max(1.0, Fa.abs().max().item() / 100.0)
    # same pair set, different per-lane fp32 summation order
    assert abs(Ea["lj"] - Eb["lj"]) <= 1e-6 * abs(Ea["lj"]) + 1e-3
    assert abs(Ea["electrostatics"] - Eb["electrostatics"]) <= 1e-6 * abs(Ea["electrostatics"]) + 1e-3
    # Newton's third law: pair forces sum to zero
    tot = Fa.double().sum(dim=1).abs().max().item()
    assert tot < 5e-2, tot
    pa = fa.neighbour_pairs(system.pos, system.box)
    pb = fb.neighbour_pairs(system.pos, system.box)
    assert torch.equal(pa, pb)
    # translation by whole box vectors (unwrapped coordinates) must not change the pair set
    shifted = system.pos.clone()
    shifted[0, ::7] += torch.tensor(sysd["box"], device=DEV) * torch.tensor([1.0, -2.0, 3.0], device=DEV)
    pc = fa.neighbour_pairs(shifted, system.box)
    assert pc.shape[0] > 0.999 * pa.shape[0]


def test_api_errors_and_formats():
    from torchmd_b200 import Forces

    g = load_golden("water291_rf_switch")
    par = params_from_golden(g, device=DEV)
    with pytest.raises(RuntimeError):
        Forces(par, terms=None)
    with pytest.raises(ValueError):
        Forces(par, terms=["lj", "magic"])
    with pytest.raises(RuntimeError):
        Forces(par, terms=["1-4"])
    f = Forces(par, terms=["LJ", "Electrostatics", "Bonds", "Angles"], **golden_cfg(g))  # case-insensitive
    pos, box = golden_system_tensors(g, torch.float32, DEV)
    F = torch.zeros_like(pos)
    if DEV != "cpu":  # (test_mirrors_on_interpreter.py runs this function on the host interpreter)
        with pytest.raises(RuntimeError):
            f.compute(pos.cpu(), box.cpu(), F.cpu())  # no CPU path
    with pytest.raises(RuntimeError):
        f.compute(pos, box, F, explicit_forces=False)  # needs requires_grad, like the reference
    t = f.compute(pos, box, F, toNumpy=False)
    assert torch.is_tensor(t) and t.shape == (2,)
    d = f.compute(pos, box, F, returnDetails=True, toNumpy=False)
    assert set(d[0]) == {"lj", "electrostatics", "bonds", "angles", "external"}
    e = f.compute(pos, box, None, calculateForces=False)
    assert abs(e[0] - float(t[0])) < 1e-2

    class Ext:
        def calculate(self, pos, box):
            return torch.full((pos.shape[0],), 2.5, device=pos.device), torch.ones_like(pos)

    fe = Forces(par, terms=["lj"], external=Ext(), **golden_cfg(g))
    F2 = torch.zeros_like(pos)
    d2 = fe.compute(pos, box, F2, returnDetails=True)
    f0 = Forces(par, terms=["lj"], **golden_cfg(g))
    F3 = torch.zeros_like(pos)
    f0.compute(pos, box, F3)
    assert d2[0]["external"] == 2.5 and torch.allclose(F2, F3 + 1.0, atol=1e-5)


def test_nonperiodic_cutoff_with_distinct_replicas():
    """No box (all-zero box: no wrapping, forces.py:361) with a cutoff -- the layout of
    BASELINE.json config 5 (protein in vacuum, several replicas): the cell grid comes from the
    device-side bounding box, every replica has its own positions and its own lists."""
    from torchmd_b200 import Forces

    g = load_golden("water999_eq")
    terms = ["lj", "electrostatics", "bonds", "angles"]
    cfg = dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    nrep = 3
    rng = np.random.default_rng(0)
    base = g["coords"].astype(np.float64)
    coords = np.stack([base + rng.normal(scale=0.02 * r, size=base.shape) + 50.0 * r for r in range(nrep)]).astype(np.float32)
    pos = torch.tensor(coords, device=DEV)
    box = torch.zeros(nrep, 3, 3, device=DEV)
    f = Forces(params_from_golden(g, device=DEV), terms=terms, **cfg)
    F = torch.empty_like(pos)
    E = f.compute(pos, box, F, returnDetails=True)
    st = f.stats()
    assert st["ncells"][0] > 1 and not st["overflow"]

    of32 = refmd.OracleForces(params_from_golden(g), terms, **cfg)
    of64 = refmd.OracleForces(params_from_golden(g, precision=torch.float64), terms, decision_dtype=torch.float32, **cfg)
    F64 = torch.zeros(nrep, len(base), 3, dtype=torch.float64)
    E64 = of64.compute(pos.cpu().double(), box.cpu().double(), F64)
    err = (F.cpu().double() - F64).abs().max().item()
    print(f"non-periodic x{nrep}: max|dF| {err:.3e}, max|F| {F64.abs().max().item():.1f}")
    assert err < force_tol(F64.numpy())
    for r in range(nrep):
        for k in terms:
            assert abs(E[r][k] - E64[r][k]) <= 1e-5 * abs(E64[r][k]) + 2e-3, (r, k)
        ref_pairs = of32.neighbour_pairs(pos[r].cpu(), torch.zeros(3)).numpy().astype(np.int32)
        assert np.array_equal(f.neighbour_pairs(pos, box, replica=r).cpu().numpy(), ref_pairs)
    # moving one replica far away re-grids that replica only; the others stay bitwise the same.
    # (at |x| ~ 1000 A fp32 coordinates carry 6e-5 A, i.e. ~0.1 kcal/mol/A on a stiff O-H bond)
    pos2 = pos.clone()
    pos2[1] += 1000.0
    F2 = torch.empty_like(pos)
    f.compute(pos2, box, F2)
    assert (F2[1] - F[1]).abs().max().item() < 0.5
    from torchmd_b200 import _lib
    if _lib.lib().tmd_pair_kernel(f._ctx) == PAIR_CLUSTER:
        # cluster half list: the partners' forces are summed by reductions at L2, in no fixed order
        tol = 5e-5 * max(1.0, F.abs().max().item() / 100.0)
        assert (F2[0] - F[0]).abs().max().item() < tol and (F2[2] - F[2]).abs().max().item() < tol
    else:
        assert torch.equal(F2[0], F[0]) and torch.equal(F2[2], F[2])


def _lj_coulomb_parameters(n, prec, dev):
    from torchmd_b200.parameters import TopologyParameters

    return TopologyParameters(atom_types=np.zeros(n, int), type_sigma=[1.2], type_epsilon=[0.05], charges=np.where(np.arange(n) % 2, 0.2, -0.2).astype(np.float32),
                              masses=np.full(n, 12.0, np.float32), precision=prec, device=dev)


def test_a_fresh_box_tensor_per_call_is_always_taken():
    """A new box tensor for every call (one per frame of a trajectory, per batch of a data loader): the caching
    allocator hands the same address back with version 0; the upload must not be skipped."""
    from torchmd_b200 import Forces

    n = 120
    rng = np.random.default_rng(5)
    lattice = np.stack(np.meshgrid(*[np.arange(5)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n] * 4.4 + 1.0
    coords = torch.tensor((lattice + rng.normal(0, 0.4, lattice.shape))[None], dtype=torch.float32)
    terms, cfg = ["lj", "electrostatics"], dict(cutoff=9.0, rfa=True, solventDielectric=78.5)
    f = Forces(_lj_coulomb_parameters(n, torch.float32, DEV), terms=terms, **cfg)
    o = refmd.OracleForces(_lj_coulomb_parameters(n, torch.float64, "cpu"), terms, decision_dtype=torch.float32, **cfg)
    p = coords.to(DEV)
    F = torch.zeros_like(p)
    seen = set()
    for L in (22.0, 23.5, 25.0, 22.0):
        box = (torch.eye(3) * L)[None].to(DEV)  # fresh tensor; the previous one was dropped at the end of the last turn
        seen.add(box.data_ptr())
        E = f.compute(p, box, F, returnDetails=True)
        F64 = torch.zeros(1, n, 3, dtype=torch.float64)
        E64 = o.compute(coords.double(), (torch.eye(3, dtype=torch.float64) * L)[None], F64)
        assert float((F.cpu().double() - F64).abs().max()) < force_tol(F64.numpy()), L
        assert abs(E[0]["electrostatics"] - E64[0]["electrostatics"]) < 1e-3, L
        del box
    # (whether the allocator really recycled the address is up to it)


def test_dense_cluster_in_a_large_box_without_the_numpy_outputs():
    """Row capacities are sized from the MEAN density: 240 atoms in a 12 A blob inside a 90 A box overflow them on the
    first build.  The toNumpy=False, autograd and vmap callers must get complete lists too (grown and recomputed)."""
    from torchmd_b200 import Forces

    n = 240
    rng = np.random.default_rng(11)
    g = np.stack(np.meshgrid(*[np.arange(7)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n] * 1.7 + 40.0
    coords = torch.tensor((g + rng.normal(0, 0.05, g.shape))[None], dtype=torch.float32)
    box = (torch.eye(3) * 90.0)[None]
    terms, cfg = ["lj", "electrostatics"], dict(cutoff=9.0, rfa=True, solventDielectric=78.5)
    o = refmd.OracleForces(_lj_coulomb_parameters(n, torch.float64, "cpu"), terms, decision_dtype=torch.float32, **cfg)
    F64 = torch.zeros(1, n, 3, dtype=torch.float64)
    E64 = o.compute(coords.double(), box.double(), F64)
    want = sum(E64[0].values()) if isinstance(E64[0], dict) else float(E64[0])

    f = Forces(_lj_coulomb_parameters(n, torch.float32, DEV), terms=terms, **cfg)
    p, b = coords.to(DEV), box.to(DEV)
    F = torch.zeros_like(p)
    E = f.compute(p, b, F, toNumpy=False)  # first call of a new context, device outputs
    assert not f.stats()["overflow"]  # (grown and recomputed inside the call)
    assert float((F.cpu().double() - F64).abs().max()) < force_tol(F64.numpy())
    assert abs(float(E[0]) - want) < 2e-3 + 1e-5 * abs(want)

    f2 = Forces(_lj_coulomb_parameters(n, torch.float32, DEV), terms=terms, **cfg)
    q = p.clone().requires_grad_(True)
    e = f2.compute(q, b, torch.zeros_like(p), toNumpy=False, explicit_forces=False)  # first call: the autograd path
    e.sum().backward()
    assert float((-q.grad.cpu().double() - F64).abs().max()) < force_tol(F64.numpy())

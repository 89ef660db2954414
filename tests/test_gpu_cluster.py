"""The cluster half-list path (torchmd_b200/csrc/cluster.cuh) on the GPU: parity with the oracle through
Forces.compute / Integrator.step, including the headline size (99,999 atoms) against the row-sampled oracle."""
import numpy as np
import pytest
import torch

from oracle import refmd
from test_simt_cluster import CFG, TERMS, _compute, _oracle, tiled_water
from torchmd_b200._lib import PAIR_CLUSTER, PAIR_ROWS_FX, PAIR_ROWS_FX2

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"


def _L():
    from torchmd_b200 import _lib

    return _lib.lib()


@pytest.mark.parametrize("thrown", [0, 3])
def test_gpu_cluster_periodic_water(thrown):
    sysd = tiled_water(2)
    coords = np.array(sysd["coords"], dtype=np.float32)
    L = float(np.asarray(sysd["box"]).ravel()[0])
    if thrown:
        rng = np.random.default_rng(5)
        sh = rng.integers(-thrown, thrown + 1, size=coords.shape).astype(np.float32)
        coords = coords + sh * (rng.random(len(coords)) < 0.3)[:, None] * np.float32(L)
    system, forces, e = _compute(sysd, coords, None, dev=DEV)
    assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER, "the cluster kernel did not run"
    f64, e_ref, pairs_ref = _oracle(sysd, system)
    pairs = forces.neighbour_pairs(system.pos, system.box).cpu().numpy()
    assert pairs.shape == pairs_ref.shape and np.array_equal(pairs, pairs_ref.astype(np.int32))
    err = (system.forces.cpu().double() - f64).abs().max().item()
    print(f"cluster path, 7992-atom water, thrown={thrown}: max|dF| vs fp64 oracle {err:.3e}")
    assert err < 1e-4, err
    for k in TERMS:
        assert abs(e[k] - e_ref[k]) <= 1e-5 * abs(e_ref[k]) + 2e-3, (k, e[k], e_ref[k])
    # repeated evaluations agree to the summation order of the reductions
    F2 = torch.empty_like(system.forces)
    forces.compute(system.pos, system.box, F2)
    assert (F2 - system.forces).abs().max().item() < 2e-5


def test_gpu_cluster_band_pairs():
    sysd = tiled_water(2)
    coords = np.array(sysd["coords"], dtype=np.float32)
    rng = np.random.default_rng(1)
    for j, k in enumerate(range(300, 3000, 150)):
        a, b = 3 * (k // 3), 3 * ((k + 1200) // 3)
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        r = np.float32(CFG["cutoff"]) * np.float32(1.0 + (j - 9) * 2.0**-23)
        shift = (coords[a].astype(np.float64) + u * float(r)) - coords[b].astype(np.float64)
        coords[b : b + 3] = (coords[b : b + 3].astype(np.float64) + shift).astype(np.float32)
    system, forces, e = _compute(sysd, coords, None, dev=DEV)
    assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    f64, e_ref, pairs_ref = _oracle(sysd, system)
    assert np.array_equal(forces.neighbour_pairs(system.pos, system.box).cpu().numpy(), pairs_ref.astype(np.int32))
    scale = max(1.0, f64.abs().max().item() / 100.0)
    assert (system.forces.cpu().double() - f64).abs().max().item() < 1e-4 * scale
    for k in ("lj", "electrostatics"):
        assert abs(e[k] - e_ref[k]) <= 1e-5 * abs(e_ref[k]) + 2e-3, (k, e[k], e_ref[k])


def test_gpu_cluster_headline_size_against_the_sampled_oracle():
    """BASELINE config 4 itself: 99,999-atom water box after equilibration.  Forces on 600 random atoms from ALL their
    partners (oracle rows, fp64 values on the reference's fp32 decisions): max |dF| < 1e-4 UNSCALED; their in-cutoff
    partner sets bit-exact against tmd_export_pairs."""
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann, testsystems

    sysd = testsystems.water_box(33333, seed=0)
    n = len(sysd["coords"])
    par = testsystems.water_parameters(sysd, device=DEV)
    system = System(n, 1, torch.float32, DEV)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    torch.manual_seed(1)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    cfg = dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    full = Forces(par, terms=["lj", "electrostatics", "bonds", "angles"], **cfg)
    eq = Integrator(system, full, 1.0, DEV, gamma=10.0, T=300.0)
    for _ in range(6):
        eq.step(niter=100)  # lattice start -> liquid (as bench.py does)
    assert _L().tmd_pair_kernel(full._ctx) == PAIR_CLUSTER
    pair_terms = ["lj", "electrostatics"]
    forces = Forces(par, terms=pair_terms, **cfg)
    F = torch.empty_like(system.pos)
    forces.compute(system.pos, system.box, F)
    assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    pairs = forces.neighbour_pairs(system.pos, system.box).cpu().numpy()
    atoms = sorted(np.random.default_rng(7).choice(n, 600, replace=False).tolist())
    par64 = testsystems.water_parameters(sysd, precision=torch.float64)
    pos64 = system.pos[0].cpu().double()
    bd = torch.diagonal(system.box[0]).cpu().double()
    f_ref, partners = refmd.sampled_rows(par64, pair_terms, pos64, bd, atoms, chunk=48, **cfg)
    err = (F[0].cpu().double()[atoms] - f_ref).abs().max().item()
    fmax = f_ref.abs().max().item()
    print(f"99,999-atom water, 600 sampled atoms: max|dF| vs fp64 oracle rows {err:.3e} (max |F| {fmax:.1f}); pairs in cutoff {len(pairs)}")
    assert err < 1e-4, err
    # partner sets of the sampled atoms from the exported pair list
    order = np.argsort(pairs[:, 1], kind="stable")
    by_second = pairs[order]
    for a, ref in zip(atoms[:200], partners[:200]):
        lo = np.searchsorted(pairs[:, 0], a), np.searchsorted(pairs[:, 0], a + 1)
        lo2 = np.searchsorted(by_second[:, 1], a), np.searchsorted(by_second[:, 1], a + 1)
        got = np.sort(np.concatenate([pairs[lo[0] : lo[1], 1], by_second[lo2[0] : lo2[1], 0]]))
        assert np.array_equal(got, ref.numpy().astype(np.int32)), a


def test_gpu_cluster_md_follows_the_full_list_trajectory(monkeypatch):
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann, testsystems

    sysd = tiled_water(2)
    out = []
    for cluster in ("1", "0"):
        monkeypatch.setenv("TMD_B200_CLUSTER", cluster)
        par = testsystems.water_parameters(sysd, device=DEV)
        system = System(len(sysd["coords"]), 1, torch.float32, DEV)
        system.set_positions(np.array(sysd["coords"], dtype=np.float32))
        system.set_box(sysd["box"])
        torch.manual_seed(3)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        forces = Forces(par, terms=TERMS, **CFG, skin=0.3)
        integ = Integrator(system, forces, 1.0, DEV, gamma=None, T=None)
        ekin, pot, temp = integ.step(niter=40)
        st = forces.stats()
        assert _L().tmd_pair_kernel(forces._ctx) == (PAIR_CLUSTER if cluster == "1" else PAIR_ROWS_FX2)
        assert st["rebuilds"] >= 3, st
        out.append((system.pos.clone(), system.vel.clone(), ekin, pot))
    # (40 steps; stiff O-H bonds amplify the 5e-5 force differences of the two summation orders)
    assert (out[0][0] - out[1][0]).abs().max().item() < 1e-3
    assert (out[0][1] - out[1][1]).abs().max().item() < 1e-2
    assert abs(out[0][3][0] - out[1][3][0]) < 1e-5 * abs(out[1][3][0]) + 2e-2


def test_gpu_cluster_capacity_growth_and_fallback(monkeypatch):
    from torchmd_b200 import testsystems

    sysd = tiled_water(2)
    coords = np.array(sysd["coords"], dtype=np.float32)
    monkeypatch.setenv("TMD_B200_CLUSTER_ECAP", "64")
    system, forces, e = _compute(sysd, coords, None, dev=DEV)
    assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    f64, e_ref, _ = _oracle(sysd, system)
    assert (system.forces.cpu().double() - f64).abs().max().item() < 1e-4
    monkeypatch.delenv("TMD_B200_CLUSTER_ECAP")
    lat = testsystems.water_box(1500, seed=0)
    system, forces, e = _compute(lat, np.array(lat["coords"], dtype=np.float32), None, dev=DEV)
    assert _L().tmd_pair_kernel(forces._ctx) in (PAIR_ROWS_FX, PAIR_ROWS_FX2), "expected the fall-back to the full rows"
    f64, e_ref, pairs_ref = _oracle(lat, system)
    assert (system.forces.cpu().double() - f64).abs().max().item() < 1e-4 * max(1.0, f64.abs().max().item() / 100.0)
    assert np.array_equal(forces.neighbour_pairs(system.pos, system.box).cpu().numpy(), pairs_ref.astype(np.int32))

"""The cluster half-list path (torchmd_b200/csrc/cluster.cuh) on the host SIMT interpreter: list build, fixed-point
pair kernel with its exact pass, masked entries, fall-backs.  Logic only (host arithmetic); the device run is
tests/test_gpu_cluster.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import test_simt_kernels as T
from conftest import load_golden
from oracle import refmd
from torchmd_b200._lib import PAIR_CLUSTER, PAIR_ROWS


@pytest.fixture(scope="module")
def simt_cl():
    return T.load(T.build_simt("_cl", T.VARIANTS["_cl"]))


@pytest.fixture
def host_cl(monkeypatch, simt_cl):
    """Forces / Integrator of the package on the interpreter build with the cluster path on (CPU tensors)."""
    from torchmd_b200 import _lib

    class _Stream:
        cuda_stream = None

    monkeypatch.setattr(_lib, "_lib", simt_cl)
    monkeypatch.setattr(_lib, "on_device", lambda t: True)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _Stream())
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return simt_cl


def tiled_water(t=2):
    """The equilibrated 999-atom water box of the goldens repeated t times along every axis: a liquid configuration
    of a box large enough for the cluster path (one image per listed pair)."""
    from torchmd_b200 import testsystems

    g = load_golden("water999_eq")
    c0 = np.asarray(g["coords"], dtype=np.float64)
    L0 = float(np.asarray(g["box"]).ravel()[0])
    cs = [c0 + np.array([a, b, c]) * L0 for a in range(t) for b in range(t) for c in range(t)]
    sysd = testsystems.water_box(333 * t**3, seed=0)
    sysd["coords"] = np.concatenate(cs).astype(np.float32)
    sysd["box"] = np.full_like(np.asarray(sysd["box"]), np.float32(L0 * t))
    return sysd


TERMS = ["lj", "electrostatics", "bonds", "angles"]
CFG = dict(cutoff=5.0, rfa=True, switch_dist=4.0)


def _compute(sysd, coords, handle, dev="cpu", **kw):
    from torchmd_b200 import Forces, System, testsystems

    par = testsystems.water_parameters(sysd, device=dev)
    system = System(len(coords), 1, torch.float32, dev)
    system.set_positions(coords)
    system.set_box(sysd["box"])
    forces = Forces(par, terms=TERMS, **CFG, **kw)
    e = forces.compute(system.pos, system.box, system.forces, returnDetails=True)[0]
    return system, forces, e


def _oracle(sysd, system):
    from torchmd_b200 import testsystems

    par64 = testsystems.water_parameters(sysd, precision=torch.float64)
    of = refmd.OracleForces(par64, TERMS, decision_dtype=torch.float32, **CFG)
    pos64 = system.pos.cpu().double()
    f64 = torch.zeros_like(pos64)
    e_ref = of.compute(pos64, system.box.cpu().double(), f64)[0]
    par32 = testsystems.water_parameters(sysd, precision=torch.float32)
    pairs = refmd.OracleForces(par32, TERMS, **CFG).neighbour_pairs(system.pos[0].cpu(), torch.diagonal(system.box[0]).cpu()).numpy()
    return f64, e_ref, pairs


@pytest.mark.parametrize("thrown", [0, 3])
def test_cluster_path_periodic_water(host_cl, thrown):
    """Pairs bit-exact, forces and energies against the fp64 oracle; `thrown`: single atoms (not molecules) moved by up to
    that many box lengths, so that clusters mix image counts and every separation needs the wrap."""
    sysd = tiled_water(2)
    coords = np.array(sysd["coords"], dtype=np.float32)
    L = float(np.asarray(sysd["box"]).ravel()[0])
    if thrown:
        rng = np.random.default_rng(5)
        sh = rng.integers(-thrown, thrown + 1, size=coords.shape).astype(np.float32)
        coords = coords + sh * (rng.random(len(coords)) < 0.3)[:, None] * np.float32(L)
    system, forces, e = _compute(sysd, coords, host_cl)
    assert host_cl.tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER, "the cluster kernel did not run"
    f64, e_ref, pairs_ref = _oracle(sysd, system)
    pairs = forces.neighbour_pairs(system.pos, system.box).numpy()
    assert pairs.shape == pairs_ref.shape and np.array_equal(pairs, pairs_ref.astype(np.int32))
    err = (system.forces.double() - f64).abs().max().item()
    assert err < 1e-4, err
    for k in TERMS:
        assert abs(e[k] - e_ref[k]) <= 1e-5 * abs(e_ref[k]) + 2e-3, (k, e[k], e_ref[k])


def test_cluster_exact_pass_decides_band_pairs(host_cl):
    """Pairs placed within a few ulp of the cutoff on both sides: the band pass must give the reference's decisions."""
    sysd = tiled_water(2)
    coords = np.array(sysd["coords"], dtype=np.float32)
    # move oxygen k next to oxygen 0 of a far-away molecule at distance cutoff * (1 +- j * 2^-23)
    rng = np.random.default_rng(1)
    n = len(coords)
    for j, k in enumerate(range(300, 3000, 150)):
        a = 3 * (k // 3)
        b = 3 * ((k + 1200) // 3)
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        r = np.float32(CFG["cutoff"]) * np.float32(1.0 + (j - 9) * 2.0**-23)
        shift = (coords[a].astype(np.float64) + u * float(r)) - coords[b].astype(np.float64)
        coords[b : b + 3] = (coords[b : b + 3].astype(np.float64) + shift).astype(np.float32)
    system, forces, e = _compute(sysd, coords, host_cl)
    assert host_cl.tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    f64, e_ref, pairs_ref = _oracle(sysd, system)
    pairs = forces.neighbour_pairs(system.pos, system.box).numpy()
    assert np.array_equal(pairs, pairs_ref.astype(np.int32))
    scale = max(1.0, f64.abs().max().item() / 100.0)  # (the moved molecules overlap their new neighbours)
    assert (system.forces.double() - f64).abs().max().item() < 1e-4 * scale
    for k in ("lj", "electrostatics"):
        assert abs(e[k] - e_ref[k]) <= 1e-5 * abs(e_ref[k]) + 2e-3, (k, e[k], e_ref[k])


@pytest.mark.parametrize("name", ["ala2_nobox_rf", "thrombin_nobox_rf"])
def test_cluster_path_without_a_box(simt_cl, name):
    """No box: the reference's float chain in packed operations; many atom types and exclusions (thrombin: 45 types)."""
    g = load_golden(name)
    c = T.Ctx(simt_cl, g)
    F, E = c.forces()
    assert simt_cl.tmd_pair_kernel(c.h) == PAIR_CLUSTER
    T.check_against_golden(c, F, E)
    F2, _ = c.forces(energies=False)
    T.check_against_golden(c, F2, {})
    if "pairs_f32" in g:
        assert np.array_equal(c.pairs(), g["pairs_f32"])
    c.close()


def test_cluster_list_capacity_grows_and_lattice_falls_back(host_cl, monkeypatch):
    """A list that overflows its reserved entries is regrown and rebuilt; a system whose clusters get too long for the box
    (a jittered lattice: sparse cell rows) drops to the full Verlet rows -- same results either way."""
    from torchmd_b200 import testsystems

    sysd = tiled_water(2)
    coords = np.array(sysd["coords"], dtype=np.float32)
    monkeypatch.setenv("TMD_B200_CLUSTER_ECAP", "64")  # start far too small
    system, forces, e = _compute(sysd, coords, host_cl)
    assert host_cl.tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    f64, e_ref, _ = _oracle(sysd, system)
    assert (system.forces.double() - f64).abs().max().item() < 1e-4
    monkeypatch.delenv("TMD_B200_CLUSTER_ECAP")
    lat = testsystems.water_box(1500, seed=0)  # lattice start, 35.5 A box: some cell rows hold only a few atoms
    system, forces, e = _compute(lat, np.array(lat["coords"], dtype=np.float32), host_cl)
    assert host_cl.tmd_pair_kernel(forces._ctx) == PAIR_ROWS, "expected the fall-back to the full rows"
    f64, e_ref, pairs_ref = _oracle(lat, system)
    assert (system.forces.double() - f64).abs().max().item() < 1e-4 * max(1.0, f64.abs().max().item() / 100.0)
    assert np.array_equal(forces.neighbour_pairs(system.pos, system.box).numpy(), pairs_ref.astype(np.int32))


def test_cluster_md_steps_follow_the_full_list_trajectory(host_cl, monkeypatch):
    """Fused MD steps with rebuilds inside the run: the cluster path and the full-row path give the same trajectory up to
    the summation order of the forces."""
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann, testsystems

    sysd = tiled_water(2)
    out = []
    for cluster in ("1", "0"):
        monkeypatch.setenv("TMD_B200_CLUSTER", cluster)
        par = testsystems.water_parameters(sysd, device="cpu")
        system = System(len(sysd["coords"]), 1, torch.float32, "cpu")
        system.set_positions(np.array(sysd["coords"], dtype=np.float32))
        system.set_box(sysd["box"])
        torch.manual_seed(3)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        forces = Forces(par, terms=TERMS, **CFG, skin=0.3)
        integ = Integrator(system, forces, 1.0, "cpu", gamma=None, T=None)
        ekin, pot, temp = integ.step(niter=12)
        st = forces.stats()
        assert host_cl.tmd_pair_kernel(forces._ctx) == (PAIR_CLUSTER if cluster == "1" else PAIR_ROWS)
        assert st["rebuilds"] >= 2, st
        out.append((system.pos.clone(), system.vel.clone(), ekin, pot))
    # (stiff O-H bonds, 900 kcal/mol/A^2, turn a 4e-6 A difference in position into 3e-3 in force and 7e-5 in velocity)
    assert (out[0][0] - out[1][0]).abs().max().item() < 5e-5
    assert (out[0][1] - out[1][1]).abs().max().item() < 5e-4
    assert abs(out[0][3][0] - out[1][3][0]) < 1e-5 * abs(out[1][3][0]) + 5e-3


@pytest.mark.parametrize("graph", ["0", "1"])
def test_step_boundary_kernel_reproduces_the_two_kernel_sequence(host_cl, monkeypatch, graph):
    """TMD_B200_FUSESTEP: the second half of a step and the first half of the next in one kernel (k_cstep_boundary), with
    the Langevin draws of the step it closes -- the same trajectory, bit for bit, as second-half kernel + first-half
    kernel (the interpreter sums in a fixed order), through rebuilds, eagerly issued and as captured steps."""
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann, testsystems

    sysd = tiled_water(2)
    monkeypatch.setenv("TMD_B200_GRAPH", graph)
    out = []
    for fuse in ("1", "0"):
        monkeypatch.setenv("TMD_B200_FUSESTEP", fuse)
        par = testsystems.water_parameters(sysd, device="cpu")
        system = System(len(sysd["coords"]), 1, torch.float32, "cpu")
        system.set_positions(np.array(sysd["coords"], dtype=np.float32))
        system.set_box(sysd["box"])
        torch.manual_seed(3)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        forces = Forces(par, terms=TERMS, **CFG, skin=0.3)
        integ = Integrator(system, forces, 1.0, "cpu", gamma=0.5, T=300.0)
        l0 = 0
        res = []
        for niter in (1, 2, 7):  # one step (no boundary), first+last, first+middle+last
            ekin, pot, temp = integ.step(niter=niter)
            res.append((float(ekin[0]), float(pot[0])))
        st = forces.stats()
        assert host_cl.tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER and st["rebuilds"] >= 2, st
        out.append((system.pos.clone(), system.vel.clone(), system.forces.clone(), res, st["kernel_launches"]))
    if os.environ.get("SIMT_SCHEDULE"):
        # another thread order: the partner forces are summed by reductions in whatever order the warps run, so even two
        # runs of the SAME configuration differ at the fp32 summation level (dpos 4e-6, dvel 2e-4 after 10 steps)
        assert (out[0][0] - out[1][0]).abs().max() < 5e-5 and (out[0][1] - out[1][1]).abs().max() < 2e-3
    else:
        assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]) and torch.equal(out[0][2], out[1][2])
        assert out[0][3] == out[1][3]
    assert out[0][4] < out[1][4]  # fewer launches


@pytest.mark.parametrize("seed", [108, 109])
def test_cluster_fuzz_sample(host_cl, seed):
    """Two seeds of scripts/fuzz_cluster.py that take the cluster path: an open system with bonds inside and across
    clusters, and two replicas of a periodic box with atoms whole boxes away -- first evaluation, list reuse, rebuild."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("fuzz_cluster", os.path.join(T.ROOT, "scripts", "fuzz_cluster.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ok, kern, desc = mod.one(seed)
    assert kern == 4 and ok, desc


def test_cluster_path_with_owned_atom_ranges(host_cl):
    """Decomposed runs: a context that owns a range of atoms builds lists only for the pairs that touch an owned atom;
    its forces on the owned atoms are the full forces, and the ranks' energy shares add up to the total."""
    from torchmd_b200 import Forces, System, _lib, testsystems

    sysd = tiled_water(2)
    coords = np.array(sysd["coords"], dtype=np.float32)
    system, forces, e_full = _compute(sysd, coords, host_cl)
    assert host_cl.tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    F_full = system.forces.clone()
    n = len(coords)
    world = 3
    chunk = -(-n // world)
    e_sum = {k: 0.0 for k in TERMS}
    for rank in range(world):
        lo, hi = rank * chunk, min(n, (rank + 1) * chunk)
        par = testsystems.water_parameters(sysd, device="cpu")
        s2 = System(n, 1, torch.float32, "cpu")
        s2.set_positions(coords)
        s2.set_box(sysd["box"])
        f2 = Forces(par, terms=TERMS, **CFG)
        ctx = f2._ensure_ctx(s2.pos)
        f2._ensure_box(s2.box)
        _lib.check(host_cl.tmd_set_owned_atoms(ctx, lo, hi - lo))
        e = f2.compute(s2.pos, s2.box, s2.forces, returnDetails=True)[0]
        assert host_cl.tmd_pair_kernel(ctx) == PAIR_CLUSTER
        assert (s2.forces[0, lo:hi] - F_full[0, lo:hi]).abs().max().item() < 3e-5
        for k in TERMS:
            e_sum[k] += e[k]
    for k in TERMS:
        assert abs(e_sum[k] - e_full[k]) <= 1e-6 * abs(e_full[k]) + 2e-3, (k, e_sum[k], e_full[k])

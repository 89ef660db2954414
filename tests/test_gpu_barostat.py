"""The Monte Carlo barostat (Integrator(..., barostat=MonteCarloBarostat(...))) on the GPU.

* an ideal gas against its analytic volume distribution, p(V) ~ V^N exp(-beta P V);
* the fast box path against a context finalised at the same box, at production size;
* a rejected move restores the state bitwise;
* the captured steps survive a run of moves without recapturing, at the same launches per step;
* rigid TIP3P water at 1 bar reaches a liquid density (no dispersion correction: not a literature comparison);
* replicas keep their own boxes and influence functions.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _water(nw, dtype, seed=0):
    from torchmd_b200 import testsystems

    sysd = testsystems.water_box(nw, seed=seed)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    return sysd, par


def _system(sysd, par, dtype, nrep=1, T=300.0):
    from torchmd_b200 import System, maxwell_boltzmann

    n = len(sysd["coords"])
    s = System(n, nrep, dtype, DEV)
    s.set_positions(np.repeat(np.asarray(sysd["coords"])[:, :, None], nrep, axis=2))
    s.set_box(np.repeat(np.asarray(sysd["box"]).reshape(3, 1), nrep, axis=1))
    s.set_velocities(maxwell_boltzmann(par.masses, T, nrep))
    return s


def _block_se(x, nblocks=20):
    b = np.array_split(np.asarray(x), nblocks)
    m = np.array([bb.mean() for bb in b])
    return m.std(ddof=1) / math.sqrt(nblocks)


def test_ideal_gas_volume_distribution():
    """N non-interacting atoms: <V> = (N+1) kT / P, Var V = (N+1) (kT / P)^2, within 4 block-averaged standard errors,
    on 2 replicas with different seeds."""
    from torchmd_b200 import Forces, Integrator, MonteCarloBarostat, System
    from torchmd_b200.barostat import BAR_TO_KCAL_PER_MOL_A3, BOLTZMAN
    from torchmd_b200.parameters import TopologyParameters

    torch.manual_seed(3)
    N, T, L0 = 100, 300.0, 50.0
    kT = BOLTZMAN * T
    P_bar = (N + 1) * kT / L0**3 / BAR_TO_KCAL_PER_MOL_A3
    par = TopologyParameters(atom_types=np.zeros(N, np.int64), type_sigma=[3.0], type_epsilon=[0.0], charges=np.zeros(N),
                             masses=np.full(N, 40.0), precision=torch.float64, device=DEV)
    rng = np.random.default_rng(0)
    s = System(N, 2, torch.float64, DEV)
    s.set_positions(rng.uniform(0, L0, (N, 3, 2)))
    s.set_box(np.full((3, 2), L0))
    f = Forces(par, terms=["lj"], cutoff=5.0)
    vols = [[], []]
    bar = MonteCarloBarostat(pressure=P_bar, frequency=1, seed=17)
    integ = Integrator(s, f, 1.0, DEV, gamma=1.0, T=T, barostat=bar)
    integ.step(500)  # equilibration
    for _ in range(8000):
        integ.step(1)
        V = torch.prod(torch.diagonal(s.box, dim1=1, dim2=2), dim=1).cpu().numpy()
        for r in range(2):
            vols[r].append(V[r])
    mean_want = (N + 1) * kT / (P_bar * BAR_TO_KCAL_PER_MOL_A3)
    var_want = (N + 1) * (kT / (P_bar * BAR_TO_KCAL_PER_MOL_A3)) ** 2
    for r in range(2):
        v = np.asarray(vols[r])
        se_m = _block_se(v)
        se_v = _block_se((v - v.mean()) ** 2)
        print(f"[ideal gas] replica {r}: <V> {v.mean():.1f} (want {mean_want:.1f} +- {se_m:.1f}), Var {v.var():.4g} "
              f"(want {var_want:.4g} +- {se_v:.3g}), stats {bar.stats()[r]}")
        assert abs(v.mean() - mean_want) <= 4 * se_m
        assert abs(v.var() - var_want) <= 4 * se_v
    assert vols[0][-1] != vols[1][-1]


def _fast_vs_fresh(nw, dtype, s):
    from torchmd_b200 import Forces, _lib
    from torchmd_b200.barostat import molecule_trees

    sysd, par = _water(nw, dtype)
    terms = ["lj", "electrostatics", "bonds", "angles"]
    cfg = dict(cutoff=9.0, switch_dist=7.5, pme=True)
    f = Forces(par, terms=terms, **cfg)
    pos = torch.tensor(np.asarray(sysd["coords"])[None], dtype=dtype, device=DEV)
    L0 = np.asarray(sysd["box"], np.float64).reshape(1, 3)
    box = torch.diag_embed(torch.tensor(L0, dtype=dtype, device=DEV))
    F = torch.zeros_like(pos)
    f.compute(pos, box, F)
    kernel0 = _lib.lib().tmd_pair_kernel(f._ctx)
    ptr, atoms, parent = molecule_trees(pos.shape[1], par.bond_params["idx"].cpu().numpy())
    L = _lib.lib()
    _lib.check(L.tmd_set_molecules(f._ctx, len(ptr) - 1, ptr.ctypes.data, atoms.ctypes.data, parent.ctypes.data))
    npd = np.float64 if dtype == torch.float64 else np.float32
    new = (L0 * s).astype(npd).astype(np.float64)
    scale = torch.tensor(new / L0, dtype=torch.float64, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    sfx = "_f64" if dtype == torch.float64 else ""
    _lib.check(getattr(L, "tmd_scale_molecules" + sfx)(f._ctx, pos.data_ptr(), scale.data_ptr(), stream))
    host = np.ascontiguousarray(new, dtype=npd)
    _lib.check(getattr(L, "tmd_rescale_box" + sfx)(f._ctx, host.ctypes.data, stream))
    idx = torch.arange(3, device=DEV)
    box[:, idx, idx] = torch.as_tensor(host).to(DEV)
    f._box_key = (box.data_ptr(), box._version, tuple(box.shape), tuple(box.stride()), box.dtype)
    f._box_ref = box
    E1 = f.compute(pos, box, F, returnDetails=True)[0]
    g = Forces(par, terms=terms, **cfg)
    F2 = torch.zeros_like(pos)
    E2 = g.compute(pos, box.clone(), F2, returnDetails=True)[0]
    assert f.pme_parameters() == g.pme_parameters()
    return kernel0, _lib.lib().tmd_pair_kernel(f._ctx), E1, E2, F, F2


@pytest.mark.parametrize("nw,dtype,s", [(33333, torch.float32, 1.005), (3333, torch.float64, 1.005), (3333, torch.float64, 0.995)])
def test_fast_path_equals_a_fresh_context(nw, dtype, s):
    k0, k1, E1, E2, F1, F2 = _fast_vs_fresh(nw, dtype, s)
    assert k0 == k1
    if dtype == torch.float32:
        assert k1 == 10  # k_cpair_ew
    rel, fa = (1e-12, 1e-9) if dtype == torch.float64 else (2e-5, 5e-4)
    for k in E1:
        assert abs(E1[k] - E2[k]) <= rel * max(1.0, abs(E2[k])), (k, E1[k], E2[k])
    err = (F1.double() - F2.double()).abs().max().item()
    print(f"[fast == fresh] nw {nw} {dtype} s {s}: max |dF| {err:.3e}, dE_elec {E1['electrostatics'] - E2['electrostatics']:.3e}")
    assert err <= fa


def _npt(nw, dtype, nrep=1, frequency=25, constraints=False, seed=0, gamma=1.0, pme=True):
    from torchmd_b200 import Constraints, Forces, Integrator, MonteCarloBarostat

    torch.manual_seed(seed)
    sysd, par = _water(nw, dtype)
    s = _system(sysd, par, dtype, nrep)
    f = Forces(par, terms=["lj", "electrostatics", "bonds", "angles"], cutoff=9.0, switch_dist=7.5, pme=pme)
    bar = MonteCarloBarostat(pressure=1.0, frequency=frequency)
    con = Constraints(par, "water") if constraints else None
    integ = Integrator(s, f, 2.0 if constraints else 1.0, DEV, gamma=gamma, T=300.0, constraints=con, barostat=bar)
    return s, f, bar, integ


def test_rejection_then_steps_match_a_run_without_the_move():
    """fp64: a forced rejection at step 25, then 10 steps, against the same run whose barostat has no move due."""
    s, f, bar, integ = _npt(1000, torch.float64, frequency=25)
    s2, f2, bar2, integ2 = _npt(1000, torch.float64, frequency=10**6)
    assert integ.seed == integ2.seed
    bar.uniforms = lambda r, k: (0.9, math.inf)  # a trial expansion, rejected whatever its energy
    integ.step(25)
    integ2.step(25)
    assert bar.stats()[0]["attempted"] == 1 and bar.stats()[0]["accepted"] == 0
    for k in ("pos", "vel", "forces", "box"):
        assert torch.equal(getattr(s, k), getattr(s2, k)), k
    integ.step(10)
    integ2.step(10)
    err = (s.pos - s2.pos).abs().max().item()
    print(f"[reject] 10 fp64 steps after a rejected move: max |dx| {err:.3e} A")
    assert err <= 1e-9


def test_rejected_move_leaves_pos_vel_forces_box_untouched():
    s, f, bar, integ = _npt(1000, torch.float32, frequency=5)
    integ.step(4)
    bar.uniforms = lambda r, k: (0.1, math.inf)
    # the state after the fifth step, before its move: rerun that step on a copy of the integrator's inputs
    integ.barostat, keep = None, bar
    integ.step(1)
    before = {k: getattr(s, k).clone() for k in ("pos", "vel", "forces", "box")}
    integ.barostat = keep
    integ._step_index = 5
    ene = integ._out[1]
    keep.attempt(f._ensure_ctx(s.pos), ene)
    for k, v in before.items():
        assert torch.equal(v, getattr(s, k)), k


def test_captures_and_launches_over_a_run_of_moves():
    from torchmd_b200 import _lib

    s, f, bar, integ = _npt(3000, torch.float32, frequency=25, constraints=True)
    # past the first rescale, the lattice start's melting (the cluster lists refuse a lattice and are retried after 1000
    # and 2000 more force calls, each a re-finalisation) and the density's settling (list capacities grow with it)
    integ.step(4000)
    L = _lib.lib()
    caps = L.tmd_step_captures(f._ctx)
    full0 = bar.stats()[0]["full_box_changes"]
    st0 = f.stats()
    integ.step(2000)
    st1 = f.stats()
    b = bar.stats()[0]
    assert L.tmd_step_captures(f._ctx) == caps, (caps, L.tmd_step_captures(f._ctx), b)
    assert b["attempted"] == 240 and b["full_box_changes"] == full0, b
    # the steps between two moves launch what the same steps launch without a barostat
    a = f.stats()["kernel_launches"]
    integ.step(24)  # (the step index is a multiple of 25: no move is due in these 24 steps)
    npt_steps = f.stats()["kernel_launches"] - a
    from torchmd_b200 import Integrator

    integ_nvt = Integrator(s, f, 2.0, DEV, gamma=1.0, T=300.0, constraints=integ.constraints)
    integ_nvt.step(1)
    a = f.stats()["kernel_launches"]
    integ_nvt.step(24)
    nvt_steps = f.stats()["kernel_launches"] - a
    print(f"[launches] 24 steps: NPT {npt_steps}, NVT {nvt_steps}; the NPT window {(st1['kernel_launches'] - st0['kernel_launches']) / 2000:.2f} "
          f"per step incl. 80 moves; captures {caps}; barostat {b}")
    assert npt_steps == nvt_steps


def test_rigid_water_density_at_one_bar():
    """Rigid TIP3P water10k with PME at 300 K, 1 bar, 2 fs, Langevin, fp32: 50 ps."""
    s, f, bar, integ = _npt(3333, torch.float32, frequency=25, constraints=True)
    mass = float(f.par.masses.sum().item())  # amu
    res = []
    for _ in range(25):
        integ.step(1000)
        V = float(torch.prod(torch.diagonal(s.box[0])).item())
        res.append(mass / V * 1.66053906660)  # amu/A^3 -> g/cm^3
    b = bar.stats()[0]
    rate = b["accepted"] / b["attempted"]
    print(f"[density] rigid TIP3P 3333 waters, PME, 300 K, 1 bar, 50 ps: density trace {np.round(res, 4).tolist()}, "
          f"final {res[-1]:.4f} g/cm^3, mean of the last 25 ps {np.mean(res[12:]):.4f}; acceptance {rate:.3f}; {b}")
    assert 0.95 <= res[-1] <= 1.05
    assert 0.25 <= rate <= 0.75


def test_replicas_keep_their_own_boxes():
    """Two replicas, one move where replica 0 accepts and replica 1 rejects: each keeps its own box, and the PME energy
    of each equals that of a fresh context at its box."""
    from torchmd_b200 import Forces

    s, f, bar, integ = _npt(3333, torch.float32, nrep=2, frequency=10)
    integ.step(9)
    box0 = s.box.clone()
    bar.uniforms = lambda r, k: (0.5 + 0.2, 0.0) if r == 0 else (0.2, math.inf)
    _, pot, _ = integ.step(1)
    b = bar.stats()
    assert b[0]["accepted"] == 1 and b[1]["accepted"] == 0
    assert not torch.equal(s.box[0], box0[0]) and torch.equal(s.box[1], box0[1])
    g = Forces(f.par, terms=f.energies, cutoff=9.0, switch_dist=7.5, pme=True)
    e = g.compute(s.pos, s.box.clone(), torch.zeros_like(s.pos))
    for r in range(2):
        assert abs(e[r] - pot[r]) <= 2e-5 * abs(e[r]), (r, e[r], pot[r])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_constraint_residuals_after_every_move_and_step(dtype, nsteps=300):
    """Rigid water10k at 2 fs, a move every 5 steps: the bounds of test_gpu_constraints.test_residuals_every_step hold
    after every step, the moves included."""
    from oracle import constraints as OC

    s, f, bar, integ = _npt(3333, dtype, frequency=5, constraints=True)
    groups = OC.groups_of(integ.constraints)
    worst = 0.0
    for _ in range(nsteps):
        integ.step(1)
        box = torch.diagonal(s.box, dim1=-2, dim2=-1).cpu().double().numpy()
        er, ev = OC.residuals(s.pos.cpu().double().numpy(), s.vel.cpu().double().numpy(), groups, box)
        worst = max(worst, er)
        if dtype == torch.float32:
            assert er <= 2 * float(np.spacing(np.float32(s.pos.abs().max().item()))), er
            assert ev <= 1e-6, ev
        else:
            assert er <= 1e-10 and ev <= 1e-12, (er, ev)
    b = bar.stats()[0]
    print(f"[constraints] {dtype}: worst |r-d| {worst:.3e} A over {nsteps} steps with {b['attempted']} moves ({b['accepted']} accepted)")
    assert b["attempted"] == nsteps // 5 and b["accepted"] > 0

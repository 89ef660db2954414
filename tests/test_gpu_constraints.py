"""Rigid water and X-H constraints (Integrator(..., constraints=...)) on the GPU.

Bounds, derived from rounding rather than measured:
* residuals: the kernels solve every group in fp64 to |r - d| <= 5e-15 d and round each coordinate once, so a
  constrained distance in fp32 is off by at most the rounding of its two end points, 2 * ulp(max |coordinate|)/2
  each; velocities are rounded once from an exact fp64 projection, so the relative velocity along a bond is
  bounded by |v| * 2^-23 ~ 1e-7 for |v| ~ 1 A/tu (bound 1e-6).  In fp64 the same reasoning gives ~1e-13 A
  (bound 1e-10 A) and ~1e-16 A/tu (bound 1e-12).
* trajectories against the fp64 oracle (oracle/constraints.py, Newton on the multipliers): fp64 runs differ
  by reordered sums only, 1e-9 after 20 steps; fp32 runs keep the bounds of the unconstrained fused-step test
  (test_gpu_integrator.test_langevin_with_injected_noise_matches_reference: 2e-5 A, 5e-5 A/tu after 4 steps).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TERMS = ["lj", "electrostatics", "bonds", "angles"]
CFG = dict(cutoff=9.0, rfa=True, switch_dist=7.5)


def _water(nw, dtype, seed=0, hh=False, nrep=1, kind="water"):
    from torchmd_b200 import Constraints, Forces, System, testsystems

    sysd = testsystems.water_box(nw, seed=seed, hh_bonds=hh)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    system = System(len(sysd["coords"]), nrep, dtype, DEV)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    forces = Forces(par, terms=TERMS, **CFG)
    return sysd, par, system, forces, Constraints(par, kind)


def _groups(con):
    from oracle import constraints as OC

    return OC.groups_of(con)


def _residuals(system, con):
    from oracle import constraints as OC

    box = torch.diagonal(system.box, dim1=-2, dim2=-1).cpu().double().numpy()
    return OC.residuals(system.pos.cpu().double().numpy(), system.vel.cpu().double().numpy(), _groups(con), box)


def _ulp32(x):
    return float(np.spacing(np.float32(x)))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_residuals_every_step(dtype, nw=3333, nsteps=1000):
    """Water at 2 fs with Langevin: every constraint holds after every step."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    sysd, par, system, forces, con = _water(nw, dtype)
    torch.manual_seed(0)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    integ = Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con)
    worst_r, worst_v = 0.0, 0.0
    for _ in range(nsteps):
        integ.step(1)
        er, ev = _residuals(system, con)
        worst_r, worst_v = max(worst_r, er), max(worst_v, ev)
        if dtype == torch.float32:
            assert er <= 2 * _ulp32(system.pos.abs().max().item()), er
            assert ev <= 1e-6, ev
        else:
            assert er <= 1e-10 and ev <= 1e-12, (er, ev)
    print(f"{dtype}: worst |r-d| {worst_r:.3e} A, worst |v_rel . r_hat| {worst_v:.3e} A/tu over {nsteps} steps")


def _oracle_run(system0, par64, con, terms, cfg, nsteps, noise, dt_fs, gamma, T, decision_dtype):
    from oracle import constraints as OC
    from oracle import refmd

    of = refmd.OracleForces(par64, terms, decision_dtype=decision_dtype, **cfg)
    pos = system0["pos"].clone()
    vel = system0["vel"].clone()
    box = system0["box"].clone()
    f = torch.zeros_like(pos)
    of.compute(pos, box, f)
    oi = OC.OracleConstrainedIntegrator(pos, vel, box, f, par64.masses, of.compute, dt_fs, _groups(con), gamma_ps=gamma, T=T)
    oi.project()
    ek, _ = oi.step(nsteps, noise=noise)
    return pos, vel, ek


def _random_rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


def _trajectory_case(dtype, name, kind, nsteps, nrep=1, seed=0, thermostat=True):
    """GPU run against the oracle's fp64 RATTLE integrator on the oracle's forces: with injected noise (the step-by-step
    launches of tmd_md_steps), or without a thermostat (the captured step graphs in fp32).  A name ending in "_rot" is
    the system turned by a random rotation about its centre (a system without a box: a turned periodic box would overlap
    its images)."""
    from torchmd_b200 import Constraints, Forces, Integrator, System, maxwell_boltzmann, testsystems

    if name.startswith("water"):
        nw = int(name[5:])
        sysd = testsystems.water_box(nw, seed=seed)
        par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
        par64 = testsystems.water_parameters(sysd, precision=torch.float64)
        coords, boxv, terms, cfg = sysd["coords"], sysd["box"], TERMS, CFG
    else:
        base = name[:-4] if name.endswith("_rot") else name
        par, coords, boxv, terms, cfg = testsystems.golden_system(base, precision=dtype, device=DEV)
        par64 = testsystems.golden_system(base, precision=torch.float64)[0]
    n = len(coords)
    system = System(n, nrep, dtype, DEV)
    rng = np.random.default_rng(seed)
    if name.endswith("_rot"):
        c = np.asarray(coords, np.float64)
        coords = ((c - c.mean(0)) @ _random_rotation(rng).T + c.mean(0)).astype(np.float32)
    x = np.repeat(np.asarray(coords, np.float64)[None], nrep, 0)
    if nrep > 1:  # replicas in different configurations: each one moved by whole boxes and jittered
        x[1:] += rng.normal(0, 0.02, x[1:].shape)
        if np.all(boxv > 0):
            x[1:] += rng.integers(-3, 4, size=(nrep - 1, n, 3)) * boxv
    system.set_positions(torch.tensor(x, dtype=dtype).permute(1, 2, 0))
    system.set_box(np.asarray(boxv))
    forces = Forces(par, terms=terms, **cfg)
    con = Constraints(par, kind)
    torch.manual_seed(seed)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, nrep))
    noise = torch.randn((nsteps, nrep, n, 3), dtype=torch.float64, generator=torch.Generator().manual_seed(seed + 1)) \
        if thermostat else None
    forces.compute(system.pos, system.box, system.forces)  # the first half-kick uses the start forces, as the oracle's
    start = {k: getattr(system, k).cpu().double().clone() for k in ("pos", "vel", "box")}
    if thermostat:
        integ = Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con)
        integ.step(nsteps, noise=noise.to(dtype))
    else:
        Integrator(system, forces, 2.0, DEV, constraints=con).step(nsteps)
    dec = torch.float32 if dtype == torch.float32 else torch.float64
    pos, vel, _ = _oracle_run(start, par64, con, terms, cfg, nsteps, noise, 2.0, 1.0 if thermostat else None,
                              300.0 if thermostat else None, dec)
    dp = (system.pos.cpu().double() - pos).abs().max().item()
    dv = (system.vel.cpu().double() - vel).abs().max().item()
    return dp, dv, system, con


@pytest.mark.parametrize("name,kind,nrep", [("water300", "water", 1), ("water300", "water", 3), ("ala2_xsc_rf", "hbonds", 1),
                                            ("ala2_nobox_rf_rot", "hbonds", 1), ("thrombin_nobox_rf", "hbonds", 1)])
def test_trajectory_against_oracle_f64(name, kind, nrep):
    dp, dv, system, con = _trajectory_case(torch.float64, name, kind, 20, nrep)
    print(f"{name} {kind} x{nrep} fp64 20 steps: dpos {dp:.2e} dvel {dv:.2e}")
    assert dp < 1e-9 and dv < 1e-9


@pytest.mark.parametrize("name,kind", [("water300", "water"), ("ala2_xsc_rf", "hbonds")])
def test_trajectory_against_oracle_f32(name, kind):
    dp, dv, system, con = _trajectory_case(torch.float32, name, kind, 4)
    print(f"{name} {kind} fp32 4 steps: dpos {dp:.2e} dvel {dv:.2e}")
    assert dp < 2e-5 and dv < 5e-5


@pytest.mark.parametrize("name,kind", [("water300", "water"), ("ala2_xsc_rf", "hbonds")])
def test_captured_step_against_oracle_f32(name, kind):
    """NVE without injected noise: tmd_md_steps replays its captured step graphs (the fused position constraint and
    preparation, the folding second kick, the velocity constraint); same bounds as the noisy fp32 case."""
    dp, dv, system, con = _trajectory_case(torch.float32, name, kind, 4, thermostat=False)
    print(f"{name} {kind} fp32 4 captured NVE steps: dpos {dp:.2e} dvel {dv:.2e}")
    assert dp < 2e-5 and dv < 5e-5


def test_integrators_sharing_one_forces():
    """The constraint tables live in the Forces object's context: an unconstrained integrator on the same Forces runs
    unconstrained, and integrators with different Constraints each run their own -- each equal to a run on a fresh Forces."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    from torchmd_b200 import Constraints, Forces, testsystems

    sysd, par, system, shared, con_w = _water(100, torch.float64, hh=True)  # H-H distance from the H-H bond: 1.5139 A
    # the same waters with the H-H distance from the angle term (1.51390065 A): other tables, other trajectory
    con_h = Constraints(testsystems.water_parameters(testsystems.water_box(100), precision=torch.float64), "water")
    assert con_h.water_d[0, 1] != con_w.water_d[0, 1]
    torch.manual_seed(2)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    shared.compute(system.pos, system.box, system.forces)
    start = [t.clone() for t in (system.pos, system.vel, system.forces)]

    def run(forces, con):
        for t, s0 in zip((system.pos, system.vel, system.forces), start):
            t.copy_(s0)
        _, _, T = Integrator(system, forces, 1.0, DEV, constraints=con).step(5)
        return system.pos.clone(), system.vel.clone(), float(T[0])

    fresh = {k: run(Forces(par, terms=TERMS, **CFG), c) for k, c in (("w", con_w), ("none", None), ("h", con_h))}
    for k, c in (("w", con_w), ("none", None), ("w", con_w), ("h", con_h), ("w", con_w)):
        pos, vel, T = run(shared, c)
        # (equal up to the order of the fp64 pair sums: the shared context's lists were built at other moments)
        assert (pos - fresh[k][0]).abs().max() < 1e-11 and (vel - fresh[k][1]).abs().max() < 1e-10, k
        assert abs(T - fresh[k][2]) < 1e-9 * T, k
    # what a mix-up would look like: the two water tables differ by 6.5e-7 A in the H-H distance
    assert abs(fresh["w"][2] - fresh["none"][2]) > 1.0 and (fresh["w"][0] - fresh["h"][0]).abs().max() > 1e-8


def test_cluster_path_reproducible_to_tolerance():
    """Cluster path (default): partner forces are summed by unordered reductions, so two runs agree to the fp32 summation
    level only -- the bound of the unconstrained cluster test (test_simt_cluster: 5e-5 A, 2e-3 A/tu after 10 steps)."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    res = []
    for _ in range(2):
        sysd, par, system, forces, con = _water(3333, torch.float32)
        torch.manual_seed(5)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        integ = Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con)
        integ.seed = 1234
        integ.step(10)
        res.append((system.pos.cpu().clone(), system.vel.cpu().clone()))
    dp = (res[0][0] - res[1][0]).abs().max().item()
    dv = (res[0][1] - res[1][1]).abs().max().item()
    print(f"cluster path, two runs of 10 steps: dpos {dp:.2e} dvel {dv:.2e}")
    assert dp < 5e-5 and dv < 2e-3


def test_stepwise_path_matches_md_steps():
    """The per-step path (duck-typed forces: tmd_vv_first / compute / tmd_vv_second) is constrained the same way."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    class Wrap:
        def __init__(self, f):
            self.f, self.par = f, f.par

        def compute(self, pos, box, forces):
            return self.f.compute(pos, box, forces)

    out = []
    for wrap in (False, True):
        sysd, par, system, forces, con = _water(300, torch.float64)
        torch.manual_seed(3)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        noise = torch.randn((6, 1, system.pos.shape[1], 3), dtype=torch.float64, generator=torch.Generator().manual_seed(4))
        integ = Integrator(system, Wrap(forces) if wrap else forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con)
        integ.step(6, noise=noise)
        out.append((system.pos.cpu().clone(), system.vel.cpu().clone()))
    assert (out[0][0] - out[1][0]).abs().max().item() < 1e-12
    assert (out[0][1] - out[1][1]).abs().max().item() < 1e-12


def test_nve_energy_conservation_f64(nw=1000, nsteps=5000):
    """Rigid water at 2 fs, NVE: the total energy fluctuates by at most 5 % of the kinetic energy's fluctuation."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    sysd, par, system, forces, con = _water(nw, torch.float64)
    torch.manual_seed(0)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con).step(500)  # melt the lattice start
    integ = Integrator(system, forces, 2.0, DEV, constraints=con)
    etot, ekin = [], []
    for _ in range(nsteps // 10):
        ek, pot, _ = integ.step(10)
        ekin.append(float(ek[0]))
        etot.append(float(ek[0]) + float(np.sum(pot[0])))
    etot, ekin = np.array(etot), np.array(ekin)
    drift = np.polyfit(np.arange(len(etot)) * 10 * 2e-6, etot, 1)[0]  # kcal/mol per ns
    print(f"NVE fp64 {nsteps} x 2 fs: rms(Etot) {etot.std():.4f}, rms(Ekin) {ekin.std():.4f} kcal/mol, "
          f"drift {drift:.3f} kcal/mol/ns ({drift / (3 * nw):.2e} per atom)")
    assert etot.std() <= 0.05 * ekin.std()


def test_langevin_temperature(nw=3333, nsteps=10000):
    """Langevin at 300 K with rigid water at 2 fs: the ndof-based temperature of the second half is 300 +- 2 K."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    sysd, par, system, forces, con = _water(nw, torch.float32)
    torch.manual_seed(0)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    integ = Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con)
    Ts = []
    for _ in range(nsteps // 50):
        _, _, T = integ.step(50)
        Ts.append(float(T[0]))
    mean = float(np.mean(Ts[len(Ts) // 2:]))
    print(f"Langevin 300 K, {nsteps} x 2 fs: mean T over the second half {mean:.2f} K (ndof {con.ndof()})")
    assert abs(mean - 300.0) <= 2.0


def test_determinism_and_split_calls(monkeypatch):
    """Full-row path: two runs are bitwise equal in fp32 and fp64, and step(10) equals step(4) then step(6)."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    monkeypatch.setenv("TMD_B200_CLUSTER", "0")
    for dtype in (torch.float32, torch.float64):
        res = []
        for split in ((10,), (10,), (4, 6)):
            sysd, par, system, forces, con = _water(300, dtype)
            torch.manual_seed(5)
            system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
            integ = Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con)
            integ.seed = 1234
            for k in split:
                integ.step(k)
            res.append((system.pos.cpu().clone(), system.vel.cpu().clone()))
        for other in res[1:]:
            assert torch.equal(res[0][0], other[0]) and torch.equal(res[0][1], other[1]), dtype


def test_kernel_launches_per_step():
    """Captured constrained step: k_vv_first, k_constrain_pos (which also prepares the force call), the pair kernel,
    the two bonded kernels, the folding second half-kick and k_constrain_vel: 7 launches per step against 4 for the
    fused unconstrained step."""
    from torchmd_b200 import Integrator, maxwell_boltzmann

    per_step = {}
    for constrained in (False, True):
        sysd, par, system, forces, con = _water(3333, torch.float32)
        torch.manual_seed(0)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        integ = Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con if constrained else None)
        integ.step(10)
        l0 = forces.stats()["kernel_launches"]
        integ.step(100)
        per_step[constrained] = (forces.stats()["kernel_launches"] - l0) / 100
    print(f"kernel launches per step: {per_step}")
    # (rebuild bodies are not counted; one launch per call outside the graphs shows up as the 0.01)
    assert round(per_step[False], 1) == 4.0
    assert round(per_step[True], 1) == 7.0

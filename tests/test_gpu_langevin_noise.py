"""The in-kernel Langevin noise, draw for draw, against the numpy restatement of oracle/philox.py.

Every Langevin run without injected noise draws its N(0,1) numbers inside the kernels: Philox4x32-10 keyed on (seed,
step, slot), then Box-Muller.  The noise of step s of atom i of replica r is ``normal3(seed, first_step + position + s,
r * N + i)`` on every path, where ``position`` is the context's Philox position before the call (``langevin_noise``).
Six kernels draw it -- k_vv_second<float>, k_vv_second_fold, k_cvv_second_fold, k_cstep_boundary, k_bonded_vv_second
and k_vv_second<double> -- and each one is checked here on the path that runs it.

a. Draw for draw.  Masses of 1e20 amu (the force term of a kick is ~1e-23 A/tu), gamma = 0 with T > 0 (the thermostat
   kicks, its friction term is exactly 0), zero start velocities, a per-atom ``vcoeff`` of distinct values and a time
   step of 1e-3 fs (no atom leaves its list): after n steps ``v = sum_s fl(xi_s * vcoeff)``, summed step after step.
   The same fp32 / fp64 sum over the restated draws must agree within the bound of oracle/philox.py per draw (fp32:
   2e-6 max(1, |xi|), fp64: 1e-14 max(1, |xi|)) plus an ulp of the running sum per step.  A draw of the wrong step,
   slot, replica or seed word changes a velocity by O(vcoeff) >= 0.05 A/tu.  Each case asserts the path it ran (the
   pair kernel id and the kernel launches per step), on two replicas in boxes of different size, with N = 7992 (not a
   multiple of the 256-thread blocks).
   Observed on an H100: max |dv| / vcoeff 0.9-2.0e-6 after 2-7 fp32 steps on every path (a few ulp of the sum),
   2.4-3.0e-15 in fp64.
b. Trajectories at production settings (gamma 50/ps, 300 K, real masses, in-kernel noise) against the fp64 oracle
   integrators fed the restated draws.  A one-step shift of the noise moves a hydrogen's velocity by about its
   vcoeff, 0.24 A/tu at 1 fs (0.34 at 2 fs); every bound is more than ten times smaller.  Observed on an H100 after 20
   steps (dpos A, dvel A/tu): fp32 flexible water on the cluster path 1.8e-5, 5.8e-4 (bounds 1e-3, 1e-2); fp32
   rigid water on the cluster path 2.0e-4, 1.3e-3 (same bounds); fp64 full rows 0, 2.2e-16; fp64 rigid water 1.9e-13,
   6.1e-13; fp64 ala2 with fixed X-H bonds 7.5e-14, 2.3e-13 (bounds 1e-9).
c. Paths against each other: bitwise on the full rows (captured against eager, one call against single steps and split
   calls, Monte Carlo barostat chunks against one call), within the fp32 summation bounds on the cluster path.

tests/test_langevin_noise_on_interpreter.py runs the draw checks on the host build of the kernels.
"""
import numpy as np
import pytest
import torch

from oracle import philox
from oracle import refmd
from torchmd_b200._lib import PAIR_CLUSTER

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
F32, F64 = torch.float32, torch.float64
POS_TOL32, VEL_TOL32 = 1e-4, 5e-4  # fp32 against fp64 after tens of steps (test_gpu_step_recovery, test_gpu_integrator)
# fp32 water with its stiff O-H bonds (or the constraints of rigid water) on the cluster path, whose force sums have no
# fixed order, against fp64: the bounds of test_gpu_cluster.test_gpu_cluster_md_follows_the_full_list_trajectory
WATER_POS_TOL32, WATER_VEL_TOL32 = 1e-3, 1e-2
HEAVY = 1e20  # amu: a kick by the forces is ~1e-23 A/tu, below the level checked even in fp64
TINY_DT = 1e-3  # fs
SEED = 0x2545F4914F6CDD1D & (2**62 - 1)
XI_BOUND = {np.float32: philox.F32_BOUND, np.float64: philox.F64_BOUND}  # per draw, relative to max(1, |xi|)


def _L():
    from torchmd_b200 import _lib

    return _lib.lib()


def _np(dtype):
    return np.float64 if dtype == F64 else np.float32


# ---------------------------------------------------------------------------------------------------- draw for draw
def heavy_water(dtype, terms=None):
    """Two replicas of the 7992-atom liquid water box of test_simt_cluster (43 A: the cluster path applies), the second
    one stretched with its box by 1.5 %; masses of 1e20 amu, zero velocities, the start forces computed."""
    from test_simt_cluster import CFG, TERMS, tiled_water
    from torchmd_b200 import Forces, System, testsystems

    sysd = tiled_water(2)
    c = np.asarray(sysd["coords"], np.float64)
    L = float(np.asarray(sysd["box"]).ravel()[0])
    s = 1.015
    x = np.stack([c, c * s])
    n = len(c)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    system = System(n, 2, dtype, DEV)
    system.set_positions(torch.tensor(x, dtype=dtype).permute(1, 2, 0))
    system.set_box(np.array([[L] * 3, [L * s] * 3]).T)
    system.set_masses(torch.full((n,), HEAVY, dtype=dtype))
    forces = Forces(par, terms=terms or TERMS, **CFG)
    forces.compute(system.pos, system.box, system.forces)
    return system, forces


def distinct_vcoeff(n, dtype, lo=0.05, hi=0.95):
    """A different coefficient for every atom (A/tu per unit draw), spread over [lo, hi)."""
    frac = np.modf(np.arange(n) * 0.6180339887498949)[0]
    return torch.tensor(lo + (hi - lo) * frac, dtype=dtype, device=DEV).view(-1, 1)


class Hidden:
    """Forces behind an object that is not a ``Forces``: the integrator drives it step by step (tmd_vv_first /
    tmd_vv_second, the duck-typed path of ``Integrator.step``)."""

    def __init__(self, f):
        self.f, self.par = f, f.par

    def compute(self, pos, box, forces):
        return self.f.compute(pos, box, forces)


def noise_integrator(system, forces, seed, stepwise=False):
    from torchmd_b200 import Integrator

    integ = Integrator(system, Hidden(forces) if stepwise else forces, TINY_DT, DEV, gamma=0.0, T=300.0)
    integ.seed = seed
    integ.vcoeff = distinct_vcoeff(system.natoms, system.pos.dtype)
    return integ


def summed_kicks(v0, xi, vc):
    """``v0 + fl(xi_1 vc) + fl(xi_2 vc) + ...`` in the precision of the draws, one rounding per operation (the kernels'
    order), and the bound on its distance from the kernels' sum: the restatement's bound per draw and one ulp of the
    running sum per step."""
    t = xi.dtype
    bound = XI_BOUND[t.type]
    vc = vc.astype(t).reshape(1, -1, 1)
    v = v0.astype(t)
    tol = np.zeros(v.shape)
    mag = np.abs(v0).astype(np.float64)
    for s in range(len(xi)):
        v = (v + (xi[s] * vc).astype(t)).astype(t)
        tol += vc * bound * np.maximum(1.0, np.abs(xi[s]))
        mag += np.abs(xi[s] * vc)
    tol += 2 * len(xi) * np.spacing(mag.astype(t)) + 1e-15
    return v, tol


def check_draws(system, integ, seed, nsteps, v0=None, position=0, first_step=0, what=""):
    """The velocities after ``nsteps`` noise-only steps against the restated draws; returns max |dv| / vcoeff."""
    dtype = _np(system.pos.dtype)
    xi = philox.langevin_noise(seed, nsteps, system.nreplicas, system.natoms, dtype, position=position, first_step=first_step)
    vc = integ.vcoeff.cpu().numpy().ravel()
    v0 = np.zeros(system.vel.shape, dtype) if v0 is None else v0
    want, tol = summed_kicks(v0, xi, vc)
    got = system.vel.cpu().numpy()
    dv = np.abs(got.astype(np.float64) - want)
    worst = float((dv / vc.reshape(1, -1, 1)).max())
    print(f"{what}: {nsteps} steps, max |dv|/vcoeff {worst:.2e} (bound {float((tol / vc.reshape(1, -1, 1)).max()):.2e})")
    bad = np.argwhere(dv > tol)
    assert len(bad) == 0, (what, len(bad), bad[:4].tolist(), float(dv.max()))
    return worst


def run_calls(integ, forces, calls):
    """Runs ``integ.step(n)`` for each n; returns the kernel launches per step of the last call."""
    per = None
    for n in calls:
        l0 = forces.stats()["kernel_launches"]
        integ.step(n)
        per = (forces.stats()["kernel_launches"] - l0) / n
    return per


# (environment, calls, terms, stepwise, precision, kernel, launches per step of the last call)
PATHS = {
    # k_vv_first_prepare -> (k_cpair + k_bonded) -> k_cstep_boundary x (n-1) ... -> k_cvv_second_fold
    "cluster_fused_2": ({}, (2,), None, False, F32, PAIR_CLUSTER, 4.5),
    "cluster_fused_7": ({}, (7,), None, False, F32, PAIR_CLUSTER, 29 / 7),
    # the same without the boundary kernel: k_cvv_second_fold every step
    "cluster_fusestep0": ({"TMD_B200_FUSESTEP": "0"}, (7,), None, False, F32, PAIR_CLUSTER, 5.0),
    # bonded terms after the pair kernel on the same stream: k_bonded_vv_second
    "cluster_overlap0": ({"TMD_B200_OVERLAP": "0"}, (7,), None, False, F32, PAIR_CLUSTER, 3.0),
    # the fused step issued kernel by kernel
    "cluster_graph0": ({"TMD_B200_GRAPH": "0"}, (7,), None, False, F32, PAIR_CLUSTER, 64 / 7),
    # full Verlet rows with the overlapped bonded kernel: k_vv_second_fold
    "full_rows": ({"TMD_B200_CLUSTER": "0"}, (7,), None, False, F32, None, 5.0),
    # no bonded kinds: k_vv_second after the cluster pair kernel
    "no_bonded": ({}, (7,), ["lj", "electrostatics"], False, F32, PAIR_CLUSTER, 3.0),
    # the duck-typed path: tmd_vv_first / compute / tmd_vv_second (k_vv_second)
    "stepwise": ({}, (7,), None, True, F32, PAIR_CLUSTER, 10.0),
    # step(1) repeated and a split call on the default path
    "single_steps": ({}, (1,) * 7, None, False, F32, PAIR_CLUSTER, 5.0),
    "split_3_4": ({}, (3, 4), None, False, F32, PAIR_CLUSTER, 17 / 4),
    # fp64: tmd_md_steps_f64 and the stepwise fp64 path (k_vv_second<double>)
    "fp64": ({}, (7,), None, False, F64, None, 12.0),
    "fp64_split": ({}, (3, 4), None, False, F64, None, 12.0),
    "fp64_stepwise": ({}, (7,), None, True, F64, None, 10.0),
}


def draw_case(monkeypatch, name, seed=SEED):
    env, calls, terms, stepwise, dtype, kernel, per_step = PATHS[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    system, forces = heavy_water(dtype, terms)
    integ = noise_integrator(system, forces, seed, stepwise)
    per = run_calls(integ, forces, calls)
    kern = _L().tmd_pair_kernel(forces._ctx)
    st = forces.stats()
    print(f"{name}: pair kernel {kern}, {per} launches per step, {st['rebuilds']} list builds")
    if kernel is not None:
        assert kern == kernel, kern
    elif dtype == F32:
        assert kern != PAIR_CLUSTER, kern
    if per_step is not None:
        assert per == pytest.approx(per_step), per
    assert not st["overflow"] and st["force_calls"] == 1 + sum(calls), st
    check_draws(system, integ, seed, sum(calls), what=f"{name} seed {seed:#x}")
    return system, integ


@pytest.mark.parametrize("name", list(PATHS))
def test_draws_on_every_path(monkeypatch, name):
    draw_case(monkeypatch, name)


@pytest.mark.parametrize("seed", [0, 2**32 - 1, 2**32, 2**62 - 1], ids=["0", "2^32-1", "2^32", "2^62-1"])
@pytest.mark.parametrize("name", ["cluster_fused_7", "fp64"])
def test_draws_at_edge_seeds(monkeypatch, name, seed):
    """Both seed words reach the key: seeds that differ only in the low or only in the high word."""
    draw_case(monkeypatch, name, seed)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_step_word_carries_into_the_high_counter_word(dtype):
    """The C entry point with ``first_step = 2^32 - 2``: the four steps of the call draw with Philox steps 2^32 - 1,
    2^32, 2^32 + 1 and 2^32 + 2, so the step's low word wraps inside the call and its high word takes the carry (the
    fp32 call runs the fused cluster step: k_cstep_boundary, then k_cvv_second_fold)."""
    from torchmd_b200 import _lib

    system, forces = heavy_water(dtype)
    integ = noise_integrator(system, forces, SEED)
    integ._require_cuda()
    ctx = forces._ensure_ctx(system.pos)
    forces._ensure_box(system.box)
    R, n, first = system.nreplicas, 4, 2**32 - 2
    ene = torch.zeros((R, _lib.NUM_ENERGIES), dtype=F64, device=DEV)
    ke = torch.zeros(R, dtype=F64, device=DEV)
    stream = torch.cuda.current_stream(system.pos.device).cuda_stream
    fn = _L().tmd_md_steps_f64 if dtype == F64 else _L().tmd_md_steps
    _lib.check(fn(ctx, n, system.pos.data_ptr(), system.vel.data_ptr(), system.forces.data_ptr(), integ.masses.data_ptr(),
                  integ.dt, 0.0, integ.vcoeff.data_ptr(), None, SEED, first, ene.data_ptr(), ke.data_ptr(), stream))
    st = forces.stats()
    assert not st["overflow"] and st["force_calls"] == 1 + n, st
    if dtype == F32:
        assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    check_draws(system, integ, SEED, n, first_step=first, what=f"first_step 2^32-2 {dtype}")


def test_recovered_call_draws_the_noise_of_its_steps(monkeypatch):
    """A call whose neighbour rows overflow at a step k >= 2 is run again from its saved state (Integrator.step); the
    discarded attempt advanced the Philox position, ``tmd_rewind_noise`` takes it back, and the rerun draws the noise
    of steps 1..n again.  The collapsing cloud of test_gpu_step_recovery, made of 1e20-amu atoms (the collapse is
    ballistic) with the restated draws on top of the start velocities; two replicas, only the second one collapses."""
    from test_gpu_step_recovery import cloud, full_rows
    from torchmd_b200 import Forces, Integrator, System

    full_rows(monkeypatch)
    spec = cloud(collapsing=(False, True))
    system = System(spec.natoms, spec.nrep, F32, DEV)
    system.pos[:] = torch.tensor(spec.coords, dtype=F32)
    system.vel[:] = torch.tensor(spec.vel, dtype=F32)
    system.set_box(spec.box)
    system.set_masses(torch.full((spec.natoms,), HEAVY))
    forces = Forces(spec.par(F32, DEV), terms=spec.terms, **spec.cfg)
    forces.compute(system.pos, system.box, system.forces)
    cap0 = forces.stats()["row_capacity"]
    integ = Integrator(system, forces, 1.0, DEV, gamma=0.0, T=300.0)
    integ.seed = SEED
    integ.vcoeff = distinct_vcoeff(spec.natoms, F32, 0.01, 0.05)
    v0 = system.vel.cpu().numpy().copy()
    niter = 30
    integ.step(niter)
    st = forces.stats()
    assert st["row_capacity"] > cap0 and st["force_calls"] > 1 + niter and not st["overflow"], (cap0, st)  # it recovered
    check_draws(system, integ, SEED, niter, v0=v0, what="recovered call")
    v1 = system.vel.cpu().numpy().copy()
    integ.step(5)  # and the call after it continues the stream
    check_draws(system, integ, SEED, 5, v0=v1, position=niter, what="the call after")


# ---------------------------------------------------------------------------------------------------- trajectories
LANGEVIN = (50.0, 300.0)  # gamma in 1/ps, T in K


def shift_scale(masses, dt_fs, gamma_ps=LANGEVIN[0], T=LANGEVIN[1]):
    """vcoeff of the lightest atom: what a one-step shift of the noise moves its velocity by (A/tu)."""
    from torchmd_b200.integrator import BOLTZMAN, PICOSEC2TIMEU, TIMEFACTOR

    m = float(np.min(np.asarray(masses, np.float64)))
    return float(np.sqrt(2.0 * gamma_ps / PICOSEC2TIMEU / m * BOLTZMAN * T * dt_fs / TIMEFACTOR))


def trajectory(dtype, par, par64, coords, box, terms, cfg, nsteps, dt_fs, kind=None, nrep=1, seed=SEED, calls=None):
    """GPU run with in-kernel noise from ``seed`` and the fp64 oracle (RATTLE with constraints) fed the restated draws of
    that seed, from the same start state.  Returns (dpos, dvel, GPU forces object)."""
    from torchmd_b200 import Constraints, Forces, Integrator, System, maxwell_boltzmann

    n = len(coords)
    system = System(n, nrep, dtype, DEV)
    x = np.repeat(np.asarray(coords, np.float64)[None], nrep, 0)
    if nrep > 1:
        x[1:] += np.random.default_rng(1).normal(0, 0.02, x[1:].shape)
    system.set_positions(torch.tensor(x, dtype=dtype).permute(1, 2, 0))
    system.set_box(np.asarray(box))
    torch.manual_seed(2)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, nrep))
    forces = Forces(par, terms=terms, **cfg)
    con = Constraints(par, kind) if kind else None
    forces.compute(system.pos, system.box, system.forces)
    start = {k: getattr(system, k).cpu().double().clone() for k in ("pos", "vel", "box")}
    integ = Integrator(system, forces, dt_fs, DEV, gamma=LANGEVIN[0], T=LANGEVIN[1], constraints=con)
    integ.seed = seed
    for c in calls or (nsteps,):
        integ.step(c)
    noise = torch.tensor(philox.langevin_noise(seed, nsteps, nrep, n, _np(dtype))).double()
    dec = F32 if dtype == F32 else F64
    if kind:
        from test_gpu_constraints import _oracle_run

        pos, vel, _ = _oracle_run(start, par64, con, terms, cfg, nsteps, noise, dt_fs, LANGEVIN[0], LANGEVIN[1], dec)
    else:
        of = refmd.OracleForces(par64, terms, decision_dtype=dec, **cfg)
        pos, vel, box64 = start["pos"].clone(), start["vel"].clone(), start["box"].clone()
        f = torch.zeros_like(pos)
        of.compute(pos, box64, f)
        refmd.OracleIntegrator(pos, vel, box64, f, par64.masses.double(), of.compute, dt_fs, gamma_ps=LANGEVIN[0],
                               T=LANGEVIN[1]).step(nsteps, noise=noise)
    dp = (system.pos.cpu().double() - pos).abs().max().item()
    dv = (system.vel.cpu().double() - vel).abs().max().item()
    return dp, dv, forces


def test_trajectory_fp32_cluster_water():
    """7992 flexible waters in a 43 A box on the cluster path (fused steps), 20 steps at 1 fs in one call."""
    from test_simt_cluster import CFG, TERMS, tiled_water
    from torchmd_b200 import testsystems

    sysd = tiled_water(2)
    par = testsystems.water_parameters(sysd, device=DEV)
    par64 = testsystems.water_parameters(sysd, precision=F64)
    dp, dv, forces = trajectory(F32, par, par64, sysd["coords"], sysd["box"], TERMS, CFG, 20, 1.0)
    shift = shift_scale(par64.masses, 1.0)
    print(f"fp32 cluster water 20 steps: dpos {dp:.2e} A, dvel {dv:.2e} A/tu (one-step noise shift {shift:.2f} A/tu)")
    assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    assert 10 * WATER_VEL_TOL32 < shift
    assert dp < WATER_POS_TOL32 and dv < WATER_VEL_TOL32, (dp, dv)


def test_trajectory_fp64_full_rows():
    """The LJ + Coulomb cloud of test_gpu_step_recovery (two replicas) through tmd_md_steps_f64, 20 steps at 1 fs."""
    from test_gpu_step_recovery import cloud

    spec = cloud(collapsing=(False, False))
    par, par64 = spec.par(F64, DEV), spec.par(F64, "cpu")
    dp, dv, _ = trajectory(F64, par, par64, spec.coords[0], spec.box, spec.terms, spec.cfg, 20, 1.0, nrep=2)
    print(f"fp64 full rows 20 steps: dpos {dp:.2e} A, dvel {dv:.2e} A/tu (one-step noise shift {shift_scale(par64.masses, 1.0):.2f})")
    assert dp < 1e-9 and dv < 1e-9, (dp, dv)


@pytest.mark.parametrize("name,kind", [("water300", "water"), ("ala2_xsc_rf", "hbonds")])
def test_trajectory_fp64_constrained(name, kind):
    """RATTLE at 2 fs: rigid water (SETTLE groups) and alanine dipeptide with its X-H bonds fixed, 20 steps."""
    from torchmd_b200 import testsystems

    if name.startswith("water"):
        from test_gpu_constraints import CFG, TERMS

        sysd = testsystems.water_box(300, seed=0)
        par = testsystems.water_parameters(sysd, precision=F64, device=DEV)
        par64 = testsystems.water_parameters(sysd, precision=F64)
        coords, box, terms, cfg = sysd["coords"], sysd["box"], TERMS, CFG
    else:
        par, coords, box, terms, cfg = testsystems.golden_system(name, precision=F64, device=DEV)
        par64 = testsystems.golden_system(name, precision=F64)[0]
    dp, dv, _ = trajectory(F64, par, par64, coords, box, terms, cfg, 20, 2.0, kind=kind)
    print(f"fp64 {name} {kind} 20 steps: dpos {dp:.2e} A, dvel {dv:.2e} A/tu")
    assert dp < 1e-9 and dv < 1e-9, (dp, dv)


def test_trajectory_fp32_rigid_water_cluster():
    """Rigid water on the cluster path (the constrained step: no boundary kernel, k_cvv_second_fold and the velocity
    constraint), 20 steps at 2 fs in one call."""
    from test_simt_cluster import CFG, TERMS, tiled_water
    from torchmd_b200 import testsystems

    sysd = tiled_water(2)
    par = testsystems.water_parameters(sysd, device=DEV)
    par64 = testsystems.water_parameters(sysd, precision=F64)
    dp, dv, forces = trajectory(F32, par, par64, sysd["coords"], sysd["box"], TERMS, CFG, 20, 2.0, kind="water")
    print(f"fp32 rigid water, cluster path, 20 steps: dpos {dp:.2e} A, dvel {dv:.2e} A/tu")
    assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
    assert 10 * WATER_VEL_TOL32 < shift_scale(par64.masses, 2.0)
    assert dp < WATER_POS_TOL32 and dv < WATER_VEL_TOL32, (dp, dv)


# ---------------------------------------------------------------------------------------------------- paths agree
def langevin_run(spec, dtype, calls, barostat=None):
    """The cloud of test_gpu_step_recovery at gamma 50/ps, 300 K, 1 fs with in-kernel noise; returns (pos, vel)."""
    from torchmd_b200 import Forces, Integrator, System

    system = System(spec.natoms, spec.nrep, dtype, DEV)
    system.pos[:] = torch.tensor(spec.coords, dtype=dtype)
    system.vel[:] = torch.tensor(spec.vel, dtype=dtype)
    system.set_box(spec.box)
    forces = Forces(spec.par(dtype, DEV), terms=spec.terms, **spec.cfg)
    forces.compute(system.pos, system.box, system.forces)
    integ = Integrator(system, forces, 1.0, DEV, gamma=LANGEVIN[0], T=LANGEVIN[1], barostat=barostat)
    integ.seed = SEED
    for n in calls:
        integ.step(n)
    return system.pos.cpu().clone(), system.vel.cpu().clone()


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_full_rows_paths_agree_bitwise(monkeypatch, dtype):
    """Full rows, two replicas, 12 steps: captured steps, eagerly issued steps, 12 single steps and 5 + 7 end in the same
    state to the bit."""
    from test_gpu_step_recovery import cloud, full_rows

    spec = cloud(collapsing=(False, False))
    full_rows(monkeypatch)
    one = langevin_run(spec, dtype, (12,))
    for graph, calls in (("0", (12,)), ("1", (1,) * 12), ("1", (5, 7)), ("0", (5, 7))):
        full_rows(monkeypatch, graph)
        other = langevin_run(spec, dtype, calls)
        assert torch.equal(one[0], other[0]) and torch.equal(one[1], other[1]), (graph, calls)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_barostat_chunks_keep_the_philox_position(monkeypatch, dtype):
    """With a Monte Carlo barostat of frequency 4 the 14 steps run as calls of 4, 4, 4 and 2 steps; with its moves
    switched off the run must be the run without a barostat, bit for bit: the Philox position carries across chunks."""
    from test_gpu_step_recovery import cloud, full_rows
    from torchmd_b200.barostat import MonteCarloBarostat

    spec = cloud(collapsing=(False, False))
    full_rows(monkeypatch)
    plain = langevin_run(spec, dtype, (14,))
    moves = []
    monkeypatch.setattr(MonteCarloBarostat, "attempt", lambda self, ctx, ene: moves.append(1) or [0.0] * spec.nrep)
    chunked = langevin_run(spec, dtype, (14,), barostat=MonteCarloBarostat(frequency=4, seed=1))
    assert len(moves) == 3
    assert torch.equal(plain[0], chunked[0]) and torch.equal(plain[1], chunked[1])


def test_cluster_paths_agree_to_the_summation_order(monkeypatch):
    """The flexible water box on the cluster path, 12 steps: one call, single steps, 5 + 7, eagerly issued steps, and
    the unfused step (TMD_B200_FUSESTEP=0) end within the fp32 bounds of each other (their force sums differ in order)."""
    from test_simt_cluster import CFG, TERMS, tiled_water
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann, testsystems

    sysd = tiled_water(2)

    def run(calls):
        par = testsystems.water_parameters(sysd, device=DEV)
        system = System(len(sysd["coords"]), 1, F32, DEV)
        system.set_positions(np.asarray(sysd["coords"], np.float32))
        system.set_box(sysd["box"])
        torch.manual_seed(2)
        system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
        forces = Forces(par, terms=TERMS, **CFG)
        forces.compute(system.pos, system.box, system.forces)
        integ = Integrator(system, forces, 1.0, DEV, gamma=LANGEVIN[0], T=LANGEVIN[1])
        integ.seed = SEED
        for n in calls:
            integ.step(n)
        assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
        return system.pos.cpu().clone(), system.vel.cpu().clone()

    one = run((12,))
    worst = 0.0
    for env, calls in (({}, (1,) * 12), ({}, (5, 7)), ({"TMD_B200_GRAPH": "0"}, (12,)), ({"TMD_B200_FUSESTEP": "0"}, (12,))):
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            p, v = run(calls)
        dp, dv = (p - one[0]).abs().max().item(), (v - one[1]).abs().max().item()
        worst = max(worst, dv)
        assert dp < POS_TOL32 and dv < VEL_TOL32, (env, calls, dp, dv)
    print(f"cluster path, 12 steps: the paths agree to {worst:.2e} A/tu")

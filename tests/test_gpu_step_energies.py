"""The energies ``Integrator.step`` returns -- ``(Ekin, pot, T)`` and the per-term (R, NUM_ENERGIES) buffer behind ``pot``
-- on every step path, against a fresh evaluation of the final state and the fp64 oracle.

The trajectory tests compare positions and velocities; the energies of a call come from other code: the captured step
variants with energy outputs, the energy memset inside a replayed graph, the side-stream bonded kernel adding the
bonded and 1-4 energies into the slots the pair kernel fills, the kinetic energy of the last second half-kick (or of the
velocity constraint), the PME energy chain, the Monte Carlo move, and the host copies of ``tmd_md_steps_host``.

A pass's energies depend on the positions and the box alone: the pair decisions are exact, a pair's fp32 value does not
depend on which of its atoms is "i" (the fixed-point difference negates exactly, qq, A and B are symmetric), only the
order of the fp64 sums varies.  So after every call the reported energies equal a fresh ``Forces.compute(...,
returnDetails=True)`` at ``(system.pos, system.box)`` term by term to fp64 summation error, bound ``1e-10 sum|E_term| +
1e-9`` -- on the cluster path too, whose forces only reproduce to 2e-5.  ``Ekin`` is 0.5 sum m v^2 of the final
velocities in fp64 (to 2^-23 relative for fp32 state: the fp32 products and the cast of the fp64 sum; 1e-12 in fp64),
``T`` is 2 Ekin / (3 N kB), or / (ndof kB) with constraints.

Each case runs three consecutive calls on two replicas in boxes of different size (one replica where the path allows
only one) and asserts the path it ran (the pair kernel id; the kernel launches per step of the last call when no list
was rebuilt inside it).  On full rows, where split calls are bitwise equal, a twin run stops one step short of the last
call: its energies differ from the reported ones by more than 100 times the bound, so an energy one step stale fails.
Systems of at most 3000 atoms are also compared with the fp64 oracle per term at the parity bound of DESIGN.md
section 2 (fp32: 1e-5 |E| + 2e-3 with the fp32 pair decisions; fp64: 1e-10 relative).

Observed on an H100 (80 GB HBM3, 700 W): per-term |dE| against the fresh pass at most 1.5e-11 kcal/mol on the RF paths,
1.8e-10 with PME, on |E_term| up to ~3e4; Ekin within 5.0e-8 relative in fp32 and 2.6e-16 in fp64; the last step moves
E_pot by 1e6 to 3e8 bounds; oracle per term 8.0e-4 (fp32) and 1.4e-12 (fp64) on ala2.

tests/test_step_energies_on_interpreter.py runs a subset on the host build of the kernels.
"""
import numpy as np
import pytest
import torch

from oracle import refmd
from torchmd_b200._lib import PAIR_CLUSTER, PAIR_EWALD_CLUSTER, PAIR_EWALD_F64, PAIR_EWALD_FX2

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
F32, F64 = torch.float32, torch.float64
SEED = 0x5DEECE66D
LANGEVIN = (1.0, 300.0)  # gamma in 1/ps, T in K
ORACLE_MAX_ATOMS = 3000
EKIN_RTOL = {F32: 2.0**-23, F64: 1e-12}
SHIFT_FACTOR = 100.0  # a one-step shift must move the energies by this many bounds


def _L():
    from torchmd_b200 import _lib

    return _lib.lib()


def term_bound(terms, rel=1e-10):
    """fp64 summation error allowed between two passes over the same state: 1e-10 sum|E_term| + 1e-9 kcal/mol."""
    return rel * sum(abs(v) for v in terms.values()) + 1e-9


# ---------------------------------------------------------------------------------------------------- systems
class Case:
    """A system, its Forces and what the oracle needs: par64, terms, cfg, and the CMAP terms' parameters if any."""

    def __init__(self, system, forces, par64, terms, cfg, pme=False, cmap=None, constraints=None):
        self.system, self.forces, self.par64, self.terms, self.cfg = system, forces, par64, terms, cfg
        self.pme, self.cmap, self.constraints = pme, cmap, constraints


def _two_boxes(system, coords, box, nrep, s):
    """Replicas of the same coordinates, the second one in a box ``s`` times longer (its boundary layer differs)."""
    system.set_positions(torch.tensor(np.repeat(np.asarray(coords, np.float64)[:, :, None], nrep, 2)))
    b = np.asarray(box, np.float64).ravel()
    system.set_box(np.stack([b * (s if r else 1.0) for r in range(nrep)], 1))


def water8k(dtype, nrep=2, pme=False, kind=None):
    """The 7992-atom liquid water box of test_simt_cluster (43 A: the cluster path applies), real masses, Maxwell-
    Boltzmann velocities; RF at 5 A, or PME at 6 A; ``kind``: rigid water."""
    from test_simt_cluster import CFG, TERMS, tiled_water
    from torchmd_b200 import Constraints, Forces, System, maxwell_boltzmann, testsystems

    sysd = tiled_water(2)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    n = len(sysd["coords"])
    system = System(n, nrep, dtype, DEV)
    _two_boxes(system, sysd["coords"], sysd["box"], nrep, 1.015)
    torch.manual_seed(2)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, nrep))
    cfg = dict(cutoff=6.0, switch_dist=5.0) if pme else dict(CFG)
    forces = Forces(par, terms=TERMS, pme=pme, **cfg)
    return Case(system, forces, None, TERMS, cfg, pme=pme, constraints=Constraints(par, kind) if kind else None)


def ala2(dtype, nrep=2, cmap=False, kind=None):
    """Solvated alanine dipeptide (688 atoms, RF at 9 A, every bonded kind and 41 1-4 pairs on the bonded kernel),
    ``cmap``: with the backbone CMAP term of test_gpu_cmap (its energy is booked under ``dihedrals``); ``kind``: fixed
    X-H bonds."""
    from conftest import load_golden
    from torchmd_b200 import Constraints, Forces, System, maxwell_boltzmann, testsystems

    par, coords, box, terms, cfg = testsystems.golden_system("ala2_xsc_rf", precision=dtype, device=DEV)
    par64 = testsystems.golden_system("ala2_xsc_rf", precision=F64)[0]
    if cmap:
        import test_gpu_cmap

        g = load_golden("ala2_xsc_rf")
        par = test_gpu_cmap.make_params(g, "ala2_xsc_rf", dtype)
        par64 = test_gpu_cmap.make_params(g, "ala2_xsc_rf", F64)
        par64.to_("cpu")
    system = System(len(coords), nrep, dtype, DEV)
    _two_boxes(system, coords, box, nrep, 1.01)
    torch.manual_seed(3)
    system.set_velocities(maxwell_boltzmann(par.masses.cpu(), 300.0, nrep))
    forces = Forces(par, terms=terms, **cfg)
    return Case(system, forces, par64, terms, cfg, cmap=par64.cmap_params if cmap else None,
                constraints=Constraints(par, kind) if kind else None)


def protein(dtype):
    """ala2 tiled 2 x 2 x 2 (5504 atoms): the cluster path with 1-4 pairs and torsions on the overlapped bonded kernel."""
    from test_gpu_cluster_systems import params, protein as tiled
    from torchmd_b200 import Forces, System, maxwell_boltzmann

    spec = tiled(2)
    par = params(spec, dtype, DEV)
    system = System(len(spec["coords"]), 2, dtype, DEV)
    _two_boxes(system, spec["coords"], spec["box"], 2, 1.01)
    torch.manual_seed(4)
    system.set_velocities(maxwell_boltzmann(par.masses.cpu(), 300.0, 2))
    return Case(system, Forces(par, terms=spec["terms"], **spec["cfg"]), None, spec["terms"], spec["cfg"])


SYSTEMS = {"water8k": water8k, "water8k_pme": lambda d: water8k(d, pme=True), "water8k_rigid": lambda d: water8k(d, kind="water"),
           "ala2": ala2, "ala2_cmap": lambda d: ala2(d, cmap=True), "ala2_hbonds": lambda d: ala2(d, kind="hbonds"),
           "protein": protein}


class Hidden:
    """Forces behind an object that is not a ``Forces``: the integrator drives it step by step (tmd_vv_first /
    compute / tmd_vv_second)."""

    def __init__(self, f):
        self.f, self.par = f, f.par

    def compute(self, pos, box, forces):
        return self.f.compute(pos, box, forces)


def integrator(case, stepwise=False, thermostat=True, batch=None, barostat=None):
    from torchmd_b200 import Integrator

    dt = 2.0 if case.constraints is not None else 1.0
    kw = dict(gamma=LANGEVIN[0], T=LANGEVIN[1]) if thermostat else {}
    integ = Integrator(case.system, Hidden(case.forces) if stepwise else case.forces, dt, DEV, batch=batch,
                       constraints=case.constraints, barostat=barostat, **kw)
    integ.seed = SEED
    return integ


# ---------------------------------------------------------------------------------------------------- the checks
def fresh(case):
    """Per-term energies of a fresh evaluation at the system's state (its forces into a scratch buffer)."""
    s = case.system
    return case.forces.compute(s.pos, s.box, torch.empty_like(s.forces), returnDetails=True)


def kinetic64(system, masses):
    v = system.vel.double().cpu().numpy()
    m = masses.double().cpu().numpy().reshape(1, -1, 1)
    return 0.5 * (m * v * v).sum(axis=(1, 2))


def check_call(case, integ, out, what, per_term=True, rel=1e-10):
    """The returned (Ekin, pot, T) and the per-term buffer against a fresh evaluation and 0.5 sum m v^2 of the final
    state.  Returns (worst |dE| per term, worst Ekin relative error, fresh per-term energies)."""
    from torchmd_b200._lib import ENERGY_SLOTS
    from torchmd_b200.integrator import BOLTZMAN

    Ekin, pot, T = out
    s, f = case.system, case.forces
    dtype = s.pos.dtype
    ref = fresh(case)
    ene = integ._out[1].cpu().numpy()
    cols = f._energy_columns()
    worst = 0.0
    for r in range(s.nreplicas):
        bound = term_bound(ref[r], rel)
        if per_term:
            for t, c in zip(f.energies, cols):
                d = abs(ene[r, c] - ref[r][t])
                worst = max(worst, d)
                assert d <= bound, (what, r, t, ene[r, c], ref[r][t], bound)
            for c, t in enumerate(ENERGY_SLOTS):  # (the "1-4" slot stays 0: those energies are booked under lj / electrostatics)
                if c not in cols or t == "1-4":
                    assert ene[r, c] == 0.0, (what, r, t, ene[r, c])
            total = ene[r, cols].sum()  # (the barostat sums on the device: the order of a few additions differs)
            assert abs(pot[r] - total) <= 1e-14 * np.abs(ene[r, cols]).sum(), (what, r, pot[r], total)
        else:
            d = abs(pot[r] - sum(ref[r][t] for t in f.energies))
            worst = max(worst, d)
            assert d <= bound, (what, r, pot[r], bound)
    if integ.batch is None:
        want = kinetic64(s, integ.masses)
        dof = np.full(s.nreplicas, 3.0 * s.natoms) if case.constraints is None else np.full(s.nreplicas, float(integ.ndof))
    else:  # one replica, one entry per group
        v = s.vel.double().cpu().numpy()[0]
        m = integ.masses.double().cpu().numpy().ravel()
        b = integ.batch.cpu().numpy()
        want = np.bincount(b, weights=0.5 * m * (v * v).sum(1))
        dof = 3.0 * np.bincount(b)
    assert Ekin.shape == want.shape, (what, Ekin.shape, want.shape)
    ek_err = np.abs(Ekin.astype(np.float64) - want) / want
    assert (ek_err <= EKIN_RTOL[dtype]).all(), (what, Ekin, want, ek_err)
    np.testing.assert_allclose(np.asarray(T, np.float64), 2.0 * Ekin.astype(np.float64) / (dof * BOLTZMAN),
                               rtol=1e-6 if dtype == F32 else 1e-14, err_msg=what)
    return worst, float(ek_err.max()), ref


def check_oracle(case, ref, what):
    """The per-term energies of the final state against the fp64 oracle at the parity bound."""
    s = case.system
    dtype = s.pos.dtype
    of = refmd.OracleForces(case.par64, case.terms, decision_dtype=dtype, **case.cfg)
    pos, box = s.pos.detach().double().cpu(), s.box.detach().double().cpu()
    E = of.compute(pos, box, torch.zeros_like(pos))
    if case.cmap is not None:
        from oracle import cmap as ocmap

        args = [case.cmap[k].cpu().numpy() for k in ("idx", "map_of", "res", "grids")]
        for r in range(s.nreplicas):
            E[r]["dihedrals"] += ocmap.energy_forces(pos[r].numpy(), *args, box=torch.diagonal(box[r]).numpy())[0]
    worst = 0.0
    for r in range(s.nreplicas):
        for t in case.forces.energies:
            e, o = ref[r][t], E[r][t]
            tol = 1e-5 * abs(o) + 2e-3 if dtype == F32 else 1e-10 * max(1.0, abs(o))
            worst = max(worst, abs(e - o))
            assert abs(e - o) <= tol, (what, r, t, e, o, tol)
    return worst


def run_calls(case, integ, calls, noise=False, per_term=True):
    """Runs ``integ.step(n)`` for each n and checks every call.  Returns (worst dE, worst Ekin error, launches per step
    of the last call, whether a list was rebuilt inside it, reported per-term energies, what each call returned)."""
    f = case.forces
    worst_e = worst_k = 0.0
    outs = []
    for k, n in enumerate(calls):
        st0 = f.stats()
        if noise:
            g = torch.Generator().manual_seed(100 + k)
            out = integ.step(n, noise=torch.randn((n,) + tuple(case.system.vel.shape), generator=g, dtype=F64))
        else:
            out = integ.step(n)
        st1 = f.stats()
        per = (st1["kernel_launches"] - st0["kernel_launches"]) / n
        rebuilt = st1["rebuilds"] != st0["rebuilds"]
        e, ek, ref = check_call(case, integ, out, f"call {k + 1} of {calls}", per_term)
        worst_e, worst_k = max(worst_e, e), max(worst_k, ek)
        outs.append((out, ref))
    return worst_e, worst_k, per, rebuilt, outs


def one_step_short(case_fn, dtype, calls, integ_kw):
    """A twin of the run whose last call is split as (n - 1, 1): returns (the twin, its per-term energies one step
    before the end)."""
    case = case_fn(dtype)
    case.forces.compute(case.system.pos, case.system.box, case.system.forces)
    integ = integrator(case, **integ_kw)
    *head, last = calls
    for n in head:
        integ.step(n)
        fresh(case)  # (as the checked run does between its calls)
    if last > 1:
        integ.step(last - 1)
    earlier = fresh(case)
    integ.step(1)
    return case, earlier


# (environment, system, precision, calls, stepwise, injected noise, pair kernel, launches per step of the last call)
PATHS = {
    # k_vv_first_prepare -> (k_cpair + k_bonded) -> k_cstep_boundary ... -> k_cvv_second_fold; variants 2, 3 and 4
    "cluster_fused_2": ({}, "water8k", F32, (2, 2, 2), False, False, PAIR_CLUSTER, 4.5),
    "cluster_fused_7": ({}, "water8k", F32, (7, 7, 7), False, False, PAIR_CLUSTER, 29 / 7),
    # k_cvv_second_fold every step: variants 0 and 1
    "cluster_fusestep0": ({"TMD_B200_FUSESTEP": "0"}, "water8k", F32, (7, 7, 7), False, False, PAIR_CLUSTER, 5.0),
    # the bonded energies from k_bonded_vv_second on the same stream
    "cluster_overlap0": ({"TMD_B200_OVERLAP": "0"}, "water8k", F32, (7, 7, 7), False, False, PAIR_CLUSTER, 3.0),
    # the fused step issued kernel by kernel: the energy memset outside a graph
    "cluster_graph0": ({"TMD_B200_GRAPH": "0"}, "water8k", F32, (7, 7, 7), False, False, PAIR_CLUSTER, 64 / 7),
    # full Verlet rows, overlapped bonded kernel, k_vv_second_fold
    "full_rows": ({"TMD_B200_CLUSTER": "0"}, "water8k", F32, (7, 7, 7), False, False, None, 5.0),
    "full_rows_graph0": ({"TMD_B200_CLUSTER": "0", "TMD_B200_GRAPH": "0"}, "water8k", F32, (5, 5, 5), False, False, None, None),
    # the duck-typed path: pot from the last compute, ke from k_vv_second
    "stepwise": ({}, "water8k", F32, (3, 3, 3), True, False, PAIR_CLUSTER, None),
    "single_steps": ({}, "water8k", F32, (1, 1, 1), False, False, PAIR_CLUSTER, None),
    "split_3_4": ({}, "water8k", F32, (3, 4, 3), False, False, PAIR_CLUSTER, None),
    # injected noise: no graph, no fused step
    "noise": ({}, "water8k", F32, (3, 3, 3), False, True, PAIR_CLUSTER, None),
    # tmd_md_steps_f64 and the stepwise fp64 path
    "fp64": ({}, "water8k", F64, (5, 5, 5), False, False, None, None),
    "fp64_split": ({}, "water8k", F64, (2, 3, 1), False, False, None, None),
    "fp64_stepwise": ({}, "water8k", F64, (3, 3, 3), True, False, None, None),
    # the PME energy chain: cluster Ewald kernel, full rows, fp64
    "pme_cluster": ({}, "water8k_pme", F32, (5, 5, 5), False, False, PAIR_EWALD_CLUSTER, None),
    "pme_full_rows": ({"TMD_B200_CLUSTER": "0"}, "water8k_pme", F32, (5, 5, 5), False, False, PAIR_EWALD_FX2, None),
    "pme_fp64": ({}, "water8k_pme", F64, (3, 3, 3), False, False, PAIR_EWALD_F64, None),
    # ke from the velocity constraint: rigid water (cluster path in fp32), X-H bonds of ala2
    "rigid_water": ({}, "water8k_rigid", F32, (5, 5, 5), False, False, PAIR_CLUSTER, None),
    "rigid_water_fp64": ({}, "water8k_rigid", F64, (3, 3, 3), False, False, None, None),
    "hbonds": ({}, "ala2_hbonds", F32, (5, 5, 5), False, False, None, None),
    "hbonds_fp64": ({}, "ala2_hbonds", F64, (5, 5, 5), False, False, None, None),
    # CMAP under dihedrals, 1-4 under lj / electrostatics, from the overlapped bonded kernel
    "cmap": ({}, "ala2_cmap", F32, (5, 5, 5), False, False, None, None),
    "cmap_fp64": ({}, "ala2_cmap", F64, (5, 5, 5), False, False, None, None),
    "pairs14_cluster": ({}, "protein", F32, (7, 7, 7), False, False, PAIR_CLUSTER, None),
}


def energy_case(monkeypatch, name):
    env, sysname, dtype, calls, stepwise, noise, kernel, per_step = PATHS[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    case = SYSTEMS[sysname](dtype)
    case.forces.compute(case.system.pos, case.system.box, case.system.forces)
    integ = integrator(case, stepwise)
    worst_e, worst_k, per, rebuilt, outs = run_calls(case, integ, calls, noise, per_term=not stepwise)
    st = case.forces.stats()
    kern = _L().tmd_pair_kernel(case.forces._ctx)
    line = (f"{name}: pair kernel {kern}, {per:.3f} launches per step{' (a list rebuilt)' if rebuilt else ''}, "
            f"{st['rebuilds']} list builds; worst per-term |dE| {worst_e:.2e} kcal/mol, Ekin rel. error {worst_k:.2e}")
    if kernel is not None:
        assert kern == kernel, (name, kern)
    elif dtype == F32:
        assert kern not in (PAIR_CLUSTER, PAIR_EWALD_CLUSTER), (name, kern)
    if per_step is not None and not rebuilt:
        assert per == pytest.approx(per_step), (name, per)
    assert not st["overflow"], st
    if case.system.natoms <= ORACLE_MAX_ATOMS and not case.pme:
        wo = check_oracle(case, outs[-1][1], name)
        line += f"; oracle per-term |dE| {wo:.2e}"
    print(line)
    return case, integ, outs


@pytest.mark.parametrize("name", list(PATHS))
def test_energies_on_every_path(monkeypatch, name):
    energy_case(monkeypatch, name)


SHIFT_CASES = ["full_rows", "full_rows_graph0", "fp64", "fp64_split", "hbonds_fp64", "cmap"]


@pytest.mark.parametrize("name", SHIFT_CASES)
def test_a_one_step_shift_is_detected(monkeypatch, name):
    """On full rows a call split as (n - 1, 1) ends bitwise where the whole call ends: the state one step before the
    reported one has energies more than 100 bounds away from those reported, per replica."""
    env, sysname, dtype, calls, stepwise, noise, kernel, _ = PATHS[name]
    case, integ, outs = energy_case(monkeypatch, name)
    twin, earlier = one_step_short(SYSTEMS[sysname], dtype, calls, dict(stepwise=stepwise))
    assert torch.equal(twin.system.pos, case.system.pos) and torch.equal(twin.system.vel, case.system.vel), name
    reported = outs[-1][1]
    for r in range(case.system.nreplicas):
        bound = term_bound(reported[r])
        shift = abs(sum(earlier[r].values()) - sum(reported[r].values()))
        print(f"{name} replica {r}: E_pot moved {shift:.3e} kcal/mol in the last step, {shift / bound:.1e} bounds")
        assert shift > SHIFT_FACTOR * bound, (name, r, shift, bound)


def test_batch_groups(monkeypatch):
    """``batch=``: Ekin and T per group of one replica (the kinetic energy of each group from the final velocities)."""
    monkeypatch.setenv("TMD_B200_CLUSTER", "0")
    case = water8k(F32, nrep=1)
    case.forces.compute(case.system.pos, case.system.box, case.system.forces)
    n = case.system.natoms
    batch = torch.tensor(np.repeat(np.arange(3), [n // 3, n // 3, n - 2 * (n // 3)]), device=DEV)
    integ = integrator(case, batch=batch)
    worst_e, worst_k, *_ = run_calls(case, integ, (3, 3))
    print(f"batch groups: worst per-term |dE| {worst_e:.2e}, Ekin rel. error {worst_k:.2e}")


# ---------------------------------------------------------------------------------------------------- barostat
# In fp32 the energy of a replica is not independent of the other replicas' boxes: after a move of replica 0, replica 1
# at bitwise the same positions and box evaluates 2e-6 relative away from its energy before the move (a fresh context
# on the new boxes gives the new value; host build).  So the fp32 NPT calls are held to the fp32 parity bound, relative
# to sum|E_term|; fp64 keeps the fp64 summation bound.
NPT_REL32 = 1e-5
def barostat_case(dtype, kind):
    """Two replicas of 300 waters (rigid with ``kind``), a move after every second step whose draws are forced: replica
    0 accepts its first move and rejects its second, replica 1 the other way round; the third call ends between moves."""
    from torchmd_b200 import Constraints, Forces, MonteCarloBarostat, System, maxwell_boltzmann, testsystems

    sysd = testsystems.water_box(300, seed=0)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    par64 = testsystems.water_parameters(sysd, precision=F64)
    terms, cfg = ["lj", "electrostatics", "bonds", "angles"], dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    system = System(len(sysd["coords"]), 2, dtype, DEV)
    _two_boxes(system, sysd["coords"], sysd["box"], 2, 1.01)
    torch.manual_seed(5)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, 2))
    case = Case(system, Forces(par, terms=terms, **cfg), par64, terms, cfg, constraints=Constraints(par, kind) if kind else None)
    case.forces.compute(system.pos, system.box, system.forces)
    bar = MonteCarloBarostat(pressure=1.0, frequency=2, seed=1)
    # u_volume 0.9: a 0.8 dV_max expansion; u_accept 0 accepts any move, inf rejects it
    bar.uniforms = lambda r, a: (0.9, 0.0 if (r + a) % 2 == 0 else float("inf"))
    integ = integrator(case, barostat=bar)
    start = torch.diagonal(system.box, dim1=1, dim2=2).cpu().double().numpy().copy()
    boxes = []
    worst_e = worst_k = 0.0
    for k, n in enumerate((2, 2, 3)):
        out = integ.step(n)
        e, ek, ref = check_call(case, integ, out, f"NPT call {k + 1}", rel=NPT_REL32 if dtype == F32 else 1e-10)
        worst_e, worst_k = max(worst_e, e), max(worst_k, ek)
        boxes.append(torch.diagonal(system.box, dim1=1, dim2=2).cpu().double().numpy().copy())
    st = bar.stats()
    # moves after steps 2, 4 and 6 (the third call goes on for a step after its move)
    assert [s["attempted"] for s in st] == [3, 3] and [s["accepted"] for s in st] == [2, 1], st
    # replica 0 took the first move and kept its box at the second, replica 1 the other way round
    assert not np.array_equal(boxes[0][0], start[0]) and np.array_equal(boxes[1][0], boxes[0][0])
    assert np.array_equal(boxes[0][1], start[1]) and not np.array_equal(boxes[1][1], start[1])
    wo = check_oracle(case, ref, f"NPT {dtype} {kind}")
    print(f"barostat {dtype} {kind or 'flexible'}: worst per-term |dE| {worst_e:.2e}, Ekin rel. error {worst_k:.2e}, "
          f"oracle |dE| {wo:.2e}; moves accepted {[s['accepted'] for s in st]}")


@pytest.mark.parametrize("kind", [None, "water"], ids=["flexible", "rigid"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_barostat_energies_describe_the_final_state(dtype, kind):
    barostat_case(dtype, kind)


# ---------------------------------------------------------------------------------------------------- decomposed
def test_decomposed_world1_energies():
    """DecomposedIntegrator with one rank: (Ekin, pot, T) against a fresh evaluation and 0.5 sum m v^2."""
    import os

    import torch.distributed as dist
    from torchmd_b200.domain import DecomposedIntegrator
    from torchmd_b200.integrator import BOLTZMAN

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29571")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device(DEV))
    from test_gpu_domain import _setup

    s, forces = _setup()  # (the system of test_gpu_domain: 1000 waters on full rows)
    case = Case(s, forces, None, forces.energies, {})
    integ = DecomposedIntegrator(s, forces, 1.0, DEV, gamma=LANGEVIN[0], T=LANGEVIN[1])
    for n in (5, 5, 5):
        Ekin, pot, T = integ.step(n)
        ref = fresh(case)[0]
        d = abs(pot[0] - sum(ref.values()))
        want = kinetic64(s, integ.integ.masses)
        ek = float(abs(Ekin[0] - want[0]) / want[0])
        print(f"decomposed world 1, {n} steps: |dE_pot| {d:.2e} kcal/mol, Ekin rel. error {ek:.2e}")
        assert d <= term_bound(ref), (pot, ref)
        assert ek <= EKIN_RTOL[F32], (Ekin, want)
        np.testing.assert_allclose(T, 2.0 * Ekin / (3 * s.natoms * BOLTZMAN), rtol=1e-6)


# ---------------------------------------------------------------------------------------------------- host state
def test_md_steps_host_matches_md_steps(monkeypatch):
    """tmd_md_steps_host (host pos / vel in pinned memory, copied in and out around the steps) against tmd_md_steps from
    the same start on full rows: the final state bitwise, ``energies_host`` / ``ke_host`` equal to the device outputs."""
    from torchmd_b200 import _lib

    monkeypatch.setenv("TMD_B200_CLUSTER", "0")
    L = _L()
    res = []
    for host in (False, True):
        case = water8k(F32)
        s, f = case.system, case.forces
        f.compute(s.pos, s.box, s.forces)
        integ = integrator(case)
        integ._require_cuda()
        ctx = f._ensure_ctx(s.pos)
        f._ensure_box(s.box)
        R = s.nreplicas
        stream = torch.cuda.current_stream(s.pos.device).cuda_stream
        dt, gamma, vcoeff = integ.dt, float(integ.gamma), integ.vcoeff.data_ptr()
        pin = s.pos.is_cuda  # (the host build of the kernels runs on CPU tensors: no pinned memory there)
        for n in (4, 3):
            if host:
                ph, vh = (t.cpu().pin_memory() if pin else t.cpu().clone() for t in (s.pos, s.vel))
                ene = np.zeros((R, _lib.NUM_ENERGIES))
                ke = np.zeros(R)
                _lib.check(L.tmd_md_steps_host(ctx, n, ph.data_ptr(), vh.data_ptr(), s.forces.data_ptr(), integ.masses.data_ptr(),
                                               s.pos.data_ptr(), s.vel.data_ptr(), dt, gamma, vcoeff, SEED, 0,
                                               ene.ctypes.data, ke.ctypes.data, stream))
                state = (ph.clone(), vh.clone())
            else:
                ene_d = torch.zeros((R, _lib.NUM_ENERGIES), dtype=F64, device=DEV)
                ke_d = torch.zeros(R, dtype=F64, device=DEV)
                _lib.check(L.tmd_md_steps(ctx, n, s.pos.data_ptr(), s.vel.data_ptr(), s.forces.data_ptr(), integ.masses.data_ptr(),
                                          dt, gamma, vcoeff, None, SEED, 0, ene_d.data_ptr(), ke_d.data_ptr(), stream))
                ene, ke = ene_d.cpu().numpy(), ke_d.cpu().numpy()
                state = (s.pos.cpu().clone(), s.vel.cpu().clone())
            assert not f.stats()["overflow"]
            res.append((n, state, ene.copy(), ke.copy()))
        assert _L().tmd_pair_kernel(f._ctx) not in (PAIR_CLUSTER, PAIR_EWALD_CLUSTER)
    dev, hst = res[:2], res[2:]
    for (n, (p0, v0), e0, k0), (_, (p1, v1), e1, k1) in zip(dev, hst):
        assert torch.equal(p0, p1) and torch.equal(v0, v1), n
        # (the overlapped bonded kernel adds into the energies with atomics: equal to the order of the fp64 sums)
        for r in range(len(e0)):
            assert np.abs(e0[r] - e1[r]).max() <= 1e-10 * np.abs(e0[r]).sum() + 1e-9, (n, r, e0[r], e1[r])
        assert np.abs(k0 - k1).max() <= 1e-12 * k0.max(), (n, k0, k1)
        assert (e0[:, 5] != 0).all() and (k0 > 0).all()
    print(f"tmd_md_steps_host: 4 + 3 steps bitwise equal to tmd_md_steps; E_pot {dev[-1][2].sum(1)}, ke {dev[-1][3]}")

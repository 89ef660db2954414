"""Parallel tempering on the GPU: per-replica temperatures in the Langevin kernels and replica exchanges on the device.

1. No change without exchanges: a ladder of equal temperatures is the scalar run, and replica k of a ladder run is
   replica k of a scalar run at T[k] with the same seed (bitwise on the full rows and in fp64, within the fp32
   summation bounds on the cluster path).
2. Decisions: every attempt's new ladder is oracle/remd.py's, fed the energies the kernel consumed, the ladder before
   it, the attempt index and the seed; the velocities after it are the oracle's scaling of those before it, bitwise.
   On the fp32 cluster and full-row paths, in fp64, with rigid water, and on the step-by-step path with an external
   term.
3. Graphs: exchanges rewrite the ladder's contents, never its address: the captured steps are not recaptured, and the
   captured k_cstep_boundary reads the new row (draw for draw, after an accepted swap).
4. Sampling of a harmonic system whose potential energy is Gamma distributed.
5. Refusals through the library.

tests/test_remd_on_interpreter.py runs the small cases on the host build of the kernels.
"""
import numpy as np
import pytest
import torch

from oracle import philox
from oracle import remd
from torchmd_b200._lib import PAIR_CLUSTER

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
F32, F64 = torch.float32, torch.float64
SEED = 0x2545F4914F6CDD1D & (2**62 - 1)
TIE = 1e-12  # a decision may differ from the oracle's only where |u - exp(D)| is below this


def _L():
    from torchmd_b200 import _lib

    return _lib.lib()


def _np(dtype):
    return np.float64 if dtype == F64 else np.float32


class Recording:
    """Wraps a ReplicaExchange's ``attempt``: the energies it consumes, the ladder and the velocities before and after
    each attempt (synchronising: test only)."""

    def __init__(self, rex):
        self.rex, self.log = rex, []
        inner = rex.attempt

        def attempt(ctx, energies, stride, nterms):
            integ = rex._integ
            before = (energies.cpu().numpy().copy(), integ._ladder.cpu().numpy().copy(), integ.systems.vel.cpu().numpy().copy(),
                      rex.attempts, stride, nterms)
            inner(ctx, energies, stride, nterms)
            self.log.append(before + (integ._ladder.cpu().numpy().copy(), integ.systems.vel.cpu().numpy().copy()))

        rex.attempt = attempt


def check_decisions(rec, temps, seed, dtype):
    """Every logged attempt against the oracle; returns (attempts, accepted swaps)."""
    accepted = 0
    for ene, lad0, v0, a, stride, nterms, lad1, v1 in rec.log:
        U = remd.potentials(ene, stride, nterms)
        want, factor, tried = remd.exchange(lad0, U, temps, seed, a)
        if not np.array_equal(want, lad1):
            near = [t for t in tried if abs(t[2] - np.exp(t[1])) <= TIE]
            assert near, (a, lad0, want, lad1, tried)
            continue
        accepted += sum(t[3] for t in tried)
        assert np.array_equal(remd.scale(v0, factor, _np(dtype)), v1), a
    return len(rec.log), accepted


# ------------------------------------------------------------------------------------------------------ systems
def cloud_system(dtype, nrep, seed=SEED):
    """The LJ + Coulomb cloud of test_gpu_step_recovery, ``nrep`` replicas with their own thermal velocities."""
    from test_gpu_step_recovery import cloud
    from torchmd_b200 import Forces, System

    spec = cloud(collapsing=(False,) * nrep)
    system = System(spec.natoms, spec.nrep, dtype, DEV)
    system.pos[:] = torch.tensor(spec.coords, dtype=dtype)
    system.vel[:] = torch.tensor(spec.vel, dtype=dtype)
    system.set_box(spec.box)
    forces = Forces(spec.par(dtype, DEV), terms=spec.terms, **spec.cfg)
    forces.compute(system.pos, system.box, system.forces)
    return system, forces


def water_system(dtype, nrep, n=None, cluster=False, rigid=False):
    """Liquid water: the 7992-atom box of test_simt_cluster (cluster lists) or ``n`` molecules of testsystems.water_box;
    Maxwell-Boltzmann velocities drawn per replica."""
    from torchmd_b200 import Constraints, Forces, System, maxwell_boltzmann, testsystems

    if cluster:
        from test_simt_cluster import CFG, TERMS, tiled_water

        sysd = tiled_water(2)
    else:
        from test_gpu_constraints import CFG, TERMS

        sysd = testsystems.water_box(n, seed=0)
    par = testsystems.water_parameters(sysd, precision=dtype, device=DEV)
    natoms = len(sysd["coords"])
    system = System(natoms, nrep, dtype, DEV)
    system.set_positions(np.repeat(np.asarray(sysd["coords"])[:, :, None], nrep, 2))
    system.set_box(np.repeat(np.asarray(sysd["box"], np.float64).reshape(3, 1), nrep, 1))
    torch.manual_seed(3)
    system.set_velocities(maxwell_boltzmann(par.masses, 300.0, nrep))
    forces = Forces(par, terms=TERMS, **CFG)
    forces.compute(system.pos, system.box, system.forces)
    return system, forces, (Constraints(par, "water") if rigid else None)


def run(system, forces, T, calls, gamma=10.0, dt=1.0, seed=SEED, rex=None, constraints=None):
    from torchmd_b200 import Integrator

    integ = Integrator(system, forces, dt, DEV, gamma=gamma, T=T, replica_exchange=rex, constraints=constraints)
    integ.seed = seed
    out = None
    for n in calls:
        out = integ.step(n)
    return integ, out


# ------------------------------------------------------------------------------------------------------ 1. no change
@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32_full_rows", "fp64"])
def test_equal_temperatures_are_the_scalar_run(monkeypatch, dtype):
    """T=[T0]*R against T=T0, 50 steps with in-kernel noise: the same positions and velocities to the bit."""
    from test_gpu_step_recovery import full_rows

    full_rows(monkeypatch)
    a, fa = cloud_system(dtype, 3)
    run(a, fa, 300.0, (50,))
    b, fb = cloud_system(dtype, 3)
    integ, _ = run(b, fb, [300.0] * 3, (50,))
    assert integ.vcoeff.shape == (3, a.natoms, 1)
    if dtype == F32:
        assert _L().tmd_pair_kernel(fb._ctx) != PAIR_CLUSTER
    assert torch.equal(a.pos, b.pos) and torch.equal(a.vel, b.vel)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32_full_rows", "fp64"])
def test_ladder_replica_is_the_scalar_run_at_its_temperature(monkeypatch, dtype):
    """Without exchanges, replica k of a run on the ladder T is replica k of a scalar run at T[k] with the same seed."""
    from test_gpu_step_recovery import full_rows

    full_rows(monkeypatch)
    temps = [300.0, 360.0, 450.0]
    b, fb = cloud_system(dtype, 3)
    run(b, fb, temps, (20, 30))
    for k, t in enumerate(temps):
        a, fa = cloud_system(dtype, 3)
        run(a, fa, t, (20, 30))
        assert torch.equal(a.pos[k], b.pos[k]) and torch.equal(a.vel[k], b.vel[k]), k


def test_equal_temperatures_on_the_cluster_path():
    """The flexible water box on the cluster path (fused steps): T=[T0]*2 against T=T0 within the fp32 bounds of
    test_gpu_langevin_noise (the cluster force sums have no fixed order)."""
    from test_gpu_langevin_noise import POS_TOL32, VEL_TOL32

    out = []
    for T in (300.0, [300.0, 300.0]):
        system, forces, _ = water_system(F32, 2, cluster=True)
        l0 = forces.stats()["kernel_launches"]
        run(system, forces, T, (12,))
        assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
        assert (forces.stats()["kernel_launches"] - l0) / 12 == pytest.approx(4.0 + 1 / 12)  # the fused step
        out.append((system.pos.cpu(), system.vel.cpu()))
    dp, dv = (out[0][0] - out[1][0]).abs().max().item(), (out[0][1] - out[1][1]).abs().max().item()
    print(f"cluster path, equal temperatures against the scalar run: dpos {dp:.2e}, dvel {dv:.2e}")
    assert dp < POS_TOL32 and dv < VEL_TOL32


LADDER_PATHS = ["cluster_fused_7", "cluster_fusestep0", "cluster_overlap0", "full_rows", "no_bonded", "stepwise", "fp64",
                "fp64_stepwise"]


@pytest.mark.parametrize("name", LADDER_PATHS)
def test_ladder_row_on_every_path(monkeypatch, name):
    """The six Langevin kernels read row ladder[r]: the draw-for-draw set-up of test_gpu_langevin_noise (1e20-amu
    waters, gamma 0, distinct per-atom coefficients) with a different vcoeff row per temperature and the ladder [1, 0],
    on the paths that run k_cstep_boundary and k_cvv_second_fold (cluster_fused_7), k_cvv_second_fold (fusestep0),
    k_bonded_vv_second (overlap0), k_vv_second_fold (full_rows), k_vv_second<float> (no_bonded, stepwise) and
    k_vv_second<double> (fp64, fp64_stepwise).  A wrong row moves a velocity by O(vcoeff)."""
    from test_gpu_langevin_noise import PATHS, Hidden, distinct_vcoeff, heavy_water, run_calls, summed_kicks
    from torchmd_b200 import Integrator

    env, calls, terms, stepwise, dtype, kernel, per_step = PATHS[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    system, forces = heavy_water(dtype, terms)
    integ = Integrator(system, Hidden(forces) if stepwise else forces, 1e-3, DEV, gamma=0.0, T=[300.0, 330.0])
    integ.seed = SEED
    n = system.natoms
    integ.vcoeff = torch.stack([distinct_vcoeff(n, dtype), distinct_vcoeff(n, dtype, 1.0, 1.9)]).contiguous()
    integ._ladder.copy_(torch.tensor([1, 0], dtype=torch.int32))
    per = run_calls(integ, forces, calls)
    if kernel is not None:
        assert _L().tmd_pair_kernel(forces._ctx) == kernel
    if per_step is not None:
        assert per == pytest.approx(per_step), per
    nsteps = sum(calls)
    xi = philox.langevin_noise(SEED, nsteps, 2, n, _np(dtype))
    vc = integ.vcoeff.cpu().numpy()[:, :, 0]
    got = system.vel.cpu().numpy().astype(np.float64)
    for r, k in enumerate((1, 0)):
        want, tol = summed_kicks(np.zeros((1, n, 3), _np(dtype)), xi[:, r:r + 1], vc[k])
        dv = np.abs(got[r] - want[0])
        assert (dv <= tol[0]).all(), (name, r, float(dv.max()))
        wrong, _ = summed_kicks(np.zeros((1, n, 3), _np(dtype)), xi[:, r:r + 1], vc[1 - k])
        assert np.abs(got[r] - wrong[0]).max() > 0.1


# ------------------------------------------------------------------------------------------------------ 2. decisions
def decision_case(monkeypatch, name):
    from torchmd_b200 import ReplicaExchange

    temps = [300.0, 302.0, 304.0, 306.0, 308.0]
    constraints, dt, kernel = None, 1.0, None
    if name == "cluster":
        temps = temps[:4]
        system, forces, _ = water_system(F32, 4, cluster=True)
        kernel = PAIR_CLUSTER
    elif name in ("full_rows", "fp64"):
        from test_gpu_step_recovery import full_rows

        full_rows(monkeypatch)
        system, forces = cloud_system(F64 if name == "fp64" else F32, 5)
    elif name == "rigid_water":
        system, forces, constraints = water_system(F64, 5, n=300, rigid=True)
        dt = 2.0
    else:  # the step-by-step path: an external term makes Integrator.step drive tmd_vv_first / tmd_vv_second
        from torchmd_b200 import Forces

        system, f0 = cloud_system(F32, 5)
        forces = Forces(f0.par, terms=f0.terms, external=Tether(system.pos.clone()), **CLOUD_CFG())
        forces.compute(system.pos, system.box, system.forces)
    rex = ReplicaExchange(frequency=3, seed=SEED ^ 0x5A5A)
    rec = Recording(rex)
    integ, (ekin, pot, T) = run(system, forces, temps, (7, 8, 6), rex=rex, constraints=constraints, dt=dt)
    assert rex.attempts == 7 and len(rec.log) == 7
    if kernel is not None:
        assert _L().tmd_pair_kernel(forces._ctx) == kernel
    n, acc = check_decisions(rec, temps, rex.seed, system.pos.dtype)
    print(f"{name}: {n} attempts, {acc} swaps accepted, ladder {rex.ladder().tolist()}, acceptance {rex.acceptance()}")
    assert 0 < acc, "no swap was accepted: the case does not test the scaling"
    # the call ended with an attempt (step 21): the returned kinetic energy is that of the scaled velocities
    from torchmd_b200 import kinetic_energy

    ke = kinetic_energy(integ.masses.double(), system.vel.double()).cpu().numpy().ravel()
    assert np.allclose(ekin, ke, rtol=1e-5 if system.pos.dtype == F32 else 1e-12)
    assert np.array_equal(rex.counts().sum(axis=1) > 0, np.ones(len(temps) - 1, bool))
    return rex


def CLOUD_CFG():
    from test_gpu_step_recovery import cloud

    return cloud(collapsing=(False,)).cfg


class Tether:
    """An external term: a harmonic tether of every atom to its start position, 0.05 kcal/mol/A^2."""

    def __init__(self, ref):
        self.ref = ref

    def calculate(self, pos, box):
        d = pos - self.ref
        return 0.025 * (d * d).sum(dim=(1, 2)), -0.05 * d


@pytest.mark.parametrize("name", ["cluster", "full_rows", "fp64", "rigid_water", "stepwise"])
def test_exchange_decisions_follow_the_oracle(monkeypatch, name):
    decision_case(monkeypatch, name)


# ------------------------------------------------------------------------------------------------------ 3. graphs
def force_swap(integ, rex, ctx):
    """One attempt whose energies make the pair of slots (0, 1) swap (D >= 0), on an even attempt index."""
    R = integ.systems.nreplicas
    if rex.attempts % 2:
        rex.attempt(ctx, torch.zeros((R, 1), dtype=F64, device=DEV), 1, 1)  # (odd: tries no pair of two replicas)
    owner = np.argsort(rex.ladder())
    e = torch.zeros((R, 1), dtype=F64, device=DEV)
    e[int(owner[0]), 0] = 1e6  # the replica at the lower temperature has the higher energy
    rex.attempt(ctx, e, 1, 1)


def test_exchanges_keep_the_captured_steps(monkeypatch):
    """20 exchanges inside the step(n) loop cost no recapture; after an accepted swap the captured k_cstep_boundary of
    the fused cluster step reads the new rows, draw for draw (the noise-only set-up of test_gpu_langevin_noise)."""
    from test_gpu_langevin_noise import distinct_vcoeff, heavy_water, summed_kicks
    from torchmd_b200 import Integrator, ReplicaExchange

    system, forces = heavy_water(F32)
    rex = ReplicaExchange(frequency=2, seed=7)
    integ = Integrator(system, forces, 1e-3, DEV, gamma=0.0, T=[300.0, 330.0], replica_exchange=rex)
    integ.seed = SEED
    n = system.natoms
    integ.vcoeff = torch.stack([distinct_vcoeff(n, F32), distinct_vcoeff(n, F32, 1.0, 1.9)]).contiguous()
    integ.step(2)  # the ladder is set and the steps captured
    c0 = _L().tmd_step_captures(forces._ctx)
    integ.step(40)
    assert rex.attempts == 21 and _L().tmd_step_captures(forces._ctx) == c0
    ctx = forces._ctx
    before = rex.ladder()
    force_swap(integ, rex, ctx)
    ladder = rex.ladder()
    assert np.array_equal(ladder, before[::-1]), (before, ladder)
    system.vel.zero_()
    position = integ._step_index
    rex.frequency = 10**9  # no attempt inside the next call
    l0 = forces.stats()["kernel_launches"]
    integ.step(7)
    assert (forces.stats()["kernel_launches"] - l0) / 7 == pytest.approx(29 / 7)  # k_cstep_boundary between the steps
    assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER and _L().tmd_step_captures(forces._ctx) == c0
    xi = philox.langevin_noise(SEED, 7, 2, n, np.float32, position=position)
    vc = integ.vcoeff.cpu().numpy()[:, :, 0]
    got = system.vel.cpu().numpy().astype(np.float64)
    for r in range(2):
        want, tol = summed_kicks(np.zeros((1, n, 3), np.float32), xi[:, r:r + 1], vc[ladder[r]])
        wrong, _ = summed_kicks(np.zeros((1, n, 3), np.float32), xi[:, r:r + 1], vc[1 - ladder[r]])
        dv = np.abs(got[r] - want[0])
        assert (dv <= tol[0]).all(), (r, float(dv.max()))
        assert np.abs(got[r] - wrong[0]).max() > 0.1  # the other row is far off


# ------------------------------------------------------------------------------------------------------ 4. sampling
def dimers(nrep, ndimers=64, k=1.0, mass=12.0, spacing=30.0):
    """``ndimers`` independent harmonic dimers (r0 = 0, force constant k kcal/mol/A^2, ``mass`` amu): the relative
    coordinate of each is a 3D oscillator, so with no other term U ~ Gamma(3 ndimers / 2, kT)."""
    from torchmd_b200 import Forces, System, TopologyParameters

    n = 2 * ndimers
    g = np.arange(ndimers)
    grid = np.stack([g % 4, (g // 4) % 4, g // 16], axis=1).astype(np.float64) * spacing
    x = np.repeat(grid, 2, axis=0)
    x[1::2, 0] += 0.5
    bonds = (np.stack([2 * g, 2 * g + 1], axis=1), np.stack([g, np.zeros_like(g)], axis=1), np.array([[k, 0.0]]))
    par = TopologyParameters(atom_types=np.zeros(n, np.int64), type_sigma=[1.0], type_epsilon=[0.0], charges=np.zeros(n),
                             masses=np.full(n, mass), bonds=bonds, precision=F64, device=DEV)
    system = System(n, nrep, F64, DEV)
    system.set_positions(np.repeat(x[:, :, None], nrep, 2))
    return system, Forces(par, terms=["bonds"])


def test_sampling_matches_the_gamma_distribution():
    """8 replicas of 64 dimers, ladder 300 * 1.1^k K, gamma 1/ps, 1 fs, an attempt every 100 steps, 200 000 steps (fp64,
    one seeded run).  Per temperature: <U> against 96 kT and <E_kin> against (3N/2) kT (plus the gamma dt / 2 bias of
    the integrator's kinetic temperature), each pair's acceptance against its value for two Gamma(96) distributions,
    all within 5 block standard errors; every replica visits both ends of the ladder."""
    from torchmd_b200 import Integrator, ReplicaExchange, maxwell_boltzmann
    from torchmd_b200.integrator import BOLTZMAN

    R, nd, gamma_ps, dt_fs = 8, 64, 1.0, 1.0
    temps = [300.0 * 1.1**k for k in range(R)]
    system, forces = dimers(R, nd)
    torch.manual_seed(11)
    system.set_velocities(maxwell_boltzmann(forces.par.masses, temps, R))
    forces.compute(system.pos, system.box, system.forces)
    rex = ReplicaExchange(frequency=100, seed=12345)
    integ = Integrator(system, forces, dt_fs, DEV, gamma=gamma_ps, T=temps, replica_exchange=rex)
    integ.seed = 678
    integ.step(10000)  # equilibration: ten friction times
    nchunks = 1900
    U, K = np.zeros((nchunks, R)), np.zeros((nchunks, R))
    counts = np.zeros((nchunks + 1, R - 1, 2))
    counts[0] = rex.counts()
    visits = np.zeros((R, 2), bool)
    lad = rex.ladder()
    for c in range(nchunks):
        ekin, pot, _ = integ.step(100)  # ends with an attempt
        U[c, lad] = pot  # (the positions the attempt found, at the temperatures of the chunk)
        lad = rex.ladder()
        K[c, lad] = ekin  # (the velocities after the attempt's scaling, at their new temperatures)
        counts[c + 1] = rex.counts()
        visits[lad == 0, 0] = True
        visits[lad == R - 1, 1] = True
    kT = BOLTZMAN * np.asarray(temps)
    nb = 19

    def blocks(x):
        b = x.reshape(nb, -1).mean(axis=1)
        return b.mean(), b.std(ddof=1) / np.sqrt(nb)

    bias = gamma_ps * dt_fs * 1e-3 / 2
    for k in range(R):
        mu, se = blocks(U[:, k])
        print(f"T {temps[k]:.1f} K: <U> {mu:.3f} expected {96 * kT[k]:.3f} (se {se:.3f})")
        assert abs(mu - 96 * kT[k]) <= 5 * se, (k, mu, 96 * kT[k], se)
        mk, sk = blocks(K[:, k])
        want = 1.5 * (2 * nd) * kT[k]
        print(f"T {temps[k]:.1f} K: <Ekin> {mk:.3f} expected {want:.3f} (se {sk:.3f})")
        assert abs(mk - want) <= 5 * sk + bias * want, (k, mk, want, sk)
    per_block = np.diff(counts[:: nchunks // nb], axis=0)  # (nb, R-1, 2)
    for k in range(R - 1):
        want = remd.pair_acceptance_gamma(96, kT[k], kT[k + 1])
        rates = per_block[:, k, 1] / per_block[:, k, 0]
        mu, se = rates.mean(), rates.std(ddof=1) / np.sqrt(nb)
        print(f"pair {k}: acceptance {mu:.3f} expected {want:.3f} (se {se:.3f})")
        assert abs(mu - want) <= 5 * se, (k, mu, want, se)
    assert visits.all(), visits


# ------------------------------------------------------------------------------------------------------ 5. refusals
def test_refusals_through_the_library():
    """Both exchange entry points: R > 1024 is TMD_ERR_ARG, a decomposed context TMD_ERR_UNSUPPORTED."""
    import ctypes as C

    from torchmd_b200 import _lib

    L = _L()
    dev = torch.device(DEV).index or 0
    for f64 in (False, True):
        dt = F64 if f64 else F32
        fn = L.tmd_replica_exchange_f64 if f64 else L.tmd_replica_exchange
        for nrep, owned in ((1025, False), (4, True)):
            if owned and f64:  # (fp64 contexts refuse tmd_set_owned_atoms: they cannot be decomposed)
                continue
            h = C.c_void_p()
            _lib.check(L.tmd_create(C.byref(h), dev, 20, nrep))
            try:
                if f64:
                    _lib.check(L.tmd_set_precision(h, 64))
                if owned:
                    _lib.check(L.tmd_set_owned_atoms(h, 0, 10))
                e = torch.zeros((nrep, 1), dtype=F64, device=DEV)
                v = torch.zeros((nrep, 20, 3), dtype=dt, device=DEV)
                counts = torch.zeros((nrep - 1, 2), dtype=torch.int64, device=DEV)
                rc = fn(h, e.data_ptr(), 1, 1, 1, 0, v.data_ptr(), counts.data_ptr(), None)
                assert rc == (_lib.ERR_UNSUPPORTED if owned else -1), (f64, nrep, rc)
                assert int(counts.abs().sum()) == 0
            finally:
                L.tmd_destroy(h)

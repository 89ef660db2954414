"""Replica exchange on the host: the refusals of Integrator / ReplicaExchange, maxwell_boltzmann's draws, the rule of
oracle/remd.py on hand-made cases, and the exchange draws' Philox domain against the Langevin counters."""
import numpy as np
import pytest
import torch

from oracle import philox
from oracle import remd


def _system(nrep, dtype=torch.float32):
    from torchmd_b200 import Forces, System, TopologyParameters

    n = 4
    par = TopologyParameters(atom_types=np.zeros(n, np.int64), type_sigma=[1.0], type_epsilon=[0.1], charges=np.zeros(n),
                             masses=np.full(n, 12.0), bonds=(np.array([[0, 1], [2, 3]]), np.array([[0, 0], [1, 0]]),
                                                             np.array([[1.0, 0.0]])))
    system = System(n, nrep, dtype, "cpu")
    system.set_positions(np.repeat(np.arange(12.0).reshape(4, 3)[:, :, None], nrep, 2))
    system.set_box(np.full((3, nrep), 30.0))
    return system, Forces(par, terms=["bonds"])


def test_refusals():
    from torchmd_b200 import Integrator, MonteCarloBarostat, ReplicaExchange
    from torchmd_b200.domain import DecomposedIntegrator

    system, f = _system(3)
    for kw in (dict(frequency=0), dict(frequency=1.5)):
        with pytest.raises(ValueError):
            ReplicaExchange(**kw)
    with pytest.raises(ValueError, match="sequence"):
        Integrator(system, f, 1.0, "cpu", gamma=1.0, T=300.0, replica_exchange=ReplicaExchange())
    with pytest.raises(ValueError, match="temperatures for 3 replicas"):
        Integrator(system, f, 1.0, "cpu", gamma=1.0, T=[300.0, 310.0], replica_exchange=ReplicaExchange())
    with pytest.raises(ValueError, match="temperatures for 3 replicas"):
        Integrator(system, f, 1.0, "cpu", gamma=1.0, T=[300.0, 310.0])
    for T in ([300.0, 310.0, 305.0], [300.0, 300.0, 310.0]):
        with pytest.raises(ValueError, match="strictly increasing"):
            Integrator(system, f, 1.0, "cpu", gamma=1.0, T=T, replica_exchange=ReplicaExchange())
    one, f1 = _system(1)
    with pytest.raises(ValueError, match="at least two"):
        Integrator(one, f1, 1.0, "cpu", gamma=1.0, T=[300.0], replica_exchange=ReplicaExchange())
    with pytest.raises(RuntimeError, match="thermostat"):
        Integrator(system, f, 1.0, "cpu", T=[300.0, 310.0, 320.0], replica_exchange=ReplicaExchange())
    with pytest.raises(RuntimeError, match="thermostat"):
        Integrator(system, f, 1.0, "cpu", gamma=1.0, replica_exchange=ReplicaExchange())
    with pytest.raises(RuntimeError, match="barostat"):
        Integrator(system, f, 1.0, "cpu", gamma=1.0, T=[300.0, 310.0, 320.0], replica_exchange=ReplicaExchange(),
                   barostat=MonteCarloBarostat())
    with pytest.raises(NotImplementedError, match="per-replica temperatures"):
        DecomposedIntegrator(one, f1, 1.0, "cpu", gamma=1.0, T=[300.0])
    # a sequence without exchanges is allowed; its vcoeff rows are the scalar runs' vcoeff, bitwise
    temps = [300.0, 333.0, 371.5]
    integ = Integrator(system, f, 1.0, "cpu", gamma=1.0, T=temps)
    assert integ.vcoeff.shape == (3, 4, 1) and integ._ladder.tolist() == [0, 1, 2]
    for k, t in enumerate(temps):
        assert torch.equal(integ.vcoeff[k], Integrator(system, f, 1.0, "cpu", gamma=1.0, T=t).vcoeff)


def test_maxwell_boltzmann_scalar_draws_are_unchanged():
    """The scalar call consumes torch's generator as before (the expression of the reference); a sequence draws
    replica r at T[r] from the same stream."""
    from torchmd_b200 import maxwell_boltzmann
    from torchmd_b200.integrator import BOLTZMAN

    masses = torch.tensor([1.008, 12.0, 15.999, 22.99]).view(-1, 1)
    torch.manual_seed(123)
    got = maxwell_boltzmann(masses, 300.0, 3)
    torch.manual_seed(123)
    scale = torch.sqrt(300.0 * BOLTZMAN / masses)
    want = torch.stack([scale * torch.randn((4, 3)).type_as(masses) for _ in range(3)], dim=0)
    assert torch.equal(got, want)
    torch.manual_seed(123)
    seq = maxwell_boltzmann(masses, [300.0, 300.0, 300.0], 3)
    assert torch.equal(seq, want)
    torch.manual_seed(123)
    seq = maxwell_boltzmann(masses, [300.0, 400.0, 500.0], 3)
    torch.manual_seed(123)
    for r, t in enumerate([300.0, 400.0, 500.0]):
        assert torch.equal(seq[r], torch.sqrt(t * BOLTZMAN / masses) * torch.randn((4, 3)).type_as(masses))
    with pytest.raises(ValueError):
        maxwell_boltzmann(masses, [300.0, 400.0], 3)


TEMPS = [300.0, 320.0, 345.0, 370.0, 400.0]


def test_oracle_accepts_every_downhill_swap():
    """D >= 0 (the colder replica has the higher energy) always swaps, whatever the uniform."""
    U = np.array([50.0, 40.0, 30.0, 20.0, 10.0])
    for a in range(6):
        lad, factor, tried = remd.exchange(np.arange(5), U, TEMPS, seed=a, attempt=a)
        assert all(t[3] and t[1] > 0 for t in tried)
        assert [t[0] for t in tried] == list(range(a % 2, 4, 2))
        want = np.arange(5)
        for k in range(a % 2, 4, 2):
            want[k], want[k + 1] = k + 1, k
        assert np.array_equal(lad, want)
        moved = lad != np.arange(5)
        assert np.array_equal(factor[moved], np.sqrt(np.asarray(TEMPS)[lad[moved]] / np.asarray(TEMPS)[moved.nonzero()[0]]))
        assert (factor[~moved] == 1.0).all()
    U = np.zeros(5)  # D = 0: accepted
    assert all(t[3] for t in remd.exchange(np.arange(5), U, TEMPS, 1, 0)[2])


def test_oracle_pairs_alternate_and_odd_ladders_leave_an_end():
    """Even attempts try (0,1), (2,3); odd ones (1,2), (3,4): with R = 5 an even attempt leaves slot 4 alone and an odd
    one slot 0.  Uphill swaps are accepted exactly when u < exp(D); a permuted ladder is read through its inverse."""
    lad0 = np.array([2, 0, 4, 1, 3])
    U = 10.0 * (lad0 + 1)  # every pair uphill: the replica at the colder slot has the lower energy
    owner = np.argsort(lad0)
    for a in (0, 1, 2**32 + 1, 2**40):
        lad, factor, tried = remd.exchange(lad0, U, TEMPS, 99, a)
        ks = [t[0] for t in tried]
        assert ks == ([0, 2] if a % 2 == 0 else [1, 3])
        untouched = 4 if a % 2 == 0 else 0
        assert lad[owner[untouched]] == untouched
        for k, d, u, ok in tried:
            i, j = owner[k], owner[k + 1]
            beta = 1.0 / (remd.BOLTZMAN * np.asarray(TEMPS))
            assert d == (beta[k] - beta[k + 1]) * (U[i] - U[j]) and d < 0
            assert u == remd.uniform(99, a, k) and ok == (u < np.exp(d))
            assert (lad[i], lad[j]) == ((k + 1, k) if ok else (k, k + 1))


def test_oracle_sums_terms_in_order_and_scales_once():
    e = np.array([[1e16, 1.0, -1e16, 0.5], [0.1, 0.2, 0.3, 9.0]])
    U = remd.potentials(e, 4, 3)
    assert U[0] == (1e16 + 1.0) - 1e16 and U[1] == (0.1 + 0.2) + 0.3
    v = np.array([[[1.0, -2.0, 3.0]], [[0.1, 0.2, 0.3]]], np.float32)
    out = remd.scale(v, np.array([1.0, np.sqrt(1.1)]), np.float32)
    assert np.array_equal(out[0], v[0])
    assert np.array_equal(out[1], (v[1].astype(np.float64) * np.sqrt(1.1)).astype(np.float32))


def test_exchange_domain_never_meets_a_langevin_counter():
    """The exchange counter (k, 0x40000000, a lo, a hi): word 1 is 2^30.  A Langevin draw's word 1 is the slot's high
    word (slot = r N + i < 2^62 for any run that fits in memory, so below 2^30), or that word with bit 31 set for the
    second fp64 block: never 2^30."""
    for slot in (0, 2**32 - 1, 2**32, 7 * 2**32 + 5, 2**62 - 1):
        (c0, c1, c2, c3), _ = philox._words(1, 2, slot)
        for w1 in (int(c1), int(c1) | 0x80000000):
            assert w1 != remd.DOMAIN
    assert (2**62 - 1) >> 32 < remd.DOMAIN
    # and the draws differ from the Langevin block on the same words otherwise
    u = remd.uniform(5, 3, 1)
    w = philox.philox4x32_10((1, 0, 3, 0), (5, 0))
    assert u != float(philox.u53(w[0], w[1])) and 0.0 < u < 1.0


def test_pair_acceptance_of_two_gamma_distributions():
    """The quadrature against a Monte Carlo estimate."""
    kt0, kt1 = 0.6, 0.66
    want = remd.pair_acceptance_gamma(96, kt0, kt1)
    rng = np.random.default_rng(0)
    u0, u1 = rng.gamma(96, kt0, 400000), rng.gamma(96, kt1, 400000)
    mc = np.minimum(1.0, np.exp((1 / kt0 - 1 / kt1) * (u0 - u1))).mean()
    assert abs(want - mc) < 3e-3 and 0.2 < want < 0.9

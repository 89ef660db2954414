"""Particle-mesh Ewald checks that need no GPU: the numpy oracle (oracle/pme.py) against the exact Ewald sum and a
known Madelung energy, the parameter choice, and the refusals Forces makes before any device work."""
import math

import numpy as np
import pytest
import torch

from oracle import pme as P


def _random_box(seed, n=40, charged=False):
    rng = np.random.default_rng(seed)
    L = np.array([14.0, 15.0, 16.0])
    pos = rng.uniform(0, 1, (n, 3)) * L
    q = rng.normal(size=n)
    q -= q.mean()
    if charged:
        q += 0.07
    return pos, q, L


def _pairs(pos, L, rc):
    d = pos[:, None, :] - pos[None, :, :]
    d -= L * np.rint(d / L)
    r = np.linalg.norm(d, axis=2)
    i, j = np.nonzero(np.triu(r <= rc, 1))
    return np.stack([i, j], 1)


@pytest.mark.parametrize("seed,charged", [(0, False), (1, False), (2, True), (3, True)])
def test_spme_converges_to_exact_ewald(seed, charged):
    pos, q, L = _random_box(seed, charged=charged)
    Ee, Fe = P.ewald_exact(pos, q, L)
    Ee2, Fe2 = P.ewald_exact(pos, q, L, alpha=0.45)  # the exact sum does not depend on alpha
    assert abs(Ee - Ee2) <= 1e-10 * abs(Ee) and np.abs(Fe - Fe2).max() <= 1e-9
    rc = 6.0
    pairs = _pairs(pos, L, rc)
    errs = []
    for tol in (5e-4, 1e-5, 1e-7):
        a, g = P.choose(rc, L, tol)
        E, F = P.pme(pos, q, L, a, g, pairs, np.zeros((0, 2), np.int64))
        errs.append((abs(E - Ee), np.sqrt(np.mean((F - Fe) ** 2))))
    print(seed, charged, errs)
    for k in range(2):
        assert errs[k + 1][0] < errs[k][0] and errs[k + 1][1] < 0.1 * errs[k][1], errs
    assert errs[2][1] < 1e-6 and errs[2][0] < 1e-6 * abs(Ee)


def test_exclusion_correction_removes_the_excluded_pairs():
    """With excluded pairs the PME total equals the exact Ewald sum minus the plain Coulomb of those pairs
    (minimum image), the convention of the library."""
    pos, q, L = _random_box(4)
    rc = 6.0
    excl = np.array([[0, 1], [2, 3], [3, 2], [5, 9]])  # (3, 2) repeats (2, 3): the set counts it once
    allp = _pairs(pos, L, rc)
    keep = ~np.isin(allp[:, 0] * 1000 + allp[:, 1], [0 * 1000 + 1, 2 * 1000 + 3, 5 * 1000 + 9])
    a, g = P.choose(rc, L, 1e-7)
    E, F = P.pme(pos, q, L, a, g, allp[keep], excl)
    Ee, Fe = P.ewald_exact(pos, q, L)
    for i, j in ((0, 1), (2, 3), (5, 9)):
        d = pos[i] - pos[j]
        d -= L * np.rint(d / L)
        r = np.linalg.norm(d)
        Ee -= q[i] * q[j] / r
        f = q[i] * q[j] * d / r**3
        Fe[i] -= f
        Fe[j] += f
    assert abs(E - Ee) < 1e-6 * abs(Ee) and np.abs(F - Fe).max() < 1e-6


def test_madelung_energy_of_rock_salt():
    from torchmd_b200.forces import ELEC_FACTOR

    pos, q, L = P.madelung_rocksalt(4, 2.8)
    n = len(q)
    want = -n * P.MADELUNG_NACL * ELEC_FACTOR / (2 * 2.8)
    Ee, Fe = P.ewald_exact(pos, q, L, k=ELEC_FACTOR)
    assert abs(Ee / want - 1) <= 1e-10 and np.abs(Fe).max() <= 1e-8
    rc = 9.0
    a, g = P.choose(rc, L, 1e-6)
    E, F = P.pme(pos, q, L, a, g, _pairs(pos, L, rc), np.zeros((0, 2), np.int64), ELEC_FACTOR)
    assert abs(E / want - 1) <= 1e-5, (E, want)


def test_parameter_choice():
    from torchmd_b200 import testsystems

    assert [P.smallest_235(n) for n in (7, 10, 11, 14, 17, 31, 49, 89, 91, 97, 121, 127)] == [8, 10, 12, 15, 18, 32, 50, 90, 96, 100, 125, 128]
    tol, rc = 5e-4, 9.0
    a, g = P.choose(rc, [[100.0, 100.0, 100.0]], tol)
    assert a == math.sqrt(-math.log(2 * tol)) / rc and abs(a - 0.292) < 1e-3 and g == (90, 90, 90)
    # the box of every replica counts: the largest length per axis
    assert P.choose(rc, [[30.0, 50.0, 40.0], [40.0, 20.0, 30.0]], tol)[1] == P.choose(rc, [40.0, 50.0, 40.0], tol)[1]
    assert P.choose(6.0, [[5.0, 5.0, 5.0]], tol)[1] == (10, 10, 10)  # at least 10 points
    for nw, want in ((3333, 45), (33333, 90)):  # water10k and water100k
        L = testsystems.water_box(nw)["box"]
        assert P.choose(rc, L, tol)[1] == (want,) * 3, (nw, L)


def test_forces_refusals():
    from torchmd_b200 import Forces, testsystems

    sysd = testsystems.water_box(20)
    par = testsystems.water_parameters(sysd)
    terms = ["lj", "electrostatics", "bonds", "angles"]
    with pytest.raises(RuntimeError, match="needs a cutoff"):
        Forces(par, terms=terms, pme=True)
    with pytest.raises(RuntimeError, match="exclude each other"):
        Forces(par, terms=terms, pme=True, rfa=True, cutoff=5.0)
    with pytest.raises(RuntimeError, match="electrostatics term"):
        Forces(par, terms=["lj", "bonds"], pme=True, cutoff=5.0)
    with pytest.raises(RuntimeError, match="ewald_tolerance"):
        Forces(par, terms=terms, pme=True, cutoff=5.0, ewald_tolerance=0.0)
    f = Forces(par, terms=terms, cutoff=5.0)
    assert f.pme is False and f.pme_parameters() is None


def test_decomposed_integrator_refuses_pme():
    from torchmd_b200 import Forces, System, testsystems
    from torchmd_b200.domain import DecomposedIntegrator

    sysd = testsystems.water_box(20)
    par = testsystems.water_parameters(sysd)
    system = System(len(sysd["coords"]), 1, torch.float32, "cpu")
    forces = Forces(par, terms=["lj", "electrostatics"], cutoff=4.0, pme=True)
    with pytest.raises(NotImplementedError, match="one GPU"):
        DecomposedIntegrator(system, forces, 1.0, "cpu")

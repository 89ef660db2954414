"""fp64 numpy restatement of the Urey-Bradley 1-3 terms, independent of the library.

A term joins the two end atoms (i, j) of an angle with a harmonic spring on their distance, E = k_ub (r_ij - s0)^2
(CHARMM's convention: no factor 1/2), with the minimum image of a periodic box and no cutoff.
"""
import numpy as np


def energy_forces(pos, idx, k, s0, box=None):
    """(E, F (N,3)) of the terms ``idx`` (n,2) with force constants ``k`` (n,) and distances ``s0`` (n,), fp64."""
    pos = np.asarray(pos, dtype=np.float64)
    idx = np.asarray(idx, dtype=np.int64).reshape(-1, 2)
    k, s0 = np.asarray(k, dtype=np.float64), np.asarray(s0, dtype=np.float64)
    d = pos[idx[:, 1]] - pos[idx[:, 0]]
    if box is not None:
        d = d - box * np.round(d / box)
    r = np.linalg.norm(d, axis=1)
    x = r - s0
    F = np.zeros_like(pos)
    fj = (-2.0 * k * x / r)[:, None] * d  # -dE/dx_j
    np.add.at(F, idx[:, 1], fj)
    np.add.at(F, idx[:, 0], -fj)
    return float(np.sum(k * x * x)), F

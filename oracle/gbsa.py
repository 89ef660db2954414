"""fp64 numpy restatement of Generalized Born implicit solvent, OBC2 (AMBER igb=5, OpenMM GBSAOBCForce conventions),
with the optional ACE non-polar term: Born radii, both energies and analytic forces.  Test infrastructure only, like
oracle/pme.py; the kernels are torchmd_b200/csrc/gbsa.cuh.

Per atom: radius R and screen s, rho = R - 0.09, S = s rho.  For every ordered pair j != i with rho_i < r + S_j,
L = max(rho_i, |r - S_j|), U = r + S_j:
    HCT = 1/L - 1/U + r/4 (1/U^2 - 1/L^2) + 1/(2r) ln(L/U) + S_j^2/(4r) (1/L^2 - 1/U^2)  [+ 2 (1/rho_i - 1/L) engulfed]
psi_i = rho_i/2 sum_j HCT,  B_i = 1 / (1/rho_i - tanh(psi - 0.8 psi^2 + 4.85 psi^3) / R_i).
E_pol = -1/2 k (1 - 1/eps) sum_i sum_j qi qj / f_ij (i = j included, no exclusions), f^2 = r^2 + Bi Bj exp(-r^2/4BiBj).
E_np = sum_i 4 pi sigma (R_i + 1.4)^2 (R_i / B_i)^6.
Restated from the OBC paper (Onufriev, Bashford, Case, Proteins 55, 383 (2004)) and OpenMM's reference platform; not
checked against either engine.
"""
import numpy as np
from scipy import constants as _c

# Coulomb constant in kcal A / (mol e^2), from CODATA values as torchmd_b200.forces.ELEC_FACTOR
COULOMB = _c.elementary_charge**2 / (4 * _c.pi * _c.epsilon_0) / _c.angstrom * _c.Avogadro / (_c.kilo * _c.calorie)
OFFSET = 0.09
ALPHA, BETA, GAMMA = 1.0, 0.8, 4.85
PROBE = 1.4


def hct(r, rho, S):
    """HCT descreening term of a sphere of scaled radius S at distance r from an atom of offset radius rho, and its
    derivative d/dr (broadcasting arrays, r > 0)."""
    r, rho, S = np.broadcast_arrays(np.asarray(r, np.float64), np.asarray(rho, np.float64), np.asarray(S, np.float64))
    U = r + S
    on = rho < U
    d = r - S
    L = np.maximum(rho, np.abs(d))
    lp = np.where(np.abs(d) > rho, np.sign(d), 0.0)  # dL/dr
    with np.errstate(divide="ignore", invalid="ignore"):
        iL, iU, ir = 1.0 / L, 1.0 / U, 1.0 / r
        lnr = np.log(L / U)
        t = iL - iU + 0.25 * r * (iU**2 - iL**2) + 0.5 * ir * lnr + 0.25 * S**2 * ir * (iL**2 - iU**2)
        dt = (-lp * iL**2 + iU**2 + 0.25 * (iU**2 - iL**2) + 0.25 * r * (2 * lp * iL**3 - 2 * iU**3) - 0.5 * ir**2 * lnr
              + 0.5 * ir * (lp * iL - iU) - 0.25 * S**2 * ir**2 * (iL**2 - iU**2) + 0.25 * S**2 * ir * (-2 * lp * iL**3 + 2 * iU**3))
        eng = rho < S - r
        t = t + np.where(eng, 2.0 * (1.0 / rho - iL), 0.0)
        dt = dt + np.where(eng, 2.0 * lp * iL**2, 0.0)
    return np.where(on, t, 0.0), np.where(on, dt, 0.0)


def _rows(n, chunk):
    for a in range(0, n, chunk):
        yield a, min(n, a + chunk)


def born_radii(pos, radius, screen, chunk=512):
    """(B, dB/dI, I) of one configuration pos (N,3)."""
    pos = np.asarray(pos, np.float64)
    radius = np.asarray(radius, np.float64)
    rho = radius - OFFSET
    S = np.asarray(screen, np.float64) * rho
    n = len(pos)
    I = np.zeros(n)
    for a, b in _rows(n, chunk):
        d = pos[a:b, None, :] - pos[None, :, :]
        r = np.sqrt((d * d).sum(-1))
        r[np.arange(b - a), np.arange(a, b)] = 1.0  # (self pairs masked below)
        t, _ = hct(r, rho[a:b, None], S[None, :])
        t[np.arange(b - a), np.arange(a, b)] = 0.0
        I[a:b] = t.sum(1)
    psi = 0.5 * rho * I
    th = np.tanh(psi * (ALPHA - psi * (BETA - GAMMA * psi)))
    B = 1.0 / (1.0 / rho - th / radius)
    dB = B * B * (1.0 - th * th) * (ALPHA - psi * (2 * BETA - 3 * GAMMA * psi)) / radius * 0.5 * rho
    return B, dB, I


def energy_forces(pos, charges, radius, screen, solvent_dielectric=78.5, surface_tension=0.0, coulomb=COULOMB,
                  chunk=512):
    """(E_pol, E_np, forces (N,3)) of one configuration; charges in e, coulomb in kcal A / (mol e^2)."""
    pos = np.asarray(pos, np.float64)
    q = np.asarray(charges, np.float64) * np.sqrt(coulomb)
    radius = np.asarray(radius, np.float64)
    rho = radius - OFFSET
    S = np.asarray(screen, np.float64) * rho
    n = len(pos)
    pref = -(1.0 - 1.0 / solvent_dielectric)
    B, dBdI, _ = born_radii(pos, radius, screen, chunk)
    E = 0.0
    dEdB = np.zeros(n)
    for a, b in _rows(n, chunk):
        d = pos[a:b, None, :] - pos[None, :, :]
        r2 = (d * d).sum(-1)
        D = B[a:b, None] * B[None, :]
        u = r2 / (4.0 * D)
        e = np.exp(-u)
        f = np.sqrt(r2 + D * e)
        qq = q[a:b, None] * q[None, :]
        E += 0.5 * pref * (qq / f).sum()
        dEdB[a:b] = -0.5 * pref * (qq * e * (1.0 + u) * B[None, :] / f**3).sum(1)
    s = radius / B
    enp_i = 4.0 * np.pi * surface_tension * (radius + PROBE) ** 2 * s**6
    dEdB -= 6.0 * enp_i / B
    g = dEdB * dBdI  # dE/dI
    F = np.zeros((n, 3))
    for a, b in _rows(n, chunk):
        d = pos[a:b, None, :] - pos[None, :, :]
        r2 = (d * d).sum(-1)
        idx = np.arange(b - a), np.arange(a, b)
        r2[idx] = 1.0
        r = np.sqrt(r2)
        D = B[a:b, None] * B[None, :]
        e = np.exp(-r2 / (4.0 * D))
        f = np.sqrt(r2 + D * e)
        _, dij = hct(r, rho[a:b, None], S[None, :])
        _, dji = hct(r, rho[None, :], S[a:b, None])
        c = pref * q[a:b, None] * q[None, :] * (1.0 - 0.25 * e) / f**3 - (g[a:b, None] * dij + g[None, :] * dji) / r
        c[idx] = 0.0
        F[a:b] = (c[..., None] * d).sum(1)
    return float(E), float(enp_i.sum()), F

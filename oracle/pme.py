"""Particle-mesh Ewald in numpy fp64 -- TEST INFRASTRUCTURE (the library's PME is checked against it).

Energies in kcal/mol, lengths in A; ``k`` is the Coulomb constant (``ELEC_FACTOR``).  The electrostatic energy with
PME is

    E = sum_{i<j, (i,j) not excluded, r <= rc} k qi qj erfc(a r) / r         real space (the reference's pair set)
      + smooth PME reciprocal energy, cardinal B-splines of order 5           reciprocal space
      - sum_{(i,j) excluded} k qi qj erf(a r) / r    (minimum image)          exclusion correction
      - k a / sqrt(pi) sum qi^2                                               self energy
      - k pi Q^2 / (2 V a^2)                                                  neutralising background

with a and the grid chosen from a tolerance as OpenMM does (``choose``).  ``ewald_exact`` is the classical Ewald sum
converged to 1e-12 for small systems; it checks the smooth PME here, and the library through it.
"""
import math

import numpy as np
from scipy.special import erf, erfc

ORDER = 5


def smallest_235(n):
    """Smallest 2^a 3^b 5^c >= n."""
    m = max(int(n), 1)
    while True:
        k = m
        for p in (2, 3, 5):
            while k % p == 0:
                k //= p
        if k == 1:
            return m
        m += 1


def choose(cutoff, box_lengths, tol=5e-4):
    """(alpha, grid): alpha = sqrt(-ln 2 tol) / rc; n_d = smallest 2^a 3^b 5^c >= max(2 alpha L_d / (3 tol^(1/5)), 10),
    the maximum over the replicas' boxes (box_lengths: (R,3) or (3,))."""
    alpha = math.sqrt(-math.log(2.0 * tol)) / cutoff
    L = np.atleast_2d(np.asarray(box_lengths, np.float64)).max(axis=0)
    grid = tuple(smallest_235(max(math.ceil(2.0 * alpha * float(l) / (3.0 * tol ** 0.2)), 10)) for l in L)
    return alpha, grid


def bspline(w):
    """Order-5 B-spline weights and derivatives of fractional offsets w (M,) -> (M,5), (M,5); weight j belongs to
    grid point floor(u) + j."""
    n = ORDER
    w = np.asarray(w, np.float64)
    d = np.zeros((len(w), n))
    d[:, 0] = 1.0 - w
    d[:, 1] = w
    for j in range(3, n):
        div = 1.0 / (j - 1)
        d[:, j - 1] = div * w * d[:, j - 2]
        for k in range(1, j - 1):
            d[:, j - k - 1] = div * ((w + k) * d[:, j - k - 2] + (j - k - w) * d[:, j - k - 1])
        d[:, 0] = div * (1.0 - w) * d[:, 0]
    dd = np.empty_like(d)
    dd[:, 0] = -d[:, 0]
    dd[:, 1:] = d[:, :-1] - d[:, 1:]
    div = 1.0 / (n - 1)
    d[:, n - 1] = div * w * d[:, n - 2]
    for k in range(1, n - 1):
        d[:, n - k - 1] = div * ((w + k) * d[:, n - k - 2] + (n - k - w) * d[:, n - k - 1])
    d[:, 0] = div * (1.0 - w) * d[:, 0]
    return d, dd


def bspline_moduli(K):
    """|b(m)|^2 of Essmann et al. for m = 0..K-1; the zeros an odd spline order has at m = K/2 take the mean of their
    neighbours (as OpenMM does)."""
    m0, _ = bspline(np.zeros(1))
    c = m0[0]  # M_5(1..4) and 0
    k = np.arange(ORDER)
    mod = np.empty(K)
    for m in range(K):
        s = np.sum(c * np.exp(2j * np.pi * m * k / K))
        mod[m] = abs(s) ** 2
    for m in range(K):
        if mod[m] < 1e-7:
            mod[m] = 0.5 * (mod[(m - 1) % K] + mod[(m + 1) % K])
    return mod


def influence(L, alpha, grid):
    """G(m) (K0,K1,K2) such that E_rec = 1/2 sum_m G(m) |S(m)|^2 for charges that carry sqrt(k)."""
    L = np.asarray(L, np.float64)
    V = float(np.prod(L))
    ms = []
    for d in range(3):
        m = np.arange(grid[d])
        m = np.where(m > grid[d] // 2, m - grid[d], m) / L[d]
        ms.append(m)
    mx, my, mz = np.meshgrid(*ms, indexing="ij")
    m2 = mx * mx + my * my + mz * mz
    B = np.einsum("i,j,k->ijk", *[1.0 / bspline_moduli(grid[d]) for d in range(3)])
    with np.errstate(divide="ignore", invalid="ignore"):
        G = np.exp(-np.pi**2 * m2 / alpha**2) / (np.pi * V * m2) * B
    G[0, 0, 0] = 0.0
    return G


def _splines(pos, L, grid):
    u = np.empty_like(pos)
    for d in range(3):
        f = pos[:, d] / L[d]
        f = f - np.floor(f)
        u[:, d] = f * grid[d]
    i0 = np.floor(u).astype(np.int64)
    w = u - i0
    th, dth = zip(*[bspline(w[:, d]) for d in range(3)])
    return i0, th, dth


def reciprocal(pos, q, L, alpha, grid, k=1.0):
    """Smooth PME reciprocal energy and forces of one box: (E, F (N,3))."""
    pos = np.asarray(pos, np.float64)
    L = np.asarray(L, np.float64)
    qs = np.asarray(q, np.float64) * math.sqrt(k)
    N = len(pos)
    i0, th, dth = _splines(pos, L, grid)
    Q = np.zeros(grid)
    idx = [(i0[:, d][:, None] + np.arange(ORDER)[None, :]) % grid[d] for d in range(3)]
    for a in range(ORDER):
        for b in range(ORDER):
            for c in range(ORDER):
                np.add.at(Q, (idx[0][:, a], idx[1][:, b], idx[2][:, c]), qs * th[0][:, a] * th[1][:, b] * th[2][:, c])
    S = np.fft.fftn(Q)
    G = influence(L, alpha, grid)
    E = 0.5 * float(np.sum(G * np.abs(S) ** 2))
    phi = np.real(np.fft.ifftn(G * S)) * np.prod(grid)
    F = np.zeros((N, 3))
    for a in range(ORDER):
        for b in range(ORDER):
            for c in range(ORDER):
                p = phi[idx[0][:, a], idx[1][:, b], idx[2][:, c]]
                F[:, 0] -= p * dth[0][:, a] * th[1][:, b] * th[2][:, c] * grid[0] / L[0]
                F[:, 1] -= p * th[0][:, a] * dth[1][:, b] * th[2][:, c] * grid[1] / L[1]
                F[:, 2] -= p * th[0][:, a] * th[1][:, b] * dth[2][:, c] * grid[2] / L[2]
    return E, F * qs[:, None]


def _minimg(d, L):
    return d - L * np.rint(d / L)


def real_space(pos, q, L, alpha, pairs, k=1.0):
    """sum over the (P,2) pairs of k qi qj erfc(a r) / r (minimum image): (E, F)."""
    pos = np.asarray(pos, np.float64)
    q = np.asarray(q, np.float64)
    F = np.zeros_like(pos)
    if len(pairs) == 0:
        return 0.0, F
    i, j = np.asarray(pairs).T
    d = _minimg(pos[i] - pos[j], np.asarray(L, np.float64))
    r = np.linalg.norm(d, axis=1)
    qq = k * q[i] * q[j]
    e = qq * erfc(alpha * r) / r
    dedr = -(e + qq * 2.0 * alpha / math.sqrt(math.pi) * np.exp(-(alpha * r) ** 2)) / r
    f = -(dedr / r)[:, None] * d
    np.add.at(F, i, f)
    np.add.at(F, j, -f)
    return float(e.sum()), F


def exclusion_correction(pos, q, L, alpha, pairs, k=1.0):
    """- sum over the excluded pairs of k qi qj erf(a r) / r (minimum image): (E, F).  ``pairs`` (P,2) is taken as a
    set: a pair listed twice (a bond and an angle between the same atoms) counts once."""
    pos = np.asarray(pos, np.float64)
    q = np.asarray(q, np.float64)
    F = np.zeros_like(pos)
    p = np.asarray(pairs, np.int64).reshape(-1, 2)
    p = np.unique(np.sort(p[p[:, 0] != p[:, 1]], axis=1), axis=0)
    if len(p) == 0:
        return 0.0, F
    i, j = p.T
    d = _minimg(pos[i] - pos[j], np.asarray(L, np.float64))
    r = np.linalg.norm(d, axis=1)
    qq = k * q[i] * q[j]
    e = -qq * erf(alpha * r) / r
    dedr = -e / r - qq * 2.0 * alpha / math.sqrt(math.pi) * np.exp(-(alpha * r) ** 2) / r
    f = -(dedr / r)[:, None] * d
    np.add.at(F, i, f)
    np.add.at(F, j, -f)
    return float(e.sum()), F


def self_and_background(q, L, alpha, k=1.0):
    q = np.asarray(q, np.float64)
    V = float(np.prod(L))
    return -k * alpha / math.sqrt(math.pi) * float(np.sum(q * q)) - k * math.pi * float(q.sum()) ** 2 / (2.0 * V * alpha**2)


def pme(pos, q, L, alpha, grid, pairs, excluded, k=1.0):
    """Total PME electrostatic energy and forces of one box (pairs: the real-space pair set)."""
    er, fr = real_space(pos, q, L, alpha, pairs, k)
    ek, fk = reciprocal(pos, q, L, alpha, grid, k)
    ex, fx = exclusion_correction(pos, q, L, alpha, excluded, k)
    return er + ek + ex + self_and_background(q, L, alpha, k), fr + fk + fx


def ewald_exact(pos, q, L, k=1.0, alpha=None, tol=1e-12):
    """Classical Ewald sum of point charges in a periodic box (no exclusions), converged to ``tol``: (E, F)."""
    pos = np.asarray(pos, np.float64)
    q = np.asarray(q, np.float64)
    L = np.asarray(L, np.float64)
    N = len(pos)
    V = float(np.prod(L))
    if alpha is None:
        alpha = 5.6 / float(L.min())
    s = math.sqrt(-math.log(tol))  # erfc(s) ~ exp(-s^2) ~ tol
    rmax = s / alpha + 1e-9
    nimg = [int(math.ceil(rmax / L[d])) + 1 for d in range(3)]
    E = 0.0
    F = np.zeros((N, 3))
    d0 = pos[:, None, :] - pos[None, :, :]
    qq = q[:, None] * q[None, :]
    two_a = 2.0 * alpha / math.sqrt(math.pi)
    for nx in range(-nimg[0], nimg[0] + 1):
        for ny in range(-nimg[1], nimg[1] + 1):
            for nz in range(-nimg[2], nimg[2] + 1):
                d = d0 + np.array([nx, ny, nz]) * L
                r = np.linalg.norm(d, axis=2)
                if nx == 0 and ny == 0 and nz == 0:
                    np.fill_diagonal(r, np.inf)
                m = r < rmax
                if not m.any():
                    continue
                rr = np.where(m, r, 1.0)
                e = np.where(m, qq * erfc(alpha * rr) / rr, 0.0)
                E += 0.5 * e.sum()
                dedr = np.where(m, -(e + qq * two_a * np.exp(-(alpha * rr) ** 2)) / rr, 0.0)
                F -= np.sum((dedr / rr)[:, :, None] * d, axis=1)
    kmax = [int(math.ceil(alpha * s * L[d] / math.pi)) + 1 for d in range(3)]
    mx, my, mz = np.meshgrid(*[np.arange(-kmax[d], kmax[d] + 1) / L[d] for d in range(3)], indexing="ij")
    mv = np.stack([mx.ravel(), my.ravel(), mz.ravel()], 1)
    m2 = np.sum(mv * mv, 1)
    keep = (m2 > 0) & (np.pi**2 * m2 / alpha**2 < s * s + 10)
    mv, m2 = mv[keep], m2[keep]
    ph = 2.0 * np.pi * pos @ mv.T  # (N, M)
    c, sn = np.cos(ph), np.sin(ph)
    Sc, Ss = q @ c, q @ sn
    g = np.exp(-np.pi**2 * m2 / alpha**2) / (np.pi * V * m2)
    E += 0.5 * float(np.sum(g * (Sc * Sc + Ss * Ss)))
    # dE/dr_i = sum_m g q_i 2 pi m (-sin ph_i Sc + cos ph_i Ss)
    t = q[:, None] * (-sn * Sc[None, :] + c * Ss[None, :]) * g[None, :] * 2.0 * np.pi
    F -= t @ mv
    E += self_and_background(q, L, alpha)
    return k * E, k * F


def madelung_rocksalt(n=4, d=2.8):
    """n x n x n conventional cells of rock salt (8 n^3 ions, nearest-neighbour distance d): positions, charges, box."""
    base = np.array([[0, 0, 0], [0, 1, 1], [1, 0, 1], [1, 1, 0]], np.float64)
    pos, q = [], []
    for i in range(n):
        for j in range(n):
            for k in range(n):
                o = np.array([i, j, k], np.float64) * 2
                for b in base:
                    pos.append((o + b) * d)
                    q.append(1.0)
                    pos.append((o + b + np.array([1.0, 0.0, 0.0])) * d)
                    q.append(-1.0)
    L = np.full(3, 2 * n * d)
    return np.array(pos), np.array(q), L


MADELUNG_NACL = 1.747564594633

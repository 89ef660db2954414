"""fp64 numpy restatement of the CMAP correction maps, independent of the library's host code.

A map of resolution n holds E(phi_i, psi_j) at phi_i = -pi + i 2 pi / n (psi alike), phi-major.  CHARMM's interpolation:
dE/dphi and dE/dpsi from periodic cubic splines along each axis, d2E/dphi dpsi from a periodic spline along psi of
dE/dphi (scipy's CubicSpline with periodic boundary conditions here), then the 16 coefficients of the standard bicubic
patch of every cell.  Angles are IUPAC dihedrals; a term (a, b, c, d, e) has phi = dihedral(a, b, c, d) and
psi = dihedral(b, c, d, e).
"""
import numpy as np
from scipy.interpolate import CubicSpline

_M = np.array([[1, 0, 0, 0], [0, 0, 1, 0], [-3, 3, -2, -1], [2, -2, 1, 1]], dtype=np.float64)


def _slopes(y, axis):
    """Derivative in grid units of the periodic cubic spline through y along ``axis`` (at the nodes)."""
    n = y.shape[axis]
    closed = np.concatenate([y, np.take(y, [0], axis=axis)], axis=axis)
    return CubicSpline(np.arange(n + 1.0), closed, axis=axis, bc_type="periodic").derivative()(np.arange(n, dtype=np.float64))


def coefficients(grid):
    """(n, n, 4, 4) bicubic coefficients a[i, j, p, q] of u^p v^q in cell (i, j), u and v its unit coordinates."""
    E = np.asarray(grid, dtype=np.float64)
    du, dv = _slopes(E, 0), _slopes(E, 1)
    duv = _slopes(du, 1)
    r = lambda g: np.roll(g, -1, axis=0)  # noqa: E731  (value at i+1)
    c = lambda g: np.roll(g, -1, axis=1)  # noqa: E731  (value at j+1)
    F = np.empty(E.shape + (4, 4))
    F[..., 0, :] = np.stack([E, c(E), dv, c(dv)], -1)
    F[..., 1, :] = np.stack([r(E), r(c(E)), r(dv), r(c(dv))], -1)
    F[..., 2, :] = np.stack([du, c(du), duv, c(duv)], -1)
    F[..., 3, :] = np.stack([r(du), r(c(du)), r(duv), r(c(duv))], -1)
    return _M @ F @ _M.T


def map_energy(coef, phi, psi):
    """E, dE/dphi, dE/dpsi of one map's coefficients at angles phi, psi (radians, arrays)."""
    n = coef.shape[0]
    h = 2 * np.pi / n
    x, y = (np.asarray(phi) + np.pi) / h, (np.asarray(psi) + np.pi) / h
    fx, fy = np.floor(x), np.floor(y)
    u, v = x - fx, y - fy
    a = coef[fx.astype(np.int64) % n, fy.astype(np.int64) % n]
    up = np.stack([np.ones_like(u), u, u * u, u**3], -1)
    vp = np.stack([np.ones_like(v), v, v * v, v**3], -1)
    dup = np.stack([np.zeros_like(u), np.ones_like(u), 2 * u, 3 * u * u], -1)
    dvp = np.stack([np.zeros_like(v), np.ones_like(v), 2 * v, 3 * v * v], -1)
    E = np.einsum("...p,...pq,...q->...", up, a, vp)
    return E, np.einsum("...p,...pq,...q->...", dup, a, vp) / h, np.einsum("...p,...pq,...q->...", up, a, dvp) / h


def _image(d, box):
    return d if box is None else d - box * np.round(d / box)


def dihedral(x0, x1, x2, x3, box=None):
    """IUPAC dihedral angles of (N,3) position arrays and their gradients with respect to the four atoms."""
    b1, b2, b3 = _image(x1 - x0, box), _image(x2 - x1, box), _image(x3 - x2, box)
    m, n = np.cross(b1, b2), np.cross(b2, b3)
    nb2 = np.linalg.norm(b2, axis=-1)
    phi = np.arctan2(nb2 * np.einsum("...k,...k", b1, n), np.einsum("...k,...k", m, n))
    g0 = -(nb2 / np.einsum("...k,...k", m, m))[..., None] * m
    g3 = (nb2 / np.einsum("...k,...k", n, n))[..., None] * n
    s1 = (np.einsum("...k,...k", b1, b2) / nb2**2)[..., None]
    s3 = (np.einsum("...k,...k", b3, b2) / nb2**2)[..., None]
    g1 = -(1 + s1) * g0 + s3 * g3  # (Blondel & Karplus 1996, in these bond vectors)
    g2 = -(g0 + g1 + g3)
    return phi, (g0, g1, g2, g3)


def energy_forces(pos, idx, map_of, res, grids, box=None):
    """Total CMAP energy and (N,3) forces of one configuration.  pos (N,3); idx (n,5); map_of (n,); res (nmaps,);
    grids flat, phi-major maps one after another; box: (3,) lengths for the minimum image, or None."""
    pos = np.asarray(pos, dtype=np.float64)
    idx, map_of, res = np.asarray(idx, np.int64), np.asarray(map_of, np.int64), np.asarray(res, np.int64)
    grids = np.asarray(grids, dtype=np.float64).reshape(-1)
    box = None if box is None or not np.any(box) else np.asarray(box, dtype=np.float64)
    off = np.concatenate([[0], np.cumsum(res * res)])
    x = [pos[idx[:, k]] for k in range(5)]
    phi, gphi = dihedral(x[0], x[1], x[2], x[3], box)
    psi, gpsi = dihedral(x[1], x[2], x[3], x[4], box)
    E = np.zeros(len(idx))
    dphi, dpsi = np.zeros(len(idx)), np.zeros(len(idx))
    for m in range(len(res)):
        sel = map_of == m
        if sel.any():
            coef = coefficients(grids[off[m] : off[m + 1]].reshape(res[m], res[m]))
            E[sel], dphi[sel], dpsi[sel] = map_energy(coef, phi[sel], psi[sel])
    F = np.zeros_like(pos)
    for k in range(4):
        np.add.at(F, idx[:, k], -dphi[:, None] * gphi[k])
        np.add.at(F, idx[:, k + 1], -dpsi[:, None] * gpsi[k])
    return float(E.sum()), F

"""The fp64 Generalized Born oracle (oracle/gbsa.py) pinned on its own: the HCT pair term against a quadrature of the
descreening integral, the single-ion and far-apart-ions limits, and its analytic forces against central finite
differences of its energy and against an independently written torch-autograd energy."""
import numpy as np
import pytest
import torch
from scipy import integrate

from conftest import load_golden
from oracle import gbsa

K = gbsa.COULOMB


def descreening_integral(r, rho, S):
    """(1/4 pi) integral of |x|^-4 over the part of a sphere of radius S centred r away that lies outside radius rho,
    by quadrature over shells |x| = t: the shell's fraction inside the sphere is (S^2 - (t - r)^2) / (4 t r) where it
    cuts the sphere, 1 where the sphere holds it whole."""
    def frac(t):
        if t + r <= S:
            return 1.0
        if t >= r + S or t <= r - S:
            return 0.0
        return (S * S - (t - r) ** 2) / (4.0 * t * r)

    lo, hi = rho, r + S
    if hi <= lo:
        return 0.0
    pts = sorted(p for p in (abs(r - S), S - r) if lo < p < hi)
    total, a = 0.0, lo
    for b in pts + [hi]:
        v, _ = integrate.quad(lambda t: frac(t) / (t * t), a, b, epsabs=0.0, epsrel=1e-13, limit=200)
        total += v
        a = b
    return total


@pytest.mark.parametrize("r,rho,S", [
    (6.0, 1.41, 1.2),    # separated, small x
    (2.2, 1.21, 1.5),    # separated, x near 0.7
    (1.5, 1.61, 1.3),    # overlapping, L = rho
    (0.9, 1.21, 1.4),    # overlapping, j's centre inside i
    (0.3, 0.71, 1.6),    # i engulfed in j
    (0.05, 1.0, 1.5),    # i engulfed, nearly concentric
    (0.5, 1.61, 0.9),    # j inside rho: no term
])
def test_hct_term_is_the_descreening_integral(r, rho, S):
    t, _ = gbsa.hct(r, rho, S)
    want = 2.0 * descreening_integral(r, rho, S)
    assert abs(float(t) - want) <= 1e-8 * max(abs(want), 1e-300), (float(t), want)


@pytest.mark.parametrize("r,rho,S", [(6.0, 1.41, 1.2), (1.5, 1.61, 1.3), (0.3, 0.71, 1.6), (2.2, 1.21, 1.5)])
def test_hct_derivative(r, rho, S):
    h = 1e-6
    _, d = gbsa.hct(r, rho, S)
    fd = (gbsa.hct(r + h, rho, S)[0] - gbsa.hct(r - h, rho, S)[0]) / (2 * h)
    assert abs(float(d) - float(fd)) <= 1e-7 * abs(float(d)), (float(d), float(fd))


def test_single_ion():
    for q, R, eps in ((1.0, 1.5, 78.5), (-2.0, 2.3, 4.0)):
        B, _, I = gbsa.born_radii(np.zeros((1, 3)), [R], [0.8])
        assert I[0] == 0.0 and B[0] == R - 0.09
        E, _, F = gbsa.energy_forces(np.zeros((1, 3)), [q], [R], [0.8], solvent_dielectric=eps)
        want = -0.5 * K * (1 - 1 / eps) * q * q / (R - 0.09)
        assert abs(E - want) <= 4e-16 * abs(want)  # (the charges carry sqrt(k): k q^2 to rounding)
        assert not F.any()


def test_far_ions_give_screened_coulomb():
    q, R, eps = np.array([1.0, -1.0]), np.array([1.7, 1.5]), 78.5
    for r in (40.0, 80.0):
        pos = np.array([[0.0, 0.0, 0.0], [r, 0.0, 0.0]])
        E, _, _ = gbsa.energy_forces(pos, q, R, [0.8, 0.85], solvent_dielectric=eps)
        B, _, _ = gbsa.born_radii(pos, R, [0.8, 0.85])
        self_terms = -0.5 * K * (1 - 1 / eps) * (q * q / B).sum()
        total = E - self_terms + K * q[0] * q[1] / r
        want = K * q[0] * q[1] / (eps * r)
        assert abs(total - want) <= 1e-10 * abs(want), (total, want)


def _system(name):
    g = load_golden(name + "_amber_nocut")
    gb = load_golden("gb_radii")
    return g["coords_replicas"].astype(np.float64), g["par_charges"], gb[name + "_radii"], gb[name + "_screen"]


def _torch_energy(pos, q, radius, screen, eps, sigma):
    """OBC2 written again in torch, from the formulas, for autograd."""
    rho = radius - 0.09
    S = screen * rho
    n = len(q)
    d = pos[:, None, :] - pos[None, :, :]
    eye = torch.eye(n, dtype=torch.bool)
    r2 = (d * d).sum(-1)
    r = torch.sqrt(torch.where(eye, torch.ones_like(r2), r2))
    rho_i, S_j = rho[:, None].expand(n, n), S[None, :].expand(n, n)
    U = r + S_j
    L = torch.maximum(rho_i, torch.abs(r - S_j))
    on = (rho_i < U) & ~eye
    Ls, Us = torch.where(on, L, torch.ones_like(L)), torch.where(on, U, 2 * torch.ones_like(U))
    t = 1 / Ls - 1 / Us + r / 4 * (1 / Us**2 - 1 / Ls**2) + torch.log(Ls / Us) / (2 * r) + S_j**2 / (4 * r) * (1 / Ls**2 - 1 / Us**2)
    t = t + torch.where(rho_i < S_j - r, 2 * (1 / rho_i - 1 / Ls), torch.zeros_like(t))
    psi = 0.5 * rho * torch.where(on, t, torch.zeros_like(t)).sum(1)
    B = 1 / (1 / rho - torch.tanh(psi - 0.8 * psi**2 + 4.85 * psi**3) / radius)
    D = B[:, None] * B[None, :]
    f = torch.sqrt(r2 + D * torch.exp(-r2 / (4 * D)))
    qk = q * np.sqrt(K)
    e_pol = -0.5 * (1 - 1 / eps) * (qk[:, None] * qk[None, :] / f).sum()
    e_np = (4 * np.pi * sigma * (radius + 1.4) ** 2 * (radius / B) ** 6).sum()
    return e_pol + e_np


@pytest.mark.parametrize("name", ["ligand", "benzamidine"])
@pytest.mark.parametrize("sigma", [0.0, 0.0054])
def test_forces_are_the_gradient(name, sigma):
    coords, q, radius, screen = _system(name)
    eps = 78.5
    for pos in coords:
        E, Enp, F = gbsa.energy_forces(pos, q, radius, screen, eps, sigma)
        fmax = np.abs(F).max()
        p = torch.tensor(pos, requires_grad=True)
        Et = _torch_energy(p, torch.tensor(q), torch.tensor(radius), torch.tensor(screen), eps, sigma)
        assert abs(Et.item() - (E + Enp)) <= 1e-12 * abs(E + Enp)
        Et.backward()
        assert np.abs(-p.grad.numpy() - F).max() <= 1e-7 * fmax
        h = 1e-5
        fd = np.zeros_like(F)
        for i in range(len(pos)):
            for k in range(3):
                pp, pm = pos.copy(), pos.copy()
                pp[i, k] += h
                pm[i, k] -= h
                ep = sum(gbsa.energy_forces(pp, q, radius, screen, eps, sigma)[:2])
                em = sum(gbsa.energy_forces(pm, q, radius, screen, eps, sigma)[:2])
                fd[i, k] = -(ep - em) / (2 * h)
        assert np.abs(fd - F).max() <= 1e-7 * fmax, np.abs(fd - F).max() / fmax


def test_thrombin_takes_seconds():
    import time

    g = load_golden("thrombin_nobox_rf")
    gb = load_golden("gb_radii")
    t0 = time.perf_counter()
    E, Enp, F = gbsa.energy_forces(g["coords"], g["par_charges"], gb["thrombin_radii"], gb["thrombin_screen"], 78.5, 0.0054)
    assert time.perf_counter() - t0 < 60.0
    assert np.isfinite(F).all() and E < 0 and Enp > 0
    assert abs(F.sum(0)).max() <= 1e-8 * np.abs(F).max() * len(F)  # Newton's third law

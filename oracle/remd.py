"""Temperature replica exchange restated in numpy: the rule of ``k_remd_exchange`` and ``k_remd_scale``
(``torchmd_b200/csrc/remd.cuh``), for tests.

Written from the Metropolis criterion of parallel tempering (Sugita and Okamoto, Chem. Phys. Lett. 314, 141 (1999);
Earl and Deem, PCCP 7, 3910 (2005)) and from the device code.  Replica r holds temperature slot ``ladder[r]``; an
attempt ``a`` tries the pairs of slots (k, k+1) with k = a (mod 2), held by replicas i = owner[k] and j = owner[k+1]:

    D = (beta_k - beta_{k+1}) * (U_i - U_j),  beta = 1 / (BOLTZMAN * T)
    accept when D >= 0, otherwise when u < exp(D)

with ``u = u53(x, y)`` of Philox4x32-10 on the counter (k, DOMAIN, a lo, a hi) under the key ``seed``.  The Langevin
draws (oracle/philox.py) put the slot's high word in counter word 1, below 2^30 for any run that fits in memory (and
set bit 31 for the fp64 second block), so the two streams never share a counter.  Every tried pair draws.

Agreement with the device: the energy sums (one fp64 addition per term, in term order), beta, D, u and the velocity
factors sqrt(T_new / T_old) are exactly rounded operations and agree bitwise; ``exp`` is within an ulp, so a decision
can differ only where |u - exp(D)| is of the order of 1e-16.
"""
import numpy as np

from . import philox

BOLTZMAN = 0.001987191  # kcal/(mol K), the integrator's
DOMAIN = 0x40000000  # counter word 1 of the exchange draws
MAX_REPLICAS = 1024


def uniform(seed, attempt, k):
    """The uniform of pair (k, k+1) at attempt ``attempt``."""
    a = int(attempt) % (1 << 64)
    s = int(seed) % (1 << 64)
    w = philox.philox4x32_10((k, DOMAIN, a & 0xFFFFFFFF, a >> 32), (s & 0xFFFFFFFF, s >> 32))
    return float(philox.u53(w[0], w[1]))


def potentials(energies, stride, nterms):
    """U_r = sum_{t < nterms} energies[r*stride + t], added one term at a time in term order (fp64)."""
    e = np.asarray(energies, dtype=np.float64).ravel()
    R = len(e) // stride
    out = np.zeros(R)
    for r in range(R):
        acc = 0.0
        for t in range(nterms):
            acc += float(e[r * stride + t])
        out[r] = acc
    return out


def exchange(ladder, U, temps, seed, attempt):
    """One attempt.  Returns (new ladder, per-replica velocity factor, tried) with ``tried`` a list of
    (k, D, u, accepted) per pair of slots tried."""
    ladder = np.asarray(ladder, dtype=np.int64)
    R = len(ladder)
    temps = np.asarray(temps, dtype=np.float64)
    owner = np.empty(R, dtype=np.int64)
    owner[ladder] = np.arange(R)
    new = ladder.copy()
    tried = []
    for k in range(int(attempt) % 2, R - 1, 2):
        i, j = int(owner[k]), int(owner[k + 1])
        bk, bk1 = 1.0 / (BOLTZMAN * temps[k]), 1.0 / (BOLTZMAN * temps[k + 1])
        d = (bk - bk1) * (float(U[i]) - float(U[j]))
        u = uniform(seed, attempt, k)
        ok = bool(d >= 0.0 or u < np.exp(d))
        tried.append((k, d, u, ok))
        if ok:
            new[i], new[j] = k + 1, k
    factor = np.ones(R)
    moved = new != ladder
    factor[moved] = np.sqrt(temps[new[moved]] / temps[ladder[moved]])
    return new, factor, tried


def scale(vel, factor, dtype):
    """``k_remd_scale``: v = dtype(float64(v) * factor[r]) for the replicas whose factor is not 1."""
    v = np.array(vel, dtype=dtype, copy=True)
    for r, f in enumerate(factor):
        if f != 1.0:
            v[r] = (v[r].astype(np.float64) * f).astype(dtype)
    return v


def pair_acceptance_gamma(shape, kT_lo, kT_hi):
    """The mean acceptance of swaps between two temperatures whose potential energies are Gamma(shape, kT) distributed
    (a harmonic system with 2 * shape degrees of freedom): E[min(1, exp((1/kT_lo - 1/kT_hi)(U_lo - U_hi)))] with
    U_lo ~ Gamma(shape, kT_lo), U_hi ~ Gamma(shape, kT_hi) independent, by quadrature."""
    from scipy import integrate, stats

    db = 1.0 / kT_lo - 1.0 / kT_hi
    lo, hi = stats.gamma(shape, scale=kT_lo), stats.gamma(shape, scale=kT_hi)

    def inner(u_hi):
        # P(accept | U_hi): 1 for U_lo >= U_hi, exp(db (U_lo - U_hi)) below
        below = integrate.quad(lambda x: np.exp(db * (x - u_hi)) * lo.pdf(x), 0.0, u_hi, limit=200)[0]
        return (below + lo.sf(u_hi)) * hi.pdf(u_hi)

    top = hi.ppf(1 - 1e-12)
    return integrate.quad(inner, 0.0, top, limit=200)[0]

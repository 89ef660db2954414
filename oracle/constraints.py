"""fp64 numpy reference for holonomic constraints (rigid water, X-H bonds): what the constraint kernels
(torchmd_b200/csrc/constrain.cuh) are checked against.

The algorithms differ from the kernels on purpose, so that agreement is evidence:
* positions: every group is solved by Newton iteration on its Lagrange multipliers with the full group
  Jacobian (the kernels run Gauss-Seidel SHAKE), to |r - d| < 1e-13 A;
* velocities: the group's linear system is solved with numpy.linalg.solve.
Groups are unwrapped around their first atom with the minimum image; each atom's displacement is added
to its own image.
"""
import numpy as np
import torch

from .refmd import TIMEFACTOR, PICOSEC2TIMEU, BOLTZMAN

TOL = 1e-13


def groups_of(con):
    """[(atoms, [(local a, local b, d), ...])] of a torchmd_b200 ``Constraints`` object."""
    out = []
    for w, (doh, dhh) in zip(con.water_idx, con.water_d):
        out.append((list(map(int, w)), [(0, 1, float(doh)), (0, 2, float(doh)), (1, 2, float(dhh))]))
    for c in range(con.nclusters):
        lo, hi = int(con.cluster_ptr[c]), int(con.cluster_ptr[c + 1])
        atoms = list(map(int, con.cluster_idx[lo:hi]))
        out.append((atoms, [(0, k + 1, float(con.cluster_d[lo - c + k])) for k in range(hi - lo - 1)]))
    return out


def _unwrap(x, atoms, L):
    p = x[atoms].astype(np.float64).copy()
    if L is not None:
        d = p[1:] - p[0]
        p[1:] = p[0] + np.where(L > 0, d - L * np.rint(d / np.where(L > 0, L, 1.0)), d)
    return p


def _box(box, r):
    if box is None:
        return None
    L = np.asarray(box, np.float64).reshape(-1, 3)[r]
    return L if np.any(L > 0) else None


def constrain_positions(pos, ref, masses, groups, box=None):
    """Solve every group's distance constraints (R,N,3 float64 arrays); returns (new positions, displacement)."""
    pos = np.array(pos, np.float64)
    disp = np.zeros_like(pos)
    im_all = 1.0 / np.asarray(masses, np.float64).reshape(-1)
    for r in range(pos.shape[0]):
        L = _box(box, r)
        for atoms, cons in groups:
            x0 = _unwrap(pos[r], atoms, L)
            q = _unwrap(ref[r], atoms, L)
            im = im_all[atoms]
            G = np.zeros((len(cons), len(atoms), 3))  # direction of multiplier l on each atom (reference vectors)
            for l, (a, b, _) in enumerate(cons):
                G[l, a] = q[a] - q[b]
                G[l, b] = -(q[a] - q[b])
            d = np.array([c[2] for c in cons])
            lam = np.zeros(len(cons))
            for _ in range(100):
                x = x0 + np.einsum("l,lik->ik", lam, G) * im[:, None]
                rv = np.array([x[a] - x[b] for a, b, _ in cons])
                F = np.einsum("lk,lk->l", rv, rv) - d * d
                if np.all(np.abs(np.sqrt(np.einsum("lk,lk->l", rv, rv)) - d) < TOL):
                    break
                J = np.zeros((len(cons), len(cons)))
                for k, (a, b, _) in enumerate(cons):
                    J[k] = 2.0 * np.einsum("k,lk->l", rv[k], im[a] * G[:, a] - im[b] * G[:, b])
                lam -= np.linalg.solve(J, F)
            else:
                raise RuntimeError(f"Newton did not converge for group {atoms}")
            dx = x - x0
            pos[r, atoms] += dx
            disp[r, atoms] = dx
    return pos, disp


def constrain_velocities(pos, vel, masses, groups, box=None):
    """Remove every constrained bond's relative velocity along it (exact linear solve per group)."""
    vel = np.array(vel, np.float64)
    im_all = 1.0 / np.asarray(masses, np.float64).reshape(-1)
    for r in range(pos.shape[0]):
        L = _box(box, r)
        for atoms, cons in groups:
            x = _unwrap(pos[r], atoms, L)
            v = vel[r, atoms]
            im = im_all[atoms]
            G = np.zeros((len(cons), len(atoms), 3))
            for l, (a, b, _) in enumerate(cons):
                G[l, a] = x[a] - x[b]
                G[l, b] = -(x[a] - x[b])
            M = np.einsum("kia,lia,i->kl", G, G, im)
            lam = np.linalg.solve(M, -np.einsum("kia,ia->k", G, v))
            vel[r, atoms] = v + np.einsum("l,lia->ia", lam, G) * im[:, None]
    return vel


def residuals(pos, vel, groups, box=None):
    """(max |r - d|, max |(v_a - v_b) . r_hat|) over every constraint."""
    pos = np.asarray(pos, np.float64)
    vel = np.asarray(vel, np.float64)
    a = np.array([atoms[c[0]] for atoms, cons in groups for c in cons], np.int64)
    b = np.array([atoms[c[1]] for atoms, cons in groups for c in cons], np.int64)
    d = np.array([c[2] for _, cons in groups for c in cons])
    er, ev = 0.0, 0.0
    for r in range(pos.shape[0]):
        L = _box(box, r)
        rv = pos[r, a] - pos[r, b]
        if L is not None:
            rv = np.where(L > 0, rv - L * np.rint(rv / np.where(L > 0, L, 1.0)), rv)
        n = np.linalg.norm(rv, axis=1)
        er = max(er, float(np.abs(n - d).max()))
        ev = max(ev, float(np.abs(np.einsum("ck,ck->c", vel[r, a] - vel[r, b], rv) / n).max()))
    return er, ev


class OracleConstrainedIntegrator:
    """refmd.OracleIntegrator with RATTLE: half-kick + drift, position constraint against the pre-drift
    positions (velocity += displacement / dt), force call, Langevin kick, second half-kick, velocity constraint.
    State: float64 torch tensors (R,N,3)."""

    def __init__(self, pos, vel, box, forces_buf, masses, force_fn, timestep_fs, groups, gamma_ps=None, T=None):
        self.pos, self.vel, self.box, self.f = pos, vel, box, forces_buf
        self.masses = masses.view(-1, 1).double()
        self.force_fn = force_fn
        self.groups = groups
        self.dt = timestep_fs / TIMEFACTOR
        self.gamma = gamma_ps / PICOSEC2TIMEU if gamma_ps is not None else None
        self.T = T
        if T:
            self.vcoeff = torch.sqrt(2.0 * self.gamma / self.masses * BOLTZMAN * T * self.dt)
        self._boxnp = None if box is None else torch.diagonal(box, dim1=-2, dim2=-1).numpy() if box.dim() == 3 else box.numpy()

    def project(self):
        m = self.masses.numpy().reshape(-1)
        p, _ = constrain_positions(self.pos.numpy(), self.pos.numpy(), m, self.groups, self._boxnp)
        self.pos.copy_(torch.from_numpy(p))
        self.vel.copy_(torch.from_numpy(constrain_velocities(p, self.vel.numpy(), m, self.groups, self._boxnp)))

    def step(self, niter=1, noise=None):
        dt, m = self.dt, self.masses
        mn = m.numpy().reshape(-1)
        pot = None
        for it in range(niter):
            ref = self.pos.numpy().copy()
            acc = self.f / m
            self.pos += self.vel * dt + 0.5 * acc * dt * dt
            self.vel += 0.5 * dt * acc
            p, dx = constrain_positions(self.pos.numpy(), ref, mn, self.groups, self._boxnp)
            self.pos.copy_(torch.from_numpy(p))
            self.vel += torch.from_numpy(dx) / dt
            pot = self.force_fn(self.pos, self.box, self.f)
            if self.T:
                xi = noise[it] if noise is not None else torch.randn_like(self.vel)
                self.vel += -self.gamma * self.vel * dt + xi * self.vcoeff
            self.vel += 0.5 * dt * (self.f / m)
            self.vel.copy_(torch.from_numpy(constrain_velocities(self.pos.numpy(), self.vel.numpy(), mn, self.groups, self._boxnp)))
        ekin = torch.sum(0.5 * m * torch.sum(self.vel * self.vel, dim=2, keepdim=True), dim=1).flatten().numpy()
        return ekin, pot

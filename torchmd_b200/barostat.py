"""``MonteCarloBarostat``: constant pressure (NPT) for ``Integrator`` by Monte Carlo volume moves.

Every ``frequency`` steps each replica attempts an isotropic volume change (OpenMM's MonteCarloBarostat):

1. draw dV uniform in [-dV_max, dV_max], s = ((V + dV) / V)^(1/3);
2. move every molecule rigidly with its centroid by s (``tmd_scale_molecules``, csrc/barostat.cuh) and give the
   context the scaled box (``tmd_rescale_box``: in stream order, no re-finalisation, the captured steps stay valid;
   ``tmd_set_box`` when the box cannot take that path);
3. one energy + force evaluation at the trial state, into a scratch force buffer;
4. accept with probability min(1, exp(-w / kT)), w = dE + P dV - N_mol kT ln(V' / V);
5. accepted: the scratch forces become ``systems.forces`` and the box is written into ``systems.box``;
   rejected: positions, velocities and box go back to what they were, bitwise; ``systems.forces`` was never touched.

Every 10 attempts of a replica dV_max is adapted as OpenMM does: x0.9 below 25 % acceptance, x1.1 above 75 %,
at most 0.3 V.  Molecules are the connected components of the bond graph; velocities are not scaled (with constraints they
are projected at the moved positions).
Replicas are independent: each has its own box, random stream, dV_max and decision.
"""
import math
from collections import deque

import numpy as np
import torch

from . import _lib

# 1 bar = 1e5 Pa = 1e5 J/m^3.  Per mole: 1e5 J/m^3 * 6.02214076e23 / mol * 1e-30 m^3/A^3 = 6.02214076e-2 J/(mol A^3),
# and / 4184 J/kcal = 1.43933e-5 kcal/(mol A^3).
BAR_TO_KCAL_PER_MOL_A3 = 1e5 * 6.02214076e23 * 1e-30 / 4184.0
BOLTZMAN = 0.001987191  # kcal/(mol K), as in integrator.py


def acceptance_work(dE, dV, V, pressure_bar, nmol, kT):
    """w = dE + P dV - N_mol kT ln((V + dV) / V) in kcal/mol (P in bar, V in A^3)."""
    return dE + pressure_bar * BAR_TO_KCAL_PER_MOL_A3 * dV - nmol * kT * math.log((V + dV) / V)


def accept(w, kT, u):
    """Metropolis: accept when u < min(1, exp(-w / kT)), u uniform in [0, 1) (u = inf rejects any move)."""
    return u < (1.0 if w <= 0.0 else math.exp(-w / kT))


def adapt_dv_max(dv_max, attempted, accepted, volume):
    """OpenMM's adaptation after a batch of attempts: x0.9 below 25 % acceptance, x1.1 above 75 %, capped at 0.3 V."""
    if attempted <= 0:
        return dv_max
    rate = accepted / attempted
    if rate < 0.25:
        dv_max *= 0.9
    elif rate > 0.75:
        dv_max = min(dv_max * 1.1, 0.3 * volume)
    return dv_max


def molecule_trees(natoms, bonds):
    """Molecules as a CSR for ``tmd_set_molecules``: ``(ptr, atoms, parent)`` int32, each molecule in breadth-first
    order of its bond graph from its smallest atom, ``parent`` the atom each was reached from (the first: itself).
    Components from ``wrapper._components``; atoms without bonds are one-atom molecules."""
    from .wrapper import _components

    groups, single = _components(natoms, bonds)
    adj = [[] for _ in range(natoms)]
    if bonds is not None and len(bonds):
        for i, j in np.asarray(bonds, dtype=np.int64).reshape(-1, 2):
            adj[int(i)].append(int(j))
            adj[int(j)].append(int(i))
    ptr, atoms, parent = [0], [], []
    for g in groups:
        seen = {g[0]}
        queue = deque([(g[0], g[0])])
        while queue:
            a, p = queue.popleft()
            atoms.append(a)
            parent.append(p)
            for b in sorted(adj[a]):
                if b not in seen:
                    seen.add(b)
                    queue.append((b, a))
        ptr.append(len(atoms))
    for a in single:
        atoms.append(a)
        parent.append(a)
        ptr.append(len(atoms))
    return (np.asarray(ptr, dtype=np.int32), np.asarray(atoms, dtype=np.int32), np.asarray(parent, dtype=np.int32))


class MonteCarloBarostat:
    """Isotropic Monte Carlo barostat for ``Integrator(..., barostat=...)``.

    pressure : bar.  temperature : K, the integrator's ``T`` by default.  frequency : a move per replica after every
    ``frequency``-th step, counted on the integrator's step index across ``step`` calls.  seed : of the replicas'
    random streams, by default drawn from torch's generator (``torch.manual_seed`` makes runs reproducible).
    ``uniforms``, when set, is a callable ``(replica, attempt) -> (u_volume, u_accept)`` that replaces the draws
    (tests).
    """

    def __init__(self, pressure=1.0, temperature=None, frequency=25, seed=None):
        if not float(pressure) > 0.0:
            raise ValueError("MonteCarloBarostat: pressure must be positive (bar)")
        if temperature is not None and not float(temperature) > 0.0:
            raise ValueError("MonteCarloBarostat: temperature must be positive (K)")
        if int(frequency) < 1 or int(frequency) != frequency:
            raise ValueError("MonteCarloBarostat: frequency must be an integer >= 1")
        self.pressure = float(pressure)
        self.temperature = None if temperature is None else float(temperature)
        self.frequency = int(frequency)
        self.seed = int(torch.randint(0, 2**62, (1,)).item()) if seed is None else int(seed)
        self.uniforms = None
        self._integ = None

    # ------------------------------------------------------------------ set-up
    def _bind(self, integ):
        """Checks the integrator can run NPT and sets up the per-replica state (called by Integrator)."""
        from .forces import Forces

        if not isinstance(integ.forces, Forces) or integ.forces.external is not None:
            raise RuntimeError("MonteCarloBarostat needs a native torchmd_b200.Forces without an external plugin")
        if not integ.T or integ.gamma is None:
            raise RuntimeError("MonteCarloBarostat needs a thermostat: give the Integrator T and gamma")
        self.kT = BOLTZMAN * (self.temperature if self.temperature is not None else float(integ.T))
        par = integ.forces.par
        bonds = par.bond_params["idx"].cpu().numpy() if par.bond_params is not None else None
        natoms = integ.systems.pos.shape[1]
        self._ptr, self._atoms, self._parent = molecule_trees(natoms, bonds)
        self.nmol = len(self._ptr) - 1
        self._integ = integ
        self._ctx_bound = None
        self._replicas = None

    def _setup(self, ctx, nrep, box_diag):
        if self._replicas is None or len(self._replicas) != nrep:
            self._replicas = []
            for r in range(nrep):
                V = float(np.prod(box_diag[r]))
                self._replicas.append(dict(
                    rng=np.random.default_rng([self.seed, r]), dv_max=0.01 * V, attempted=0, accepted=0,
                    batch_attempted=0, batch_accepted=0, fast=0, full=0))
        if self._ctx_bound != ctx.value:
            _lib.check(_lib.lib().tmd_set_molecules(ctx, self.nmol, self._ptr.ctypes.data, self._atoms.ctypes.data,
                                                    self._parent.ctypes.data))
            self._ctx_bound = ctx.value

    def stats(self):
        """Per replica: moves attempted and accepted, the current dV_max (A^3), and the box changes that took the fast
        device path (``tmd_rescale_box``) and the full one (``tmd_set_box``)."""
        if self._replicas is None:
            return []
        return [dict(attempted=s["attempted"], accepted=s["accepted"], dv_max=s["dv_max"], fast_box_changes=s["fast"],
                     full_box_changes=s["full"]) for s in self._replicas]

    # ------------------------------------------------------------------ the move
    def _draw(self, r):
        s = self._replicas[r]
        if self.uniforms is not None:
            return self.uniforms(r, s["attempted"])
        return float(s["rng"].random()), float(s["rng"].random())

    def _set_box(self, ctx, diag, counts):
        """Hand the box diagonal (R,3) to the context: the fast path, else the full one.  ``counts``: replicas whose box
        changed, counted as a fast or full change."""
        L = _lib.lib()
        f64 = self._integ.systems.pos.dtype == torch.float64
        host = np.ascontiguousarray(diag, dtype=np.float64 if f64 else np.float32)
        stream = torch.cuda.current_stream(self._integ.systems.pos.device).cuda_stream
        rc = (L.tmd_rescale_box_f64 if f64 else L.tmd_rescale_box)(ctx, host.ctypes.data, stream)
        kind = "fast"
        if rc == _lib.ERR_UNSUPPORTED:
            _lib.check((L.tmd_set_box_f64 if f64 else L.tmd_set_box)(ctx, host.ctypes.data))
            kind = "full"
        else:
            _lib.check(rc)
        for r in counts:
            self._replicas[r][kind] += 1

    def _write_box(self, diag):
        """``systems.box`` diagonal in place, and the Forces box key moved along so that no tmd_set_box follows."""
        s, f = self._integ.systems, self._integ.forces
        box = s.box
        idx = torch.arange(3, device=box.device)
        box[:, idx, idx] = torch.as_tensor(diag, dtype=box.dtype).to(box.device)
        f._box_key = (box.data_ptr(), box._version, tuple(box.shape), tuple(box.stride()), box.dtype)
        f._box_ref = box

    def attempt(self, ctx, energies):
        """One move of every replica from the state whose (R, NUM_ENERGIES) device energies are ``energies``.
        Returns the per-replica potential energies (host floats) of the state it leaves."""
        integ = self._integ
        s, f = integ.systems, integ.forces
        L = _lib.lib()
        f64 = s.pos.dtype == torch.float64
        sfx = "_f64" if f64 else ""
        nrep = s.pos.shape[0]
        np_dtype = np.float64 if f64 else np.float32
        cols = f._energy_columns()
        e_old = energies[:, cols].sum(dim=1).cpu().numpy()
        old = torch.diagonal(s.box, dim1=1, dim2=2).detach().cpu().numpy().astype(np.float64)
        self._setup(ctx, nrep, old)
        new = old.copy()
        dV = np.zeros(nrep)
        u_acc = np.zeros(nrep)
        for r in range(nrep):
            uv, ua = self._draw(r)
            V = float(np.prod(old[r]))
            dv = (2.0 * uv - 1.0) * self._replicas[r]["dv_max"]
            sc = ((V + dv) / V) ** (1.0 / 3.0)
            new[r] = (old[r] * sc).astype(np_dtype).astype(np.float64)  # a box the state's precision holds
            dV[r] = float(np.prod(new[r])) - V
            u_acc[r] = ua
        stream = torch.cuda.current_stream(s.pos.device).cuda_stream
        saved = s.pos.clone()
        saved_vel = s.vel.clone() if integ.constraints is not None else None
        scale = torch.as_tensor(new / old, dtype=torch.float64).to(s.pos.device)
        _lib.check(getattr(L, "tmd_scale_molecules" + sfx)(ctx, s.pos.data_ptr(), scale.data_ptr(), stream))
        self._set_box(ctx, new, range(nrep))
        if integ.constraints is not None:
            # the moved coordinates' rounding back onto the constraints, and the velocities projected at them (the
            # directions of the bonds moved by that rounding); a rejected replica gets both back from the copies
            _lib.check(getattr(L, "tmd_constrain" + sfx)(ctx, s.pos.data_ptr(), s.vel.data_ptr(), integ.masses.data_ptr(), stream))
        self._write_box(new)
        if f._scratch_forces is None or f._scratch_forces.shape != s.pos.shape or f._scratch_forces.dtype != s.pos.dtype:
            f._scratch_forces = torch.empty_like(s.pos)
        trial_f = f._scratch_forces
        ene = f._evaluate(s.pos, s.box, trial_f)  # (synchronises: the one read-back of the move)
        e_new = ene[:, cols].sum(dim=1).cpu().numpy()
        ok = np.zeros(nrep, dtype=bool)
        for r in range(nrep):
            V = float(np.prod(old[r]))
            w = acceptance_work(float(e_new[r] - e_old[r]), dV[r], V, self.pressure, self.nmol, self.kT)
            ok[r] = accept(w, self.kT, u_acc[r])
            st = self._replicas[r]
            st["attempted"] += 1
            st["batch_attempted"] += 1
            st["accepted"] += int(ok[r])
            st["batch_accepted"] += int(ok[r])
            if st["batch_attempted"] >= 10:
                vol = float(np.prod(new[r] if ok[r] else old[r]))
                st["dv_max"] = adapt_dv_max(st["dv_max"], st["batch_attempted"], st["batch_accepted"], vol)
                st["batch_attempted"] = st["batch_accepted"] = 0
        for r in range(nrep):  # (per replica slices: no mask, no host round trip)
            if ok[r]:
                s.forces[r].copy_(trial_f[r])
            else:
                s.pos[r].copy_(saved[r])
                if saved_vel is not None:
                    s.vel[r].copy_(saved_vel[r])
        if not ok.all():
            back = np.where(ok[:, None], new, old)
            self._set_box(ctx, back, [r for r in range(nrep) if not ok[r]])
            self._write_box(back)
        return np.where(ok, e_new, e_old)

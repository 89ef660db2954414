"""CPU oracle for the torchmd hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain torch-CPU restatement of what ``torchmd/forces.py`` and
``torchmd/integrator.py`` compute, written so that every floating-point value is
produced by the same sequence of rounded operations as the reference (the
cutoff decision of a pair depends on it bit for bit, SURVEY.md section 7-1).
It is pinned against the unmodified reference by ``tests/golden/make_golden.py``
(run in the build container, where ``/root/reference`` is importable) and
against the committed fixtures by ``tests/test_oracle.py``.

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may import this module; the product
package ``torchmd_b200`` never does.

Every function cites the reference lines it restates (paths relative to the
reference checkout).  Algorithmic structure is the reference's: an all-pairs
table minus exclusions built once (O(N^2)), all pair distances every step, a
``dist <= cutoff`` mask, per-term energy/force, ``index_add_`` scatter.
"""
import math

import numpy as np
import torch
from scipy import constants as _sc

TIMEFACTOR = 48.88821  # integrator.py:4  (fs per internal time unit)
BOLTZMAN = 0.001987191  # integrator.py:5  (kcal/mol/K)
PICOSEC2TIMEU = 1000.0 / TIMEFACTOR  # integrator.py:77

# forces.py:375-378 -- Coulomb constant in kcal*A/(mol*e^2), from CODATA values
COULOMB = (
    1.0
    / (4.0 * _sc.pi * _sc.epsilon_0)
    * _sc.elementary_charge**2
    / _sc.angstrom
    * _sc.Avogadro
    / (_sc.kilo * _sc.calorie)
)

BONDED_TERMS = ("bonds", "angles", "dihedrals", "impropers", "1-4")
PAIR_TERMS = ("electrostatics", "lj", "repulsion", "repulsioncg")


# ----------------------------------------------------------------------------
# pair table  (forces.py:348-357)
# ----------------------------------------------------------------------------
def all_pairs_minus_exclusions(natoms, excluded):
    """Row-major (i<j) list of every atom pair that is not excluded.

    This ordering (i ascending, then j ascending) is the reference's canonical
    neighbour order; the cutoff mask preserves it.
    """
    allowed = np.ones((natoms, natoms), dtype=bool)
    if len(excluded):
        e = np.asarray(excluded, dtype=np.int64)
        allowed[e[:, 0], e[:, 1]] = False
        allowed[e[:, 1], e[:, 0]] = False
    ii, jj = np.nonzero(np.triu(allowed, 1))
    return torch.from_numpy(np.stack([ii, jj], axis=1))


# ----------------------------------------------------------------------------
# geometry  (forces.py:360-372)
# ----------------------------------------------------------------------------
def minimum_image(delta, box_diag):
    """delta - box*round(delta/box); identity when the box is absent/all zero.

    Four separately rounded elementwise ops (div, round-half-even, mul, sub),
    exactly the reference's sequence (forces.py:361-364).
    """
    if box_diag is None or bool(torch.all(box_diag == 0)):
        return delta
    b = box_diag.unsqueeze(0)
    return delta - b * torch.round(delta / b)


def pair_geometry(xyz, pairs, box_diag):
    """(dist, unit vector, vector) of pos[i]-pos[j] under the minimum image.

    The distance goes through ``torch.norm(dim=1)`` like the reference
    (forces.py:370): on CPU that is sqrt_rn(fma(z,z,fma(y,y,x*x))) in fp32,
    measured in tests/golden/make_golden.py -- NOT torch.sqrt of a sum.
    """
    vec = minimum_image(xyz[pairs[:, 0]] - xyz[pairs[:, 1]], box_diag)
    dist = torch.norm(vec, dim=1)
    return dist, vec / dist.unsqueeze(1), vec


# ----------------------------------------------------------------------------
# pair potentials  (forces.py:381-491)
# ----------------------------------------------------------------------------
def lj_pair(dist, A, B, scale, switch_dist, cutoff, true_gradient=False):
    """12-6 energy and dE/dr, optional quintic switch (forces.py:389-415).

    With switching the 'force' is s*dE/dr + E*s'/r  -- the extra 1/r is the
    reference's (forces.py:410-412) and is reproduced on purpose.  ``true_gradient``: the
    derivative autograd takes of the same energy, s*dE/dr + E*s' (the reference's
    explicit_forces=False path, forces.py:328-336).
    """
    rinv = 1 / dist
    r6 = rinv**6
    r12 = r6 * r6
    ene = ((A * r12) - (B * r6)) / scale
    dedr = (-12 * A * r12 + 6 * B * r6) * rinv / scale
    if switch_dist is not None and cutoff is not None:
        outer = dist > switch_dist
        t = (dist[outer] - switch_dist) / (cutoff - switch_dist)
        sw = 1 + t * t * t * (-10 + t * (15 - t * 6))
        dsw = t * t * (-30 + t * (60 - t * 30)) / (cutoff - switch_dist)
        dedr[outer] = sw * dedr[outer] + (ene[outer] * dsw if true_gradient else ene[outer] * dsw / dist[outer])
        ene[outer] = ene[outer] * sw
    return ene, dedr


def coulomb_pair(dist, qi, qj, scale, cutoff, rfa, eps_solvent):
    """Plain or reaction-field Coulomb energy and dE/dr (forces.py:453-491)."""
    if rfa:
        denom = (2 * eps_solvent) + 1
        krf = (1 / cutoff**3) * (eps_solvent - 1) / denom
        crf = (1 / cutoff) * (3 * eps_solvent) / denom
        pref = COULOMB * qi * qj / scale
        d2 = dist**2
        ene = pref * ((1 / dist) + krf * d2 - crf)
        dedr = pref * (2 * krf * dist - 1 / d2)
    else:
        ene = COULOMB * qi * qj / dist / scale
        dedr = -ene / dist
    return ene, dedr


def repulsion_pair(dist, A):
    """A/r^12 only (forces.py:418-433)."""
    rinv = 1 / dist
    r6 = rinv**6
    r12 = r6 * r6
    return A * r12, (-12 * A * r12) * rinv


def repulsion_cg_pair(dist, B):
    """B/r^6 only (forces.py:436-450)."""
    rinv = 1 / dist
    r6 = rinv**6
    return B * r6, (-6 * B * r6) * rinv


# ----------------------------------------------------------------------------
# bonded potentials  (forces.py:494-605)
# ----------------------------------------------------------------------------
def harmonic_bond(dist, prm):
    """k (r-r0)^2 and 2k(r-r0)  (forces.py:494-503)."""
    dev = dist - prm[:, 1]
    return prm[:, 0] * dev**2, 2 * prm[:, 0] * dev


def harmonic_angle(r21, r23, prm):
    """k (theta-theta0)^2 and the three per-atom force vectors (forces.py:506-539)."""
    k, theta0 = prm[:, 0], prm[:, 1]
    inv21 = 1 / torch.norm(r21, dim=1)
    inv23 = 1 / torch.norm(r23, dim=1)
    cosang = torch.clamp(torch.sum(r23 * r21, dim=1) * inv21 * inv23, -1, 1)
    dtheta = torch.acos(cosang) - theta0
    ene = k * dtheta * dtheta
    sinang = torch.sqrt(1.0 - cosang * cosang)
    coef = torch.zeros_like(sinang)
    ok = sinang != 0  # guard: zero force where sin(theta)==0 (forces.py:523-526)
    coef[ok] = -2.0 * k[ok] * dtheta[ok] / sinang[ok]
    c = cosang[:, None]
    f_a = coef[:, None] * (c * r21 * inv21[:, None] - r23 * inv23[:, None]) * inv21[:, None]
    f_c = coef[:, None] * (c * r23 * inv23[:, None] - r21 * inv21[:, None]) * inv23[:, None]
    return ene, (f_a, -(f_a + f_c), f_c)


def torsion(r12, r23, r34, term_row, prm):
    """Proper/improper torsion energy per dihedral and the four force vectors.

    phi = -atan2(sin, cos) from cross products (forces.py:544-553); periodic
    (AMBER) form iff *every* periodicity is > 0, else harmonic (CHARMM) form with
    +-2pi unwrap (forces.py:566-579); several terms per dihedral accumulate
    through ``term_row``; forces follow the OpenMM-style projection
    (forces.py:584-603).
    """
    cA = torch.cross(r12, r23, dim=1)
    cB = torch.cross(r23, r34, dim=1)
    cC = torch.cross(r23, cA, dim=1)
    nA = torch.norm(cA, dim=1)
    nB = torch.norm(cB, dim=1)
    nC = torch.norm(cC, dim=1)
    uB = cB / nB.unsqueeze(1)
    cosphi = torch.sum(cA * uB, dim=1) / nA
    sinphi = torch.sum(cC * uB, dim=1) / nC
    phi = -torch.atan2(sinphi, cosphi)

    n = r12.shape[0]
    ene = torch.zeros(n, dtype=r12.dtype)
    coef = torch.zeros(n, dtype=r12.dtype)
    k, phi0, per = prm[:, 0], prm[:, 1], prm[:, 2]
    if bool(torch.all(per > 0)):
        arg = per * phi[term_row] - phi0
        ene = torch.scatter_add(ene, 0, term_row, k * (1 + torch.cos(arg)))
        coef = torch.scatter_add(coef, 0, term_row, -per * k * torch.sin(arg))
    else:
        arg = phi[term_row] - phi0
        arg[arg < -math.pi] = arg[arg < -math.pi] + 2 * math.pi
        arg[arg > math.pi] = arg[arg > math.pi] - 2 * math.pi
        ene = torch.scatter_add(ene, 0, term_row, k * arg**2)
        coef = torch.scatter_add(coef, 0, term_row, 2 * k * arg)

    n23 = torch.norm(r23, dim=1)
    n23sq = n23**2
    g0 = (-coef * n23) / (nA**2)
    g1 = torch.sum(r12 * r23, dim=1) / n23sq
    g2 = torch.sum(r34 * r23, dim=1) / n23sq
    g3 = (coef * n23) / (nB**2)
    v0 = g0.unsqueeze(1) * cA
    v3 = g3.unsqueeze(1) * cB
    s = g1.unsqueeze(1) * v0 - g2.unsqueeze(1) * v3
    return ene, (-v0, v0 + s, v3 - s, -v3)


# ----------------------------------------------------------------------------
# Forces.compute  (forces.py:83-346, explicit-force path)
# ----------------------------------------------------------------------------
class OracleForces:
    """All-pairs evaluation of a parameter set; mirrors ``Forces`` semantics.

    ``par`` is any object with the reference ``Parameters`` attribute layout
    (the reference's own object or ``torchmd_b200.parameters.TopologyParameters``).
    """

    def __init__(
        self,
        par,
        terms,
        cutoff=None,
        rfa=False,
        solventDielectric=78.5,
        switch_dist=None,
        exclusions=("bonds", "angles", "1-4"),
        decision_dtype=None,
        true_gradient=False,
    ):
        """``true_gradient``: forces as the exact gradient of the energy -- what the reference returns
        with ``explicit_forces=False`` (autograd, forces.py:328-336); only the switched LJ differs
        from the explicit formulas.
        ``decision_dtype``: evaluate the ``dist <= cutoff`` masks in this dtype (e.g. the
        reference's fp32 decisions) while the energies/forces use the dtype of ``pos`` --
        the yardstick for an fp32 kernel: same pair set, exact values.  ``None`` = the
        reference's behaviour (decisions in the dtype of ``pos``)."""
        self.decision_dtype = decision_dtype
        self.true_gradient = bool(true_gradient)
        self.par = par
        self.terms = [t.lower() for t in terms]
        for t in self.terms:
            if t not in BONDED_TERMS + PAIR_TERMS:
                raise ValueError(f"Force term {t} is not implemented.")
        if "1-4" in self.terms and "dihedrals" not in self.terms:
            raise RuntimeError(
                "You cannot enable 1-4 interactions without enabling dihedrals"
            )
        if par.nonbonded_params is not None and "lj" in self.terms:
            par.A, par.B = par.get_AB()  # forces.py:45-46
        self.natoms = len(par.masses)
        self.needs_pairs = any(t in PAIR_TERMS for t in self.terms)
        self.pairs = (
            all_pairs_minus_exclusions(self.natoms, par.get_exclusions(exclusions))
            if self.needs_pairs
            else None
        )
        self.cutoff = cutoff
        self.rfa = rfa
        self.eps_solvent = solventDielectric
        self.switch_dist = switch_dist

    # the reference's "neighbour list": rows of the pair table with dist<=cutoff
    def neighbour_pairs(self, xyz, box_diag):
        dist, _, _ = pair_geometry(xyz, self.pairs, box_diag)
        if self.cutoff is None:
            return self.pairs
        return self.pairs[dist <= self.cutoff]  # forces.py:77

    def _inside(self, xyz, idx, bd, dist):
        """dist <= cutoff, decided in ``decision_dtype`` when one is set (forces.py:77)."""
        dd = self.decision_dtype
        if dd is None or dd == xyz.dtype:
            return dist <= self.cutoff
        d, _, _ = pair_geometry(xyz.to(dd), idx, bd.to(dd))
        return d <= self.cutoff

    def compute(self, pos, box, forces):
        """Fill ``forces`` (R,N,3) in place, return list of {term: float}."""
        par, terms = self.par, self.terms
        forces.zero_()
        out = []
        for r in range(pos.shape[0]):
            xyz = pos[r]
            bd = torch.stack([box[r][0, 0], box[r][1, 1], box[r][2, 2]])  # diagonal only, forces.py:118
            f = forces[r]
            e = {t: torch.zeros((), dtype=pos.dtype) for t in terms}

            def torsion_term(name, tp):  # forces.py:163-183 (dihedrals), 238-258 (impropers)
                idx = tp["idx"]
                _, _, r12 = pair_geometry(xyz, idx[:, [0, 1]], bd)
                _, _, r23 = pair_geometry(xyz, idx[:, [1, 2]], bd)
                _, _, r34 = pair_geometry(xyz, idx[:, [2, 3]], bd)
                ene, fs = torsion(r12, r23, r34, tp["map"][:, 0], tp["params"][tp["map"][:, 1]])
                e[name] = e[name] + ene.sum()
                for col in range(4):
                    f.index_add_(0, idx[:, col], fs[col])

            if "bonds" in terms and par.bond_params is not None:  # forces.py:122-143
                idx = par.bond_params["idx"]
                prm = par.bond_params["params"][par.bond_params["map"][:, 1]]
                dist, unit, _ = pair_geometry(xyz, idx, bd)
                if self.cutoff is not None:  # bonds are cutoff-filtered too
                    keep = self._inside(xyz, idx, bd, dist)
                    dist, unit, idx, prm = dist[keep], unit[keep], idx[keep], prm[keep]
                ene, dedr = harmonic_bond(dist, prm)
                e["bonds"] = e["bonds"] + ene.sum()
                fv = unit * dedr[:, None]
                f.index_add_(0, idx[:, 0], -fv)
                f.index_add_(0, idx[:, 1], fv)

            if "angles" in terms and par.angle_params is not None:  # forces.py:145-161
                idx = par.angle_params["idx"]
                prm = par.angle_params["params"][par.angle_params["map"][:, 1]]
                _, _, r21 = pair_geometry(xyz, idx[:, [0, 1]], bd)
                _, _, r23 = pair_geometry(xyz, idx[:, [2, 1]], bd)
                ene, fs = harmonic_angle(r21, r23, prm)
                e["angles"] = e["angles"] + ene.sum()
                for col in range(3):
                    f.index_add_(0, idx[:, col], fs[col])

            if "dihedrals" in terms and par.dihedral_params is not None:
                torsion_term("dihedrals", par.dihedral_params)

            if "1-4" in terms and par.nonbonded_14_params is not None:  # forces.py:185-236
                idx = par.nonbonded_14_params["idx"]
                prm = par.nonbonded_14_params["params"][par.nonbonded_14_params["map"][:, 1]]
                dist, unit, _ = pair_geometry(xyz, idx, bd)
                if "lj" in terms:  # scaled by scnb; no cutoff, no switch; booked under "lj"
                    ene, dedr = lj_pair(dist, prm[:, 0], prm[:, 1], prm[:, 2], None, None)
                    e["lj"] = e["lj"] + ene.sum()
                    fv = unit * dedr[:, None]
                    f.index_add_(0, idx[:, 0], -fv)
                    f.index_add_(0, idx[:, 1], fv)
                if "electrostatics" in terms:  # scaled by scee; never reaction field
                    ene, dedr = coulomb_pair(
                        dist, par.charges[idx[:, 0]], par.charges[idx[:, 1]], prm[:, 3], None, False, self.eps_solvent
                    )
                    e["electrostatics"] = e["electrostatics"] + ene.sum()
                    fv = unit * dedr[:, None]
                    f.index_add_(0, idx[:, 0], -fv)
                    f.index_add_(0, idx[:, 1], fv)

            if "impropers" in terms and par.improper_params is not None:
                torsion_term("impropers", par.improper_params)

            if self.needs_pairs and len(self.pairs):  # forces.py:261-319
                dist, unit, _ = pair_geometry(xyz, self.pairs, bd)
                pairs = self.pairs
                if self.cutoff is not None:
                    keep = self._inside(xyz, pairs, bd, dist)
                    dist, unit, pairs = dist[keep], unit[keep], pairs[keep]
                ti = par.mapped_atom_types[pairs] if par.mapped_atom_types is not None else None
                for t in terms:
                    if t == "electrostatics":
                        ene, dedr = coulomb_pair(
                            dist, par.charges[pairs[:, 0]], par.charges[pairs[:, 1]], 1, self.cutoff, self.rfa, self.eps_solvent
                        )
                    elif t == "lj":
                        ene, dedr = lj_pair(dist, par.A[ti[:, 0], ti[:, 1]], par.B[ti[:, 0], ti[:, 1]], 1, self.switch_dist, self.cutoff,
                                            self.true_gradient)
                    elif t == "repulsion":
                        ene, dedr = repulsion_pair(dist, par.A[ti[:, 0], ti[:, 1]])
                    elif t == "repulsioncg":
                        ene, dedr = repulsion_cg_pair(dist, par.B[ti[:, 0], ti[:, 1]])
                    else:
                        continue
                    e[t] = e[t] + ene.sum()
                    fv = unit * dedr[:, None]
                    f.index_add_(0, pairs[:, 0], -fv)
                    f.index_add_(0, pairs[:, 1], fv)
            out.append({k: float(v) for k, v in e.items()})
        return out


# ----------------------------------------------------------------------------
# integrator  (integrator.py:8-125)
# ----------------------------------------------------------------------------

# ----------------------------------------------------------------------------
# row-sampled evaluation for systems the all-pairs table cannot hold
# ----------------------------------------------------------------------------
def sampled_rows(par, terms, pos, box_diag, atoms, cutoff, rfa=False, solventDielectric=78.5, switch_dist=None,
                 exclusions=("bonds", "angles", "1-4"), chunk=256, true_gradient=False):
    """Non-bonded force on each atom of ``atoms`` from ALL its partners, and its in-cutoff partner sets.

    The reference's pair arithmetic (forces.py:264-319 with 360-372, 381-415, 453-491) restricted to the
    rows of the all-pairs table that contain a sampled atom: 1,000 atoms x 99,999 partners is 1e8 distances,
    where the full table (forces.py:348-357) would need 5e9.  Decisions ``dist <= cutoff`` in fp32 on fp32
    positions like the reference's fp32 path; values in the dtype of ``pos`` (fp64: the yardstick).  ``true_gradient``:
    the switched LJ as the exact gradient of its energy (OracleForces' option of the same name).
    ``pos`` (N,3), ``box_diag`` (3,).  Returns (forces (len(atoms),3), list of sorted partner index arrays)."""
    terms = [t.lower() for t in terms]
    N = pos.shape[0]
    excl = {}
    for i, j in par.get_exclusions(exclusions):
        excl.setdefault(int(i), set()).add(int(j))
        excl.setdefault(int(j), set()).add(int(i))
    if "lj" in terms:
        A, B = par.get_AB()
        A, B = A.to(pos.dtype), B.to(pos.dtype)
    types = par.mapped_atom_types
    q = par.charges.to(pos.dtype)
    pos32, bd32 = pos.to(torch.float32), box_diag.to(torch.float32)
    allj = torch.arange(N)
    out_f = torch.zeros((len(atoms), 3), dtype=pos.dtype)
    out_p = []
    for c0 in range(0, len(atoms), chunk):
        sel = torch.as_tensor(atoms[c0 : c0 + chunk], dtype=torch.long)
        ii = sel.repeat_interleave(N)
        jj = allj.repeat(len(sel))
        keep = ii != jj
        # the reference's table holds (min, max): its difference is pos[min] - pos[max] (forces.py:369)
        lo, hi = torch.minimum(ii, jj), torch.maximum(ii, jj)
        pairs = torch.stack([lo, hi], dim=1)
        d32, _, _ = pair_geometry(pos32, pairs, bd32)
        inside = (d32 <= cutoff) & keep
        for k, a in enumerate(sel.tolist()):  # exclusions of the sampled atoms
            ex = excl.get(a)
            if ex:
                inside[k * N + torch.as_tensor(sorted(ex), dtype=torch.long)] = False
        idx = pairs[inside]
        dist, unit, _ = pair_geometry(pos, idx, box_diag)
        dedr = torch.zeros_like(dist)
        if "lj" in terms:
            a_ = A[types[idx[:, 0]], types[idx[:, 1]]]
            b_ = B[types[idx[:, 0]], types[idx[:, 1]]]
            dedr += lj_pair(dist, a_, b_, 1, switch_dist, cutoff, true_gradient)[1]
        if "electrostatics" in terms:
            dedr += coulomb_pair(dist, q[idx[:, 0]], q[idx[:, 1]], 1, cutoff, rfa, solventDielectric)[1]
        fvec = unit * dedr.unsqueeze(1)  # forces.py:316-319: f[idx0] -= fvec ; f[idx1] += fvec
        row = ii[inside]  # the sampled atom of each kept pair
        sign = torch.where(idx[:, 0] == row, -1.0, 1.0).to(pos.dtype).unsqueeze(1)
        local = torch.searchsorted(sel, row) if bool(torch.all(sel[1:] > sel[:-1])) else None
        if local is None:
            lut = {a: k for k, a in enumerate(sel.tolist())}
            local = torch.as_tensor([lut[a] for a in row.tolist()], dtype=torch.long)
        out_f[c0 : c0 + len(sel)].index_add_(0, local, sign * fvec)
        partner = jj[inside]
        for k in range(len(sel)):
            out_p.append(torch.sort(partner[local == k]).values)
    return out_f, out_p


def kinetic_energy(masses, vel):
    """0.5 m v^2 summed per replica -> (R,1)  (integrator.py:8-30)."""
    return torch.sum(0.5 * masses * torch.sum(vel * vel, dim=2, keepdim=True), dim=1)


def kinetic_to_temperature(ekin, natoms):
    """T = 2 Ekin / (3 N kB): N atoms, not degrees of freedom (integrator.py:57-58)."""
    return 2.0 / (3.0 * natoms * BOLTZMAN) * ekin


def maxwell_boltzmann(masses, T, replicas=1):
    """sqrt(kB T / m) * N(0,1) per replica (integrator.py:46-54)."""
    return torch.stack(
        [torch.sqrt(T * BOLTZMAN / masses) * torch.randn((len(masses), 3)).type_as(masses) for _ in range(replicas)],
        dim=0,
    )


class OracleIntegrator:
    """Velocity Verlet with the reference's Langevin kick placement.

    Per iteration (integrator.py:115-120): half-kick+drift with the OLD forces,
    force evaluation, ``v += -gamma v dt + N(0,1) vcoeff`` (only when T is set),
    second half-kick.  ``noise`` lets a test inject the N(0,1) draws; otherwise
    they come from ``torch.randn_like`` like the reference.
    """

    def __init__(self, pos, vel, box, forces_buf, masses, force_fn, timestep_fs, gamma_ps=None, T=None):
        self.pos, self.vel, self.box, self.f = pos, vel, box, forces_buf
        self.masses = masses.view(-1, 1)
        self.force_fn = force_fn
        self.dt = timestep_fs / TIMEFACTOR
        self.gamma = gamma_ps / PICOSEC2TIMEU if gamma_ps is not None else None
        self.T = T
        if T:
            self.vcoeff = torch.sqrt(2.0 * self.gamma / self.masses * BOLTZMAN * T * self.dt)

    def step(self, niter=1, noise=None):
        dt, m = self.dt, self.masses
        pot = None
        for it in range(niter):
            acc = self.f / m
            self.pos += self.vel * dt + 0.5 * acc * dt * dt
            self.vel += 0.5 * dt * acc
            pot = self.force_fn(self.pos, self.box, self.f)
            if self.T:
                xi = noise[it] if noise is not None else torch.randn_like(self.vel)
                self.vel += -self.gamma * self.vel * dt + xi * self.vcoeff
            self.vel += 0.5 * dt * (self.f / m)
        ekin = kinetic_energy(m, self.vel).flatten().numpy()
        return ekin, pot, kinetic_to_temperature(ekin, len(m))


# ---- Wrapper (wrapper.py) ------------------------------------------------------------------
def molecule_groups(natoms, bonds):
    """wrapper.py:33-55 -- connected components of the bond graph: (groups of >= 2 atoms,
    atoms without any bond).  Breadth-first search instead of networkx; groups hold their
    atoms in ascending order, ordered by smallest atom."""
    if bonds is None or len(bonds) == 0:
        return [], list(range(natoms))
    adj = [[] for _ in range(natoms)]
    for i, j in np.asarray(bonds).astype(np.int64):
        adj[i].append(int(j))
        adj[j].append(int(i))
    seen = [False] * natoms
    groups, single = [], []
    for s in range(natoms):
        if seen[s]:
            continue
        comp, stack = [], [s]
        seen[s] = True
        while stack:
            a = stack.pop()
            comp.append(a)
            for b in adj[a]:
                if not seen[b]:
                    seen[b] = True
                    stack.append(b)
        if len(comp) == 1:
            single.append(s)
        else:
            groups.append(sorted(comp))
    return groups, single


def wrap_positions(pos, box, groups, nongrouped):
    """wrapper.py:8-30 without the wrap-index branch (which rebinds a local and has no effect on
    the caller's tensor): in place on ``pos`` (R,N,3); ``box`` (R,3,3)."""
    diag = box[:, torch.eye(3).bool()]  # :11
    if torch.all(diag == 0):  # :12-13
        return
    for group in groups:  # :23-27
        g = torch.as_tensor(group, dtype=torch.int64)
        com = torch.sum(pos[:, g], dim=1) / len(group)
        offset = torch.floor(com / diag) * diag
        pos[:, g] -= offset.unsqueeze(1)
    if len(nongrouped):  # :29-31
        n = torch.as_tensor(nongrouped, dtype=torch.int64)
        offset = torch.floor(pos[:, n] / diag.unsqueeze(1)) * diag.unsqueeze(1)
        pos[:, n] -= offset

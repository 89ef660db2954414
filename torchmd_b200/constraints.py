"""Constraint topology for rigid water and bonds to hydrogen (``Integrator(..., constraints=...)``).

``Constraints(parameters, kind)`` reads the reference ``Parameters`` layout (``bond_params`` /
``angle_params`` as ``{"idx", "map", "params"}``, plus ``masses``), so a ``TopologyParameters`` and a
reference ``Parameters`` object both work.  It builds two disjoint sets of constraint groups:

* waters: a connected component of the bond graph with exactly one heavy atom and two hydrogens of
  equal mass, both bonded to the heavy atom.  The O-H distance is the bond's r0; the H-H distance is
  the r0 of an H-H bond when the topology has one (CHARMM TIP3), else 2 r0 sin(theta0 / 2) from the
  H-O-H angle term.  The device solves all three distances.
* X-H clusters (``kind="hbonds"`` only): one heavy atom and the 1-4 hydrogens bonded to it, each held
  at its bond's r0.

A hydrogen is an atom of mass above 0 and below 4.5 amu, so hydrogen mass repartitioning (H masses of
3-4 amu) still counts as hydrogen; a group with a massless atom is refused.  ``kind="water"`` constrains the waters only; ``kind="hbonds"`` the waters and
every bond to a hydrogen.  Topologies outside this model raise ``ValueError`` naming the atoms.
"""
import numpy as np

H_MASS_LIMIT = 4.5  # amu: atoms lighter than this are hydrogens


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def _term_params(term):
    """(idx (M,k), params (M,p)): the parameter row of every term (the first map row that names it)."""
    if term is None:
        return np.zeros((0, 2), np.int64), None
    idx = _np(term["idx"]).astype(np.int64)
    pmap = _np(term["map"]).astype(np.int64)
    params = _np(term["params"]).astype(np.float64)
    row = np.full(len(idx), -1, np.int64)
    for k in range(len(pmap) - 1, -1, -1):
        row[pmap[k, 0]] = pmap[k, 1]
    return idx, (params, row)


class Constraints:
    """Constraint groups of a topology; see the module docstring.

    ``water_idx`` (W,3) heavy atom and its two hydrogens, ``water_d`` (W,2) O-H and H-H distances;
    ``cluster_ptr`` / ``cluster_idx`` CSR of the X-H clusters (heavy atom first), ``cluster_d`` one
    distance per hydrogen in ``cluster_idx`` order without the heavy atoms.
    """

    def __init__(self, parameters, kind="water", batch=None):
        if kind not in ("water", "hbonds"):
            raise ValueError(f"kind must be 'water' or 'hbonds', got {kind!r}")
        self.kind = kind
        masses = _np(parameters.masses).reshape(-1).astype(np.float64)
        self.natoms = n = len(masses)
        is_h = (masses > 0) & (masses < H_MASS_LIMIT)  # (massless dummy atoms are not hydrogens)
        bidx, bpar = _term_params(getattr(parameters, "bond_params", None))
        aidx, apar = _term_params(getattr(parameters, "angle_params", None))

        def bond_r0(k):
            if bpar is None or bpar[1][k] < 0:
                i, j = bidx[k]
                raise ValueError(f"constrained bond {i}-{j} has no parameters")
            return float(bpar[0][bpar[1][k], 1])

        nbr = [[] for _ in range(n)]
        for k, (i, j) in enumerate(bidx):
            nbr[i].append((j, k))
            nbr[j].append((i, k))
        # waters: connected components of exactly one heavy atom and two hydrogens
        comp = -np.ones(n, np.int64)
        waters, water_d = [], []
        for s in range(n):
            if comp[s] >= 0:
                continue
            stack, members = [s], []
            comp[s] = s
            while stack:
                a = stack.pop()
                members.append(a)
                for b, _ in nbr[a]:
                    if comp[b] < 0:
                        comp[b] = s
                        stack.append(b)
            if len(members) != 3:
                continue
            heavy = [a for a in members if not is_h[a]]
            hyd = sorted(a for a in members if is_h[a])
            if len(heavy) != 1 or len(hyd) != 2:
                continue
            o, h1, h2 = heavy[0], hyd[0], hyd[1]
            bonds = {frozenset((a, b)): k for a in members for b, k in nbr[a]}
            if frozenset((o, h1)) not in bonds or frozenset((o, h2)) not in bonds:
                continue
            if masses[h1] != masses[h2]:
                raise ValueError(f"water {o},{h1},{h2}: the hydrogen masses differ ({masses[h1]} and {masses[h2]})")
            r1, r2 = bond_r0(bonds[frozenset((o, h1))]), bond_r0(bonds[frozenset((o, h2))])
            if r1 != r2:
                raise ValueError(f"water {o},{h1},{h2}: the two O-H bond lengths differ ({r1} and {r2})")
            if frozenset((h1, h2)) in bonds:
                dhh = bond_r0(bonds[frozenset((h1, h2))])
            else:
                sel = []
                if len(aidx):
                    ends = np.sort(aidx[:, [0, 2]], axis=1)
                    sel = np.nonzero((aidx[:, 1] == o) & (ends[:, 0] == h1) & (ends[:, 1] == h2))[0]
                if len(sel) == 0 or apar is None or apar[1][sel[0]] < 0:
                    raise ValueError(f"water {o},{h1},{h2}: the H-O-H angle has no parameters")
                theta0 = float(apar[0][apar[1][sel[0]], 1])
                dhh = 2.0 * r1 * np.sin(theta0 / 2.0)
            waters.append((o, h1, h2))
            water_d.append((r1, dhh))
        in_water = np.zeros(n, bool)
        for w in waters:
            in_water[list(w)] = True

        ptr, cidx, cd = [0], [], []
        if kind == "hbonds":  # (kind="water" constrains no other hydrogen, so refuses nothing about them)
            for k, (i, j) in enumerate(bidx):
                if is_h[i] and is_h[j] and not (in_water[i] and in_water[j]):
                    raise ValueError(f"H-H bond {i}-{j} outside a water")
            for i in np.nonzero(is_h & ~in_water)[0]:
                if len(nbr[i]) > 1:
                    raise ValueError(f"hydrogen {i} is bonded to {len(nbr[i])} atoms ({[int(a) for a, _ in nbr[i]]})")
            hs_of = {}
            for h in np.nonzero(is_h & ~in_water)[0]:
                if nbr[h]:
                    x, k = nbr[h][0]
                    hs_of.setdefault(int(x), []).append((int(h), k))
            for x in sorted(hs_of):
                hs = sorted(hs_of[x])
                if len(hs) > 4:
                    raise ValueError(f"heavy atom {x} has {len(hs)} hydrogens (at most 4 per cluster)")
                cidx.append(x)
                for h, k in hs:
                    cidx.append(h)
                    cd.append(bond_r0(k))
                ptr.append(len(cidx))

        self.water_idx = np.asarray(waters, np.int32).reshape(-1, 3)
        self.water_d = np.asarray(water_d, np.float64).reshape(-1, 2)
        self.cluster_ptr = np.asarray(ptr, np.int32)
        self.cluster_idx = np.asarray(cidx, np.int32)
        self.cluster_d = np.asarray(cd, np.float64)
        for g in self.groups():
            if np.any(masses[g] <= 0):
                raise ValueError(f"constraint group {g} has a massless atom")
        self._water_heads = set(int(w[0]) for w in self.water_idx)
        self.batch = None
        if batch is not None:
            self.ndof(batch=batch)  # (checks that no group spans two batch groups)
            self.batch = _np(batch).astype(np.int64)

    @property
    def nwaters(self):
        return len(self.water_idx)

    @property
    def nclusters(self):
        return len(self.cluster_ptr) - 1

    def groups(self):
        """Atom lists of every constraint group: waters first, then the clusters."""
        out = [list(map(int, w)) for w in self.water_idx]
        for c in range(self.nclusters):
            out.append(list(map(int, self.cluster_idx[self.cluster_ptr[c]:self.cluster_ptr[c + 1]])))
        return out

    def ndof(self, natoms=None, batch=None):
        """3N - N_c, N_c = 3 per water + 1 per X-H bond.  With a batch (``batch`` here or at construction),
        an array with one entry per batch group."""
        natoms = self.natoms if natoms is None else natoms
        batch = self.batch if batch is None else _np(batch).astype(np.int64)
        if batch is None:
            return 3 * natoms - 3 * self.nwaters - len(self.cluster_d)
        out = 3 * np.bincount(batch, minlength=int(batch.max()) + 1)
        for g in self.groups():
            if len(set(batch[g].tolist())) != 1:
                raise ValueError(f"constraint group {g} spans batch groups {sorted(set(batch[g].tolist()))}")
            out[batch[g[0]]] -= 3 if len(g) == 3 and g[0] in self._water_heads else len(g) - 1
        return out

    def upload(self, ctx):
        """Hand the tables to a library context (tmd_set_constraints)."""
        from . import _lib

        _lib.check(_lib.lib().tmd_set_constraints(
            ctx, self.nwaters, _lib.ptr(np.ascontiguousarray(self.water_idx)), _lib.ptr(np.ascontiguousarray(self.water_d)),
            self.nclusters, _lib.ptr(self.cluster_ptr), _lib.ptr(self.cluster_idx), _lib.ptr(self.cluster_d)))

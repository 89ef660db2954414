"""torchmd YAML force fields (reference torchmd/forcefields/ff_yaml.py) and the parameter
tables the reference's ``Parameters`` builds from them (parameters.py:109-294), as a
``TopologyParameters`` -- enough to run the reference's PSF/PDB + YAML set-ups (tests/water,
tests/argon, the CG examples) without moleculekit.

Look-up semantics follow ff_yaml.py:30-50: a term key matches an atom-type tuple directly, with
any subset of positions replaced by the wildcard ``X``, reversed (bonds, angles, dihedrals) or
with positions permuted around the improper centre (impropers, position 2); the match with the
fewest wildcards wins, ties resolved in the reference's enumeration order.
"""
import math
import warnings
from itertools import permutations, product

import numpy as np
import torch
import yaml

from .parameters import TopologyParameters


class YamlForceField:
    def __init__(self, path_or_dict):
        if isinstance(path_or_dict, dict):
            self.prm = path_or_dict
        else:
            with open(path_or_dict) as fh:
                self.prm = yaml.safe_load(fh)

    @staticmethod
    def _x_variants(atomtypes):  # ff_yaml.py:13-28
        masks = sorted(product([False, True], repeat=len(atomtypes)), key=sum)
        out = []
        for m in masks:
            t = np.array(atomtypes, dtype=object)
            t[np.array(m, dtype=bool)] = "X"
            out.append(t)
        return out

    def get_parameters(self, term, atomtypes):  # ff_yaml.py:30-50
        at = np.array(atomtypes, dtype=object)
        variants = self._x_variants(at)
        if term in ("bonds", "angles", "dihedrals"):
            variants += self._x_variants(at[::-1])
        elif term == "impropers":
            for perm in (p for p in permutations((0, 1, 2, 3)) if p[2] == 2):
                variants += self._x_variants(at[list(perm)])
        variants = sorted(variants, key=lambda v: int(sum(v == "X")))  # stable: enumeration order breaks ties
        table = self.prm[term]
        for v in variants:
            key = ", ".join(v)
            if len(v) > 1:
                key = "(" + key + ")"
            if key in table:
                return table[key]
        raise RuntimeError(f"{list(atomtypes)} doesn't have {term} information in the FF")

    def get_mass(self, at):
        return self.prm["masses"][at]

    def get_LJ(self, at):
        p = self.get_parameters("lj", [at])
        return p["sigma"], p["epsilon"]

    def get_bond(self, *at):
        p = self.get_parameters("bonds", at)
        return p["k0"], p["req"]

    def get_angle(self, *at):
        p = self.get_parameters("angles", at)
        return p["k0"], math.radians(p["theta0"])

    def get_dihedral(self, *at):
        p = self.get_parameters("dihedrals", at)
        return [[t["phi_k"], math.radians(t["phase"]), t["per"]] for t in p["terms"]]

    def get_14(self, *at):  # ff_yaml.py:88-104
        p = self.get_parameters("dihedrals", at)
        lj1, lj4 = self.get_parameters("lj", [at[0]]), self.get_parameters("lj", [at[3]])
        return (p.get("scnb", 1), p.get("scee", 1), lj1["sigma14"], lj1["epsilon14"], lj4["sigma14"], lj4["epsilon14"])

    def get_improper(self, *at):
        p = self.get_parameters("impropers", at)
        return p["phi_k"], math.radians(p["phase"]), p["per"]


def _f32(rows):
    """Parameter rows as the reference holds them: rounded to fp32 (see yaml_parameters)."""
    return np.array(rows, dtype=np.float32).astype(np.float64)


def _improper_center(quad, bonded):
    """The atom of an improper bonded to the other three (parameters.py detect_improper_center)."""
    for a in quad:
        if all((a, b) in bonded for b in quad if b != a):
            return a
    raise RuntimeError(f"no central atom found for improper {list(quad)}")


def yaml_parameters(mol, forcefield, terms=None, precision=torch.float32, device="cpu"):
    """``TopologyParameters`` for a duck-typed ``mol`` (charmm.load_molecule or any object with
    atomtype / charge / masses / bonds / angles / dihedrals / impropers) and a YAML force field
    (path, dict or YamlForceField): the reference's ``Parameters(YamlForcefield(mol, yaml), mol,
    terms)`` -- same unique-term ordering, same first-appearance parameter rows.  Like the
    reference (``torch.tensor(list of Python floats)`` is fp32, then ``.type(precision)``) every
    parameter value passes through fp32, also for ``precision=torch.float64``.

    ``"cmap"`` in ``terms`` (not among the defaults) builds CMAP terms from the molecule's ``crossterms`` (C,8) with a
    force field that has ``get_cmap`` (charmm.CharmmPrmForceField); without it they are left out with a warning.  A
    cross-term must be two dihedrals that share three atoms, (a,b,c,d) and (b,c,d,e), as every backbone phi/psi pair
    is; it becomes the 5-atom term (a,b,c,d,e).  The grids keep the file's values (fp64).

    ``"ureybradley"`` (not among the defaults) builds one Urey-Bradley term per unique angle whose type has k_ub > 0,
    from a force field with ``get_urey_bradley`` (charmm.CharmmPrmForceField); ``"nbfix"`` (not among the defaults)
    passes the force field's NBFIX pairs of the molecule's types to ``TopologyParameters(nbfix=...)``, and a 1-4 pair
    whose two types have an NBFIX line takes that line's 1-4 sigma / epsilon instead of the Lorentz-Berthelot mix
    (charmm.CharmmPrmForceField documents the 1-4 rule).  Without ``"ureybradley"``, Urey-Bradley terms the file has for
    this molecule are left out with a warning; without ``"nbfix"`` the tables are the Lorentz-Berthelot ones, silently,
    as they were before NBFIX was read.  A force field without those look-ups raises when the term is asked for."""
    # a force-field object with the reference's interface (YamlForceField, charmm.CharmmPrmForceField), or a YAML path / dict
    ff = forcefield if hasattr(forcefield, "get_LJ") else YamlForceField(forcefield)
    if terms is None:
        terms = ("bonds", "angles", "dihedrals", "impropers", "1-4", "electrostatics", "lj")
    terms = [t.lower() for t in terms]
    T = np.asarray(mol.atomtype, dtype=object)
    uq, types = np.unique(T.astype(str), return_inverse=True)
    masses = getattr(mol, "masses", None)
    if masses is None or len(masses) == 0:
        masses = np.array([ff.get_mass(t) for t in T], dtype=np.float32)  # parameters.py:118-119
    sigma = eps = np.zeros(len(uq))
    if any(t in terms for t in ("lj", "repulsion", "repulsioncg")):
        lj = [ff.get_LJ(t) for t in uq]
        sigma, eps = _f32([p[0] for p in lj]), _f32([p[1] for p in lj])

    def arr(name, width):
        a = getattr(mol, name, None)
        return np.zeros((0, width), dtype=np.int64) if a is None or len(a) == 0 else np.asarray(a, dtype=np.int64).reshape(-1, width)

    def typed(idx, lookup):
        """One parameter row per distinct type tuple, in order of first appearance."""
        rows, row_of, pmap = [], {}, []
        for i, atoms in enumerate(idx):
            key = tuple(T[atoms])
            if key not in row_of:
                row_of[key] = len(rows)
                rows.append(list(lookup(*key)))
            pmap.append([i, row_of[key]])
        return idx, np.array(pmap, dtype=np.int64), _f32(rows)

    def oriented(a):  # first index below last, then unique rows (parameters.py:180-182, 203-205)
        a = a.copy()
        flip = a[:, 0] > a[:, -1]
        a[flip] = a[flip][:, ::-1]
        return np.unique(a, axis=0)

    bonds_raw, angles_raw, dih_raw, imp_raw = arr("bonds", 2), arr("angles", 3), arr("dihedrals", 4), arr("impropers", 4)
    uqbonds = np.unique(np.sort(bonds_raw, axis=1), axis=0) if len(bonds_raw) else bonds_raw
    uqangles = oriented(angles_raw) if len(angles_raw) else angles_raw
    uqdih = oriented(dih_raw) if len(dih_raw) else dih_raw
    bonds = angles = dihedrals = impropers = pairs14 = urey_bradley = nbfix = None
    for term, lookup in (("ureybradley", "get_urey_bradley"), ("nbfix", "get_nbfix")):
        if term in terms and not hasattr(ff, lookup):
            raise RuntimeError(f"'{term}' was asked for, but the force field has no {term} parameters")
    fix = {}  # (type index, type index) -> (sigma, epsilon, sigma14, epsilon14)
    if hasattr(ff, "get_nbfix"):
        for a in range(len(uq)):
            for b in range(a, len(uq)):
                v = ff.get_nbfix(uq[a], uq[b])
                if v is not None:
                    fix[(a, b)] = v
    if fix and "nbfix" in terms:
        nbfix = (np.array(list(fix), np.int64), _f32([[v[0], v[1]] for v in fix.values()]))
    if hasattr(ff, "get_urey_bradley") and len(uqangles):
        rows, row_of, pmap, keep = [], {}, [], []
        for i, atoms in enumerate(uqangles):
            key = tuple(T[atoms])
            ub = ff.get_urey_bradley(*key)
            if ub is None or not ub[0] > 0:
                continue
            if key not in row_of:
                row_of[key] = len(rows)
                rows.append(list(ub))
            pmap.append([len(keep), row_of[key]])
            keep.append(i)
        if keep and "ureybradley" not in terms:
            warnings.warn(f"the molecule has {len(keep)} angles with a Urey-Bradley term; they are left out unless terms "
                          "includes 'ureybradley'", stacklevel=2)
        elif keep:
            urey_bradley = (uqangles[keep], np.array(pmap, np.int64), _f32(rows))
    if "bonds" in terms and len(uqbonds):
        bonds = typed(uqbonds, ff.get_bond)
    if "angles" in terms and len(uqangles):
        angles = typed(uqangles, ff.get_angle)
    if "dihedrals" in terms and len(uqdih):  # parameters.py:198-222, several terms per dihedral
        prm_rows, rows_of, dmap = [], {}, []
        for i, atoms in enumerate(uqdih):
            key = tuple(T[atoms])
            if key not in rows_of:
                rows_of[key] = []
                for term in ff.get_dihedral(*key):
                    rows_of[key].append(len(prm_rows))
                    prm_rows.append(term)
            dmap += [[i, r] for r in rows_of[key]]
        dihedrals = (uqdih, np.array(dmap, dtype=np.int64), _f32(prm_rows))
    if "impropers" in terms and len(imp_raw):  # parameters.py:224-251
        uqimp = np.unique(imp_raw, axis=0)
        bonded = {(int(a), int(b)) for a, b in uqbonds} | {(int(b), int(a)) for a, b in uqbonds}
        rows, row_of, pmap = [], {}, []
        for i, quad in enumerate(uqimp):
            key = tuple(T[quad])
            try:
                prm = ff.get_improper(*key)
            except RuntimeError:
                c = _improper_center([int(q) for q in quad], bonded)
                rest = sorted(int(q) for q in quad if q != c)
                key = tuple(T[[rest[0], rest[1], c, rest[2]]])
                prm = ff.get_improper(*key)
            if key not in row_of:
                row_of[key] = len(rows)
                rows.append(list(prm))
            pmap.append([i, row_of[key]])
        impropers = (uqimp, np.array(pmap, dtype=np.int64), _f32(rows))
    if "1-4" in terms and len(uqdih):  # parameters.py:253-294
        excl = {tuple(b) for b in np.sort(uqbonds, axis=1).tolist()}
        if len(uqangles):
            excl |= {tuple(p) for p in np.sort(uqangles[:, [0, 2]], axis=1).tolist()}
        keep = np.array([tuple(sorted((int(a), int(d)))) not in excl for a, d in uqdih[:, [0, 3]]], dtype=bool)
        d14 = uqdih[keep]
        if len(d14):
            _, first = np.unique(d14[:, [0, 3]], axis=0, return_index=True)
            d14 = d14[first]
            rows, row_of, pmap = [], {}, []
            for i, atoms in enumerate(d14):
                key = tuple(T[atoms])
                scnb, scee, s1, e1, s4, e4 = ff.get_14(*key)
                sig, ep = 0.5 * (s1 + s4), math.sqrt(e1 * e4)
                fx = ff.get_nbfix(key[0], key[3]) if nbfix is not None else None
                if fx is not None:
                    sig, ep = fx[2], fx[3]
                s6 = sig**6
                if key[::-1] in row_of:
                    key = key[::-1]
                if key not in row_of:
                    row_of[key] = len(rows)
                    rows.append([ep * 4 * s6 * s6, ep * 4 * s6, scnb, scee])
                pmap.append([i, row_of[key]])
            pairs14 = (d14[:, [0, 3]], np.array(pmap, dtype=np.int64), _f32(rows))
    cross, cmaps = arr("crossterms", 8), None
    if len(cross) and "cmap" not in terms:
        warnings.warn(f"the molecule has {len(cross)} CMAP cross-terms; they are left out unless terms includes 'cmap'",
                      stacklevel=2)
    elif len(cross):
        if not hasattr(ff, "get_cmap"):
            raise RuntimeError("'cmap' was asked for, but the force field holds no CMAP maps")
        bad = np.any(cross[:, 1:4] != cross[:, 4:7], axis=1)
        if bad.any():
            raise ValueError(f"cross-term {cross[np.argmax(bad)].tolist()} is not two dihedrals (a,b,c,d), (b,c,d,e): "
                             "only that 5-atom form is supported")
        grids, map_of, map_ix = [], [], {}
        for row in cross:
            key = tuple(T[row])
            if key not in map_ix:
                map_ix[key] = len(grids)
                grids.append(np.asarray(ff.get_cmap(key), dtype=np.float64))
            map_of.append(map_ix[key])
        cmaps = (cross[:, [0, 1, 2, 3, 7]], np.array(map_of, np.int64), [len(g) for g in grids], grids)
    return TopologyParameters(
        atom_types=types,
        type_sigma=sigma,
        type_epsilon=eps,
        charges=np.asarray(mol.charge),
        masses=np.asarray(masses, dtype=np.float32),
        bonds=bonds,
        angles=angles,
        dihedrals=dihedrals,
        impropers=impropers,
        pairs14=pairs14,
        cmaps=cmaps,
        urey_bradley=urey_bradley,
        nbfix=nbfix,
        precision=precision,
        device=device,
    )

"""Minimal AMBER readers: ``.prmtop`` topology/parameters, NAMD binary coordinates, ``.xsc``.

SURVEY.md section 8f-2: the reference gets these through moleculekit + parmed
(``torchmd/run.py:158-181``, ``torchmd/forcefields/ff_parmed.py:49-129``,
``torchmd/parameters.py:109-294``), neither of which exists in this image.  This module
reads the same files directly and produces the parameter layout ``Forces`` consumes
(``torchmd_b200.parameters.TopologyParameters``), following the reference pipeline's
semantics step by step:

* moleculekit's prmtop reader: charges = CHARGE / 18.2223, atom types = AMBER_ATOM_TYPE,
  bonds / angles from the ``*_INC_HYDROGEN`` + ``*_WITHOUT_HYDROGEN`` tables (indices / 3),
  dihedral entries with a negative 4th index are impropers, the others proper dihedrals;
* parmed's ``AmberParm`` / ``AmberParameterSet.from_structure``: LJ radius and depth per
  non-bonded type from the diagonal A/B coefficients, ``sigma = 2 rmin 2^(-1/6)``; bond,
  angle and dihedral *types* keyed by AMBER atom-type names (that is how the reference looks
  them up, ``ff_parmed.py:73-129``), angles and phases carried in degrees and converted back
  with ``math.radians`` like ``ff_parmed.py:79,99``;
* the reference ``Parameters`` builder: unique bonds (i<j), angles (first<last), dihedrals
  (first<last), several terms per dihedral, impropers with the centre in the third slot, 1-4
  pairs = dihedral ends that are not bond/angle exclusions, with scnb / scee from the first
  term of the dihedral type and Lorentz-Berthelot A/B from the 1-4 LJ values;
* CMAP correction maps (ff19SB, and chamber files with the ``CHARMM_`` prefix), built only
  when ``amber_parameters`` is asked for ``"cmap"``: ``CMAP_INDEX`` rows are five atoms and a map
  number, ``CMAP_PARAMETER_nn`` is read phi-major (psi fastest) from -180 deg, the way parmed
  reads it.  That ordering is restated from format documentation, not pinned against AMBER's
  own engine.

Pinned by ``tests/test_amber_reader.py`` against the reference's stored known answers for
``tests/data/prod_alanine_dipeptide_amber`` (``tests/test_torchmd.py:517,605``,
``examples/tutorial.ipynb:105``) through the CPU oracle.  Host-only, runs once per set-up.
"""
import math
import re
import struct
import warnings
from itertools import permutations

import numpy as np
import torch

from .parameters import TopologyParameters

AMBER_CHARGE_FACTOR = 18.2223  # prmtop charges are multiplied by this


# ----------------------------------------------------------------------------------------
# file readers
# ----------------------------------------------------------------------------------------
def read_prmtop(path):
    """``{FLAG: list}`` with values typed by the ``%FORMAT`` of each section."""
    out, flag, fmt, buf = {}, None, None, []

    def flush():
        if flag is None:
            return
        m = re.match(r"\(?(\d+)?([aIEFi])(\d+)(?:\.(\d+))?\)?", fmt)
        kind, width = m.group(2), int(m.group(3))
        vals = []
        for line in buf:
            line = line.rstrip("\n")
            for k in range(0, len(line), width):
                tok = line[k : k + width]
                if not tok.strip() and kind != "a":
                    continue
                if kind == "a":
                    vals.append(tok.strip())
                elif kind in "Ii":
                    vals.append(int(tok))
                else:
                    vals.append(float(tok))
        out[flag] = vals

    with open(path) as fh:
        for line in fh:
            if line.startswith("%FLAG"):
                flush()
                flag, fmt, buf = line.split()[1], None, []
            elif line.startswith("%FORMAT"):
                fmt = line[len("%FORMAT") :].strip().replace("(", "").replace(")", "")  # also nested: (8(F9.5))
            elif line.startswith("%VERSION") or line.startswith("%COMMENT"):
                continue
            elif flag is not None:
                buf.append(line)
    flush()
    return out


def read_bincoor(path):
    """NAMD binary coordinates: int32 natoms, then natoms*3 float64 -> (N,3) float32."""
    raw = open(path, "rb").read()
    n = struct.unpack("<i", raw[:4])[0]
    xyz = np.frombuffer(raw, dtype="<f8", count=3 * n, offset=4).reshape(n, 3)
    return xyz.astype(np.float32)


def read_xsc(path):
    """Box lengths (a_x, b_y, c_z) from a NAMD/ACEMD extended-system file."""
    for line in open(path):
        if line.strip() and not line.startswith("#"):
            f = line.split()
            return np.array([float(f[1]), float(f[5]), float(f[9])], dtype=np.float32)
    raise RuntimeError(f"no data line in {path}")


# ----------------------------------------------------------------------------------------
# prmtop -> topology + typed parameters
# ----------------------------------------------------------------------------------------
def _chunks(vals, n):
    a = np.asarray(vals, dtype=np.int64)
    return a.reshape(-1, n) if len(a) else np.zeros((0, n), dtype=np.int64)


class AmberSystem:
    """Topology and per-type parameters of one prmtop (what mol + ParmedForcefield give the
    reference)."""

    def __init__(self, prmtop_path):
        p = read_prmtop(prmtop_path)
        self.natoms = p["POINTERS"][0]
        self.ntypes = p["POINTERS"][1]
        self.ifbox = p["POINTERS"][27]
        self.atomtype = np.array(p["AMBER_ATOM_TYPE"], dtype=object)
        self.charge = (np.array(p["CHARGE"], dtype=np.float64) / AMBER_CHARGE_FACTOR).astype(np.float32)
        self.masses = np.array(p["MASS"], dtype=np.float32)
        self.box = np.zeros(3, dtype=np.float32)
        if self.ifbox and "BOX_DIMENSIONS" in p:
            self.box = np.array(p["BOX_DIMENSIONS"][1:4], dtype=np.float32)

        bonds = np.concatenate([_chunks(p["BONDS_INC_HYDROGEN"], 3), _chunks(p["BONDS_WITHOUT_HYDROGEN"], 3)])
        angles = np.concatenate([_chunks(p["ANGLES_INC_HYDROGEN"], 4), _chunks(p["ANGLES_WITHOUT_HYDROGEN"], 4)])
        dih = np.concatenate([_chunks(p["DIHEDRALS_INC_HYDROGEN"], 5), _chunks(p["DIHEDRALS_WITHOUT_HYDROGEN"], 5)])
        self.bonds = bonds[:, :2] // 3
        self.angles = angles[:, :3] // 3
        quad = np.abs(dih[:, :4]) // 3
        improper = dih[:, 3] < 0
        self.dihedrals = quad[~improper]
        self.impropers = quad[improper]

        # CMAP: terms (a, b, c, d, e) -> map; phi = dihedral(a,b,c,d), psi = dihedral(b,c,d,e)
        pre = "CHARMM_" if "CHARMM_CMAP_COUNT" in p else ""
        self.cmap_idx = np.zeros((0, 5), np.int64)
        self.cmap_map = np.zeros(0, np.int64)
        self.cmap_res = np.zeros(0, np.int64)
        self.cmap_grids = []
        if pre + "CMAP_COUNT" in p:
            nterm, nmap = p[pre + "CMAP_COUNT"][:2]
            self.cmap_res = np.array(p[pre + "CMAP_RESOLUTION"][:nmap], dtype=np.int64)
            for m, r in enumerate(self.cmap_res):
                g = np.array(p[f"{pre}CMAP_PARAMETER_{m + 1:02d}"], dtype=np.float64)
                if len(g) != r * r:
                    raise ValueError(f"{prmtop_path}: CMAP map {m + 1} has {len(g)} values, resolution {r} needs {r * r}")
                self.cmap_grids.append(g.reshape(r, r))
            rows = _chunks(p[pre + "CMAP_INDEX"], 6)[:nterm] - 1
            if len(rows) != nterm or (nterm and (rows[:, 5].min() < 0 or rows[:, 5].max() >= nmap)):
                raise ValueError(f"{prmtop_path}: CMAP_INDEX does not hold {nterm} terms on maps 1..{nmap}")
            self.cmap_idx, self.cmap_map = rows[:, :5], rows[:, 5]

        # ---- per-type parameters, keyed by AMBER atom-type names like parmed's ParameterSet
        nb_idx = np.array(p["ATOM_TYPE_INDEX"], dtype=np.int64) - 1
        acoef, bcoef = p["LENNARD_JONES_ACOEF"], p["LENNARD_JONES_BCOEF"]
        nbparm = p["NONBONDED_PARM_INDEX"]
        rmin, depth = [], []
        for i in range(self.ntypes):  # parmed AmberParm.fill_LJ
            lj = nbparm[self.ntypes * i + i] - 1
            if lj < 0 or acoef[lj] < 1.0e-10:
                rmin.append(0.0)
                depth.append(0.0)
            else:
                factor = 2 * acoef[lj] / bcoef[lj]
                rmin.append(pow(factor, 1.0 / 6.0) * 0.5)
                depth.append(bcoef[lj] / 2 / factor)
        self.lj = {}  # type name -> (sigma, epsilon); first atom of a type defines it
        for i, t in enumerate(self.atomtype):
            if t not in self.lj:
                self.lj[t] = (rmin[nb_idx[i]] * 2 ** (-1.0 / 6.0) * 2, depth[nb_idx[i]])

        def put(table, key, val):
            table.setdefault(key, val)
            table.setdefault(key[::-1], val)

        T = self.atomtype
        self.bond_types, self.angle_types = {}, {}
        bk, br = p["BOND_FORCE_CONSTANT"], p["BOND_EQUIL_VALUE"]
        for a, b, k in bonds // np.array([3, 3, 1]):
            put(self.bond_types, (T[a], T[b]), (bk[k - 1], br[k - 1]))
        ak, ae = p["ANGLE_FORCE_CONSTANT"], p["ANGLE_EQUIL_VALUE"]
        for a, b, c, k in angles // np.array([3, 3, 3, 1]):
            # parmed keeps the equilibrium angle in degrees; the reference converts back (ff_parmed.py:79)
            put(self.angle_types, (T[a], T[b], T[c]), (ak[k - 1], math.radians(ae[k - 1] * 180.0 / math.pi)))

        dk, dper, dphase = p["DIHEDRAL_FORCE_CONSTANT"], p["DIHEDRAL_PERIODICITY"], p["DIHEDRAL_PHASE"]
        scee = p.get("SCEE_SCALE_FACTOR", [1.2] * len(dk))
        scnb = p.get("SCNB_SCALE_FACTOR", [2.0] * len(dk))
        # proper dihedral types: all terms of the FIRST atom quadruple seen with a given type key
        self.dihedral_types, first_quad = {}, {}
        self.improper_types = {}
        for (a, b, c, d, k), q, imp in zip(dih, quad, improper):
            key = tuple(T[q])
            term = (dk[k - 1], math.radians(dphase[k - 1] * 180.0 / math.pi), dper[k - 1], scnb[k - 1], scee[k - 1])
            if imp:
                self.improper_types.setdefault(key, term)
                continue
            canon = key if key in self.dihedral_types else (key[::-1] if key[::-1] in self.dihedral_types else None)
            if canon is None:
                self.dihedral_types[key] = [term]
                first_quad[key] = tuple(q)
            elif first_quad[canon] in (tuple(q), tuple(q[::-1])):
                self.dihedral_types[canon].append(term)

    # lookups with the reference's fall-backs (ff_parmed.py:81-129)
    def dihedral_terms(self, key):
        for var in (tuple(key), tuple(key)[::-1]):
            if var in self.dihedral_types:
                return self.dihedral_types[var]
        raise RuntimeError(f"Could not find dihedral parameters for {key}")

    def improper_term(self, key):
        types = np.array(key, dtype=object)
        for perm in (x for x in permutations((0, 1, 2, 3)) if x[2] == 2):
            k = tuple(types[list(perm)])
            if k in self.improper_types:
                return self.improper_types[k]
        raise RuntimeError(f"Could not find improper parameters for key {key}")


def amber_parameters(system, terms=None, precision=torch.float32, device="cpu"):
    """``TopologyParameters`` for an ``AmberSystem`` -- the reference's
    ``Parameters(ParmedForcefield(mol, prmtop), mol, terms)`` (parameters.py:109-294).  ``"cmap"`` in ``terms``
    (not among the defaults) also builds the file's CMAP terms; without it they are left out with a warning."""
    if terms is None:
        terms = ("bonds", "angles", "dihedrals", "impropers", "1-4", "lj")
    terms = [t.lower() for t in terms]
    T = system.atomtype
    uq, types = np.unique(T, return_inverse=True)
    sigma = [system.lj[t][0] for t in uq]
    eps = [system.lj[t][1] for t in uq]

    def typed(idx, table_lookup, nparam):
        """(idx, map, params): one parameter row per distinct type key, in order of appearance."""
        rows, row_of, pmap = [], {}, []
        for i, atoms in enumerate(idx):
            key = tuple(T[atoms])
            if key not in row_of:
                row_of[key] = len(rows)
                rows.append(list(table_lookup(key))[:nparam])
            pmap.append([i, row_of[key]])
        return idx, np.array(pmap, dtype=np.int64), np.array(rows, dtype=np.float64)

    bonds = angles = dihedrals = impropers = pairs14 = None
    uqbonds = np.unique(np.sort(system.bonds, axis=1), axis=0) if len(system.bonds) else np.zeros((0, 2), np.int64)
    if "bonds" in terms and len(uqbonds):
        bonds = typed(uqbonds, lambda k: system.bond_types[k], 2)
    uqangles = np.zeros((0, 3), np.int64)
    if len(system.angles):
        a = system.angles.copy()
        flip = a[:, 0] > a[:, 2]
        a[flip] = a[flip][:, ::-1]
        uqangles = np.unique(a, axis=0)
    if "angles" in terms and len(uqangles):
        angles = typed(uqangles, lambda k: system.angle_types[k], 2)
    uqdih = np.zeros((0, 4), np.int64)
    if len(system.dihedrals):
        d = system.dihedrals.copy()
        flip = d[:, 0] > d[:, 3]
        d[flip] = d[flip][:, ::-1]
        uqdih = np.unique(d, axis=0)
    if "dihedrals" in terms and len(uqdih):
        prm_rows, rows_of, dmap = [], {}, []
        for i, atoms in enumerate(uqdih):
            key = tuple(T[atoms])
            if key not in rows_of:
                rows_of[key] = []
                for term in system.dihedral_terms(key):
                    rows_of[key].append(len(prm_rows))
                    prm_rows.append(list(term[:3]))
            dmap += [[i, r] for r in rows_of[key]]
        dihedrals = (uqdih, np.array(dmap, dtype=np.int64), np.array(prm_rows, dtype=np.float64))
    if "impropers" in terms and len(system.impropers):
        uqimp = np.unique(system.impropers, axis=0)
        impropers = typed(uqimp, lambda k: system.improper_term(k), 3)
    if "1-4" in terms and len(uqdih):
        excl = set(map(tuple, np.sort(uqbonds, axis=1).tolist()))
        excl |= set(map(tuple, np.sort(uqangles[:, [0, 2]], axis=1).tolist()))
        keep = np.array([tuple(sorted((d0, d3))) not in excl for d0, d3 in uqdih[:, [0, 3]]], dtype=bool)
        d14 = uqdih[keep]
        if len(d14):
            _, first = np.unique(d14[:, [0, 3]], axis=0, return_index=True)
            d14 = d14[first]
            rows, row_of, pmap = [], {}, []
            for i, atoms in enumerate(d14):
                key = tuple(T[atoms])
                if key[::-1] in row_of:
                    key = key[::-1]
                if key not in row_of:
                    term = system.dihedral_terms(key)[0]
                    s1, e1 = system.lj[key[0]]
                    s4, e4 = system.lj[key[3]]
                    sig = 0.5 * (s1 + s4)
                    ep = math.sqrt(e1 * e4)
                    s6 = sig**6
                    row_of[key] = len(rows)
                    rows.append([ep * 4 * s6 * s6, ep * 4 * s6, term[3], term[4]])
                pmap.append([i, row_of[key]])
            pairs14 = (d14[:, [0, 3]], np.array(pmap, dtype=np.int64), np.array(rows, dtype=np.float64))
    cmaps = None
    if len(system.cmap_idx):
        if "cmap" in terms:
            cmaps = (system.cmap_idx, system.cmap_map, system.cmap_res, system.cmap_grids)
        else:
            warnings.warn(f"the topology has {len(system.cmap_idx)} CMAP terms; they are left out unless terms includes 'cmap'",
                          stacklevel=2)
    return TopologyParameters(
        atom_types=types,
        type_sigma=sigma,
        type_epsilon=eps,
        charges=system.charge,
        masses=system.masses,
        bonds=bonds,
        angles=angles,
        dihedrals=dihedrals,
        impropers=impropers,
        pairs14=pairs14,
        cmaps=cmaps,
        precision=precision,
        device=device,
    )

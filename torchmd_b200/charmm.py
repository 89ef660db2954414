"""Minimal CHARMM/X-PLOR PSF and PDB readers -- just what the reference takes from a
moleculekit ``Molecule`` for these formats (parameters.py:25,110-133; npzmol.py:11-39):
atom types, charges, masses, bonds, angles, dihedrals, impropers, coordinates and box.
The reference needs moleculekit for this; the hot path does not.
"""
import math
import types

import numpy as np

_SECTIONS = {"NATOM": 0, "NBOND": 2, "NTHETA": 3, "NPHI": 4, "NIMPHI": 4}


def read_psf(path):
    """dict with atomtype (object array), charge, masses (fp32), bonds (M,2), angles (K,3),
    dihedrals (D,4), impropers (I,4), crossterms (C,8) as zero-based int64 arrays, plus
    name/resname/resid/segid."""
    with open(path) as fh:
        lines = fh.read().split("\n")
    if not lines or not lines[0].startswith("PSF"):
        raise ValueError(f"{path}: not a PSF file")
    sec = {}
    i = 0
    while i < len(lines):
        ln = lines[i]
        if "!N" in ln:
            key = ln.split("!")[1].split(":")[0].split()[0]
            count = int(ln.split()[0])
            body, i = [], i + 1
            while i < len(lines) and lines[i].strip():
                body.append(lines[i])
                i += 1
            sec[key] = (count, body)
        else:
            i += 1
    if "NATOM" not in sec:
        raise ValueError(f"{path}: no !NATOM section")
    natom, rows = sec["NATOM"]
    atoms = [r.split() for r in rows]
    if len(atoms) != natom:
        raise ValueError(f"{path}: !NATOM says {natom}, found {len(atoms)} atom records")

    def index_section(key, width):
        if key not in sec:
            return np.zeros((0, width), dtype=np.int64)
        count, body = sec[key]
        flat = np.array(" ".join(body).split(), dtype=np.int64) - 1
        if len(flat) != count * width:
            raise ValueError(f"{path}: !{key} says {count} entries, found {len(flat) / width:g}")
        if len(flat) and (flat.min() < 0 or flat.max() >= natom):
            raise ValueError(f"{path}: !{key} refers to an atom outside 1..{natom}")
        return flat.reshape(-1, width)

    return {
        "segid": np.array([a[1] for a in atoms], dtype=object),
        "resid": np.array([int(a[2]) for a in atoms], dtype=np.int64),
        "resname": np.array([a[3] for a in atoms], dtype=object),
        "name": np.array([a[4] for a in atoms], dtype=object),
        "atomtype": np.array([a[5] for a in atoms], dtype=object),
        "charge": np.array([float(a[6]) for a in atoms], dtype=np.float32),
        "masses": np.array([float(a[7]) for a in atoms], dtype=np.float32),
        "bonds": index_section("NBOND", 2),
        "angles": index_section("NTHETA", 3),
        "dihedrals": index_section("NPHI", 4),
        "impropers": index_section("NIMPHI", 4),
        "crossterms": index_section("NCRTERM", 8),
    }


def read_pdb(path):
    """(coords (N,3) fp32 of the first model, box (3,) fp32 from CRYST1 or zeros)."""
    xyz, box = [], np.zeros(3, dtype=np.float32)
    with open(path) as fh:
        for line in fh:
            if line.startswith("CRYST1"):
                box = np.array([float(line[6:15]), float(line[15:24]), float(line[24:33])], dtype=np.float32)
            elif line.startswith(("ATOM", "HETATM")):
                xyz.append((float(line[30:38]), float(line[38:46]), float(line[46:54])))
            elif line.startswith("ENDMDL"):
                break
    return np.array(xyz, dtype=np.float32).reshape(-1, 3), box


def read_xtc_first_frame(path):
    """(coords (N,3) or None, box (3,)) in Angstrom from the first frame of a GROMACS .xtc file.  The header (XDR:
    magic 1995, atom count, step, time, 3x3 box in nm) is always plain; the coordinates are plain floats only for up
    to nine atoms (larger frames are compressed -- None is returned for them)."""
    import struct

    with open(path, "rb") as fh:
        b = fh.read()
    magic, natoms, _step = struct.unpack(">iii", b[:12])
    if magic != 1995:
        raise ValueError(f"{path}: not an xtc file (magic {magic})")
    box = np.array(struct.unpack(">9f", b[16:52]), dtype=np.float64).reshape(3, 3)
    xyz = None
    if natoms <= 9:
        xyz = 10.0 * np.array(struct.unpack(">%df" % (3 * natoms), b[56 : 56 + 12 * natoms]), dtype=np.float64).reshape(natoms, 3)
        xyz = xyz.astype(np.float32)
    return xyz, (10.0 * np.diag(box)).astype(np.float32)


def load_molecule(psf_path, pdb_path=None):
    """The duck-typed ``mol`` the reference's Parameters / System set-up reads
    (SURVEY.md section 8c): numAtoms, atomtype, charge, masses, bonds, angles, dihedrals,
    impropers, coords (N,3,1), box (3,1)."""
    top = read_psf(psf_path)
    mol = types.SimpleNamespace(**top)
    mol.numAtoms = len(top["atomtype"])
    mol.coords = np.zeros((mol.numAtoms, 3, 1), dtype=np.float32)
    mol.box = np.zeros((3, 1), dtype=np.float32)
    if pdb_path is not None:
        xyz, box = read_pdb(pdb_path)
        if len(xyz) != mol.numAtoms:
            raise ValueError(f"{pdb_path}: {len(xyz)} atoms, the PSF has {mol.numAtoms}")
        mol.coords = xyz[:, :, None].copy()
        mol.box = box[:, None].copy()
    return mol


class CharmmPrmForceField:
    """A CHARMM parameter file (``.prm`` / ``.par``) behind the reference's force-field interface
    (torchmd/forcefields/forcefield.py:5-43), with the look-up semantics of its parmed adapter
    (ff_parmed.py:49-129), which this image cannot run (no parmed):

    * bonds, angles: exact type tuple, either direction; Urey-Bradley columns are ignored (ff_parmed.py:73-75
      returns only k, theta_eq);
    * dihedrals: exact type tuple or its reverse (ff_parmed.py:77-95, no wildcard matching there); lines that
      repeat a key add a term, a repeated periodicity replaces the earlier one (parmed's CharmmParameterSet);
    * 1-4: scnb = scee = 1 (parmed's default for CHARMM dihedral types) and the types' 1-4 sigma / epsilon -- the
      second column triple of a NONBONDED line when present, else the ordinary values (ff_parmed.py:97-113);
    * LJ: epsilon = |eps|, sigma = (Rmin/2) * 2 * 2^(-1/6); NBFIX pairs are not used (the adapter reads only the
      per-type values; the reference's own test notes "I don't have nbfix", tests/test_torchmd.py:326);
    * impropers (harmonic, periodicity 0): parmed keys them by the SORTED type tuple; the adapter tries the
      permutations that keep position 2 (ff_parmed.py:115-129).  This part of parmed is restated from its
      documentation, not pinned: fixtures with impropers are labelled so in tests/golden.
    * CMAP (not in the reference): a header of the 8 atom types of the two dihedrals and the resolution n, then
      n * n values, one phi row of n psi values after another from -180 deg; ``get_cmap`` matches the exact 8-tuple.
    """

    SECTIONS = ("ATOMS", "BONDS", "ANGLES", "THETAS", "DIHEDRALS", "PHI", "IMPROPER", "IMPROPERS", "IMPHI", "CMAP", "NONBONDED",
                "NBONDED", "NBFIX", "HBOND", "END")

    def __init__(self, path, mol=None):
        self.mol = mol
        self.bonds, self.angles, self.dihedrals, self.impropers, self.lj, self.masses = {}, {}, {}, {}, {}, {}
        self.cmaps = {}  # 8 atom types -> (n, n) grid, phi-major
        cmap_key, cmap_vals, cmap_res = None, [], 0
        section, carry = None, ""
        for raw in open(path):
            line = raw.split("!")[0].strip()
            if not line or line.startswith("*"):
                continue
            if line.endswith("-"):  # continuation (the NONBONDED header)
                carry += line[:-1] + " "
                continue
            line, carry = carry + line, ""
            w = line.split()
            head = w[0].upper()
            if head in self.SECTIONS:
                section = {"THETAS": "ANGLES", "PHI": "DIHEDRALS", "IMPROPERS": "IMPROPER", "IMPHI": "IMPROPER", "NBONDED": "NONBONDED"}.get(head, head)
                continue
            if head == "MASS" and len(w) >= 4:
                self.masses[w[2].upper()] = float(w[3])
                continue
            try:
                if section == "BONDS":
                    a, b = w[0].upper(), w[1].upper()
                    self.bonds[(a, b)] = self.bonds[(b, a)] = (float(w[2]), float(w[3]))
                elif section == "ANGLES":
                    a, b, c = (x.upper() for x in w[:3])
                    self.angles[(a, b, c)] = self.angles[(c, b, a)] = (float(w[3]), float(w[4]))
                elif section == "DIHEDRALS":
                    key = tuple(x.upper() for x in w[:4])
                    term = [float(w[4]), math.radians(float(w[6])), int(float(w[5]))]
                    for k in (key, key[::-1]):
                        terms = [t for t in self.dihedrals.get(k, []) if t[2] != term[2]]
                        self.dihedrals[k] = terms + [term]
                elif section == "IMPROPER":
                    key = tuple(sorted(x.upper() for x in w[:4]))
                    k, per = float(w[4]), int(float(w[5]))
                    psi = float(w[6]) if len(w) > 6 else float(w[5])
                    self.impropers[key] = (k, math.radians(psi), per)
                elif section == "NONBONDED":
                    t = w[0].upper()
                    eps, rmin_half = abs(float(w[2])), float(w[3])
                    eps14, rmin14_half = (abs(float(w[5])), float(w[6])) if len(w) >= 7 else (eps, rmin_half)
                    f = 2.0 * 2.0 ** (-1.0 / 6.0)
                    self.lj[t] = (rmin_half * f, eps, rmin14_half * f, eps14)
                elif section == "CMAP":
                    if cmap_key is None:  # header: 8 atom types and the resolution
                        cmap_res = int(w[8])
                        cmap_key, cmap_vals = tuple(x.upper() for x in w[:8]), []
                    else:
                        cmap_vals += [float(x) for x in w]
                    if len(cmap_vals) >= cmap_res * cmap_res:
                        if len(cmap_vals) > cmap_res * cmap_res:
                            raise ValueError(f"{path}: CMAP {cmap_key} holds more than {cmap_res}^2 values")
                        self.cmaps[cmap_key] = np.array(cmap_vals, dtype=np.float64).reshape(cmap_res, cmap_res)
                        cmap_key = None
            except (ValueError, IndexError):
                if section == "CMAP" and cmap_key is not None:
                    raise ValueError(f"{path}: CMAP {cmap_key} ends after {len(cmap_vals)} of {cmap_res}^2 values") from None
                continue  # keyword lines inside a section (cutnb ..., HBOND CUTHB ...)

    # ---- the reference's _ForceFieldBase interface -------------------------------------------------
    def get_atom_types(self):
        return np.unique(self.mol.atomtype)

    def get_charge(self, at):
        return self.mol.charge[np.where(self.mol.atomtype == at)[0][0]]

    def get_mass(self, at):
        if self.mol is not None and getattr(self.mol, "masses", None) is not None and len(self.mol.masses):
            return self.mol.masses[np.where(self.mol.atomtype == at)[0][0]]
        return self.masses[str(at).upper()]

    def get_LJ(self, at):
        s = self.lj[str(at).upper()]
        return s[0], s[1]

    def get_bond(self, at1, at2):
        return self.bonds[(str(at1).upper(), str(at2).upper())]

    def get_angle(self, at1, at2, at3):
        k, theta = self.angles[(str(at1).upper(), str(at2).upper(), str(at3).upper())]
        return k, math.radians(theta)

    def _dihedral_terms(self, at):
        key = tuple(str(a).upper() for a in at)
        if key not in self.dihedrals:
            raise RuntimeError(f"Could not find dihedral parameters for {key}")
        return self.dihedrals[key]

    def get_dihedral(self, at1, at2, at3, at4):
        return [list(t) for t in self._dihedral_terms((at1, at2, at3, at4))]

    def get_14(self, at1, at2, at3, at4):
        self._dihedral_terms((at1, at2, at3, at4))
        l1, l4 = self.lj[str(at1).upper()], self.lj[str(at4).upper()]
        return 1.0, 1.0, l1[2], l1[3], l4[2], l4[3]

    def get_cmap(self, types8):
        """The (n, n) grid of the cross-term with these 8 atom types (exact match, phi-major, kcal/mol)."""
        key = tuple(str(a).upper() for a in types8)
        if key not in self.cmaps:
            raise RuntimeError(f"Could not find CMAP parameters for {key}")
        return self.cmaps[key]

    def get_improper(self, at1, at2, at3, at4):
        from itertools import permutations

        types = [str(a).upper() for a in (at1, at2, at3, at4)]
        for p in permutations((0, 1, 2, 3)):
            if p[2] != 2:
                continue
            key = tuple(types[i] for i in p)
            if key in self.impropers:  # (parmed's keys are sorted tuples: a permutation matches only if it is sorted)
                return self.impropers[key]
        raise RuntimeError(f"Could not find improper parameters for key {types}")

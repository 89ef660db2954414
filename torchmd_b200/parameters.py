"""Parameter container with the attribute layout the force kernels consume.

The reference builds this layout from a moleculekit ``Molecule`` plus a
force-field file (``torchmd/parameters.py:6-134``, out of scope here: it is a
once-per-run host parser).  The *layout* of its output is the input contract of
``Forces`` (SURVEY.md section 8b), so this module provides a container with the
same attribute names that is filled straight from arrays.  A reference
``Parameters`` object can be passed to ``torchmd_b200.Forces`` unchanged as well
(duck typing); nothing here is needed in that case.

Layout (per term ``bond/angle/dihedral/improper/nonbonded_14``):
``{"idx": (M,k) int64, "map": (M',2) int64 [row -> param row], "params": (K,p)}``
with p = 2 (k, r0 | k, theta0 rad), 3 (k, phi0 rad, periodicity), 4 (A, B, scnb, scee).

CMAP correction maps (not in the reference) are ``cmap_params = {"idx": (n,5) int64, "map_of": (n,) int64,
"res": (nmaps,) int64, "grids": (sum res^2,) float64}``: term t acts on atoms idx[t] with phi = dihedral(idx[t,0:4]),
psi = dihedral(idx[t,1:5]) and map map_of[t]; map m holds E(phi_i, psi_j) at phi_i = -180 deg + i 360 deg / res[m]
(psi alike), phi-major, in kcal/mol.  The grids stay fp64 in both precisions.
"""
import numpy as np
import torch


def lorentz_berthelot_AB(sigma, epsilon):
    """LJ ``A = 4 eps sigma^12``, ``B = 4 eps sigma^6`` tables over atom types.

    Same combination rule and operation order as ``torchmd/parameters.py:449-457``
    (sigma_ij = (s_i+s_j)/2, eps_ij = sqrt(e_i e_j)), evaluated in the dtype of
    ``sigma`` so the tables agree with the reference's to the last bit.
    """
    half_sum = 0.5 * (sigma + sigma[:, None])
    eps_ij = torch.sqrt(epsilon * epsilon[:, None])
    s6 = half_sum**6
    B = eps_ij * 4 * s6
    A = eps_ij * 4 * s6 * s6
    return A, B


def _term(idx, pmap, params, dtype):
    if idx is None or len(idx) == 0:
        return None
    idx = torch.as_tensor(np.asarray(idx), dtype=torch.int64)
    pmap = torch.as_tensor(np.asarray(pmap), dtype=torch.int64)
    params = torch.as_tensor(np.asarray(params, dtype=np.float64)).to(dtype)
    return {"idx": idx, "map": pmap, "params": params}


def _cmap(idx, map_of, res, grids, natoms):
    idx = torch.as_tensor(np.asarray(idx, dtype=np.int64).reshape(-1, 5))
    map_of = torch.as_tensor(np.asarray(map_of, dtype=np.int64).reshape(-1))
    res = torch.as_tensor(np.asarray(res, dtype=np.int64).reshape(-1))
    if isinstance(grids, (list, tuple)):  # one (res, res) grid per map
        grids = np.concatenate([np.ravel(np.asarray(g, dtype=np.float64)) for g in grids])
    grids = torch.as_tensor(np.ravel(np.asarray(grids, dtype=np.float64)))
    if len(map_of) != len(idx) or int(map_of.min()) < 0 or int(map_of.max()) >= len(res):
        raise ValueError("cmaps: map_of must give one map index in 0..nmaps-1 per term")
    if int(idx.min()) < 0 or int(idx.max()) >= natoms:
        raise ValueError("cmaps: atom index out of range")
    if int((res * res).sum()) != len(grids):
        raise ValueError(f"cmaps: the grids hold {len(grids)} values, the resolutions need {int((res * res).sum())}")
    return {"idx": idx, "map_of": map_of, "res": res, "grids": grids}


class TopologyParameters:
    """Array-built stand-in for the reference ``Parameters`` object."""

    def __init__(
        self,
        atom_types,
        type_sigma,
        type_epsilon,
        charges,
        masses,
        bonds=None,
        angles=None,
        dihedrals=None,
        impropers=None,
        pairs14=None,
        cmaps=None,
        precision=torch.float32,
        device="cpu",
    ):
        """
        atom_types   : (N,) integer type id per atom (``mapped_atom_types``)
        type_sigma, type_epsilon : (T,) LJ parameters per type
        charges, masses : (N,)
        bonds/angles/dihedrals/impropers/pairs14 : optional ``(idx, map, params)``
            triples in the layout described in the module docstring.
        cmaps : optional ``(idx (n,5), map_of (n,), res (nmaps,), grids)`` CMAP terms and maps (module docstring)
        """
        self.natoms = int(len(atom_types))
        self.mapped_atom_types = torch.as_tensor(
            np.asarray(atom_types), dtype=torch.int64
        )
        # reference keeps charges in the run precision and masses as (N,1)
        self.charges = torch.as_tensor(np.asarray(charges, dtype=np.float64))
        self.masses = torch.as_tensor(np.asarray(masses, dtype=np.float32))[:, None]
        nb = np.stack(
            [np.asarray(type_sigma, np.float64), np.asarray(type_epsilon, np.float64)],
            axis=1,
        )
        self.nonbonded_params = {
            "map": torch.stack(
                [torch.arange(self.natoms), self.mapped_atom_types], dim=1
            ),
            "params": torch.as_tensor(nb),
        }
        self.bond_params = _term(*bonds, torch.float64) if bonds else None
        self.angle_params = _term(*angles, torch.float64) if angles else None
        self.dihedral_params = _term(*dihedrals, torch.float64) if dihedrals else None
        self.improper_params = _term(*impropers, torch.float64) if impropers else None
        self.nonbonded_14_params = _term(*pairs14, torch.float64) if pairs14 else None
        self.cmap_params = _cmap(*cmaps, self.natoms) if cmaps is not None and len(cmaps[0]) else None
        self.A = None
        self.B = None
        self.device = "cpu"
        self.precision_(precision)
        self.to_(device)

    # -- same mutators as torchmd/parameters.py:33-87 -------------------------
    def _terms(self):
        return [
            self.nonbonded_params,
            self.bond_params,
            self.angle_params,
            self.dihedral_params,
            self.improper_params,
            self.nonbonded_14_params,
        ]

    def to_(self, device):
        self.charges = self.charges.to(device)
        self.masses = self.masses.to(device)
        self.mapped_atom_types = self.mapped_atom_types.to(device)
        for t in self._terms():
            if t is not None:
                for k in t:
                    t[k] = t[k].to(device)
        if self.cmap_params is not None:
            self.cmap_params = {k: v.to(device) for k, v in self.cmap_params.items()}
        if self.A is not None:
            self.A, self.B = self.A.to(device), self.B.to(device)
        self.device = device

    def precision_(self, precision):
        self.charges = self.charges.type(precision)
        self.masses = self.masses.type(precision)
        for t in self._terms():
            if t is not None:
                t["params"] = t["params"].type(precision)

    def get_AB(self):
        p = self.nonbonded_params["params"]
        return lorentz_berthelot_AB(p[:, 0], p[:, 1])

    def get_exclusions(self, types=("bonds", "angles", "1-4"), fullarray=False):
        """Excluded pair list: bonded pairs, angle ends, dihedral ends
        (same selection as ``torchmd/parameters.py:89-107``)."""
        out = []
        if self.bond_params is not None and "bonds" in types:
            out += self.bond_params["idx"].cpu().numpy().tolist()
        if self.angle_params is not None and "angles" in types:
            out += self.angle_params["idx"].cpu().numpy()[:, [0, 2]].tolist()
        if self.dihedral_params is not None and "1-4" in types:
            out += self.dihedral_params["idx"].cpu().numpy()[:, [0, 3]].tolist()
        if fullarray:
            mat = np.zeros((self.natoms, self.natoms), dtype=bool)
            if len(out):
                e = np.array(out)
                mat[e[:, 0], e[:, 1]] = True
                mat[e[:, 1], e[:, 0]] = True
            return mat
        return out

"""CMAP on the host: the prmtop / PSF / CHARMM parameter readers, the parameter builders, and the fp64 oracle
(oracle/cmap.py) against the map it interpolates and against finite differences of its own energy."""
import math
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import cmap as ocmap

ALA2 = "data/prod_alanine_dipeptide_amber/structure.prmtop"
C36 = "data/waterbox/parameters.prm"
ALA_KEY = ("C", "NH1", "CT1", "C", "NH1", "CT1", "C", "NH1")


def trig(phi, psi):
    return np.cos(phi) + 0.5 * np.sin(2 * psi + 0.3) + 0.2 * np.cos(phi - psi)


def grid_of(f, n):
    a = -math.pi + 2 * math.pi * np.arange(n) / n
    return f(*np.meshgrid(a, a, indexing="ij"))


def _block(flag, fmt, lines):
    return [f"%FLAG {flag}", f"%FORMAT({fmt})"] + lines


def write_cmap_prmtop(reference_inputs, path, prefix=""):
    """The alanine-dipeptide prmtop with one CMAP term C(ACE)-N-CA-C-N(NME) on a 24x24 map written as 8(F9.5)."""
    from torchmd_b200.amber import read_prmtop

    src = os.path.join(reference_inputs, ALA2)
    names = read_prmtop(src)["ATOM_NAME"]
    c_atoms = [i for i, nm in enumerate(names) if nm == "C"]
    n_atoms = [i for i, nm in enumerate(names) if nm == "N"]
    term = [c_atoms[0], n_atoms[0], names.index("CA"), c_atoms[1], n_atoms[1]]
    grid = np.round(grid_of(trig, 24), 5)
    vals = [f"{v:9.5f}" for v in grid.ravel()]
    lines = []
    lines += _block(prefix + "CMAP_COUNT", "2I8", [f"{1:8d}{1:8d}"])
    lines += _block(prefix + "CMAP_RESOLUTION", "20I4", [f"{24:4d}"])
    lines += _block(prefix + "CMAP_PARAMETER_01", "8(F9.5)", ["".join(vals[k : k + 8]) for k in range(0, len(vals), 8)])
    lines += _block(prefix + "CMAP_INDEX", "6I8", ["".join(f"{a + 1:8d}" for a in term) + f"{1:8d}"])
    with open(src) as fh:
        text = fh.read()
    with open(path, "w") as fh:
        fh.write(text.rstrip("\n") + "\n" + "\n".join(lines) + "\n")
    return term, grid


@pytest.mark.parametrize("prefix", ["", "CHARMM_"])
def test_prmtop_with_cmap_parses_and_round_trips(reference_inputs, tmp_path, prefix):
    from torchmd_b200.amber import AmberSystem, amber_parameters, read_prmtop

    path = str(tmp_path / "ala2_cmap.prmtop")
    term, grid = write_cmap_prmtop(reference_inputs, path, prefix)
    assert term == [4, 6, 8, 14, 16]
    assert len(read_prmtop(path)[prefix + "CMAP_PARAMETER_01"]) == 576  # the nested %FORMAT(8(F9.5))
    s = AmberSystem(path)
    assert s.cmap_idx.tolist() == [term] and s.cmap_map.tolist() == [0] and s.cmap_res.tolist() == [24]
    assert np.array_equal(s.cmap_grids[0], grid)
    par = amber_parameters(s, terms=("bonds", "angles", "dihedrals", "impropers", "1-4", "lj", "cmap"))
    c = par.cmap_params
    assert c["idx"].tolist() == [term] and c["res"].tolist() == [24] and c["grids"].dtype == torch.float64
    assert np.array_equal(c["grids"].numpy(), grid.ravel())
    p64 = amber_parameters(s, terms=("dihedrals", "cmap"), precision=torch.float64)
    assert torch.equal(p64.cmap_params["grids"], c["grids"])
    with pytest.warns(UserWarning, match="1 CMAP terms"):
        plain = amber_parameters(s)
    assert plain.cmap_params is None


def _same_parameters(a, b):
    assert torch.equal(a.mapped_atom_types, b.mapped_atom_types) and torch.equal(a.charges, b.charges)
    for t in ("bond_params", "angle_params", "dihedral_params", "improper_params", "nonbonded_14_params", "nonbonded_params"):
        x, y = getattr(a, t), getattr(b, t)
        assert (x is None) == (y is None), t
        if x is not None:
            assert x.keys() == y.keys() and all(torch.equal(x[k], y[k]) for k in x), t
    assert a.cmap_params is None and b.cmap_params is None


def test_cmap_request_changes_nothing_without_cross_terms(reference_inputs):
    from torchmd_b200.amber import AmberSystem, amber_parameters
    from torchmd_b200.charmm import CharmmPrmForceField, load_molecule
    from torchmd_b200.ff_yaml import yaml_parameters

    s = AmberSystem(os.path.join(reference_inputs, ALA2))
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        _same_parameters(amber_parameters(s), amber_parameters(s, terms=("bonds", "angles", "dihedrals", "impropers", "1-4", "lj", "cmap")))
        for d in ("benzamidine", "waterbox"):
            base = os.path.join(reference_inputs, "data", d)
            mol = load_molecule(os.path.join(base, "mol.psf" if d == "benzamidine" else "structure.psf"))
            ff = CharmmPrmForceField(os.path.join(base, "mol.prm" if d == "benzamidine" else "parameters.prm"), mol)
            _same_parameters(yaml_parameters(mol, ff), yaml_parameters(mol, ff, terms=("bonds", "angles", "dihedrals", "impropers", "1-4", "electrostatics", "lj", "cmap")))


def test_c36_prm_has_six_24x24_maps(reference_inputs):
    from torchmd_b200.charmm import CharmmPrmForceField

    ff = CharmmPrmForceField(os.path.join(reference_inputs, C36))
    assert len(ff.cmaps) == 6 and all(g.shape == (24, 24) for g in ff.cmaps.values())
    ala = ff.get_cmap(ALA_KEY)
    assert ala[0, 0] == 0.13 and ala[-1, -1] == -1.81  # (-180, -180) and (165, 165) in the file text
    assert ala[0, 1] == 0.77 and ala[-1, 0] == -0.81  # psi runs fastest within a "!phi" block (the "!165" one starts -0.81)
    with pytest.raises(RuntimeError, match="CMAP"):
        ff.get_cmap(("C",) * 8)


PSF = """PSF

       1 !NTITLE
 REMARKS one alanine backbone cross-term

       {n} !NATOM
{atoms}

       {nb} !NBOND: bonds
{bonds}

       0 !NTHETA: angles

       0 !NPHI: dihedrals

       0 !NIMPHI: impropers

       1 !NCRTERM: cross-terms
{cross}
"""


def write_psf(path, types, cross):
    n = len(types)
    atoms = "\n".join(f"{i + 1:8d} P1   1    ALA  A{i:<4d} {t:<6s} 0.000000 12.0110 0" for i, t in enumerate(types))
    bonds = "".join(f"{i + 1:8d}{i + 2:8d}" for i in range(n - 1))
    open(path, "w").write(PSF.format(n=n, atoms=atoms, nb=n - 1, bonds=bonds, cross="".join(f"{a + 1:8d}" for a in cross)))


def test_psf_cross_term_finds_the_alanine_map(reference_inputs, tmp_path):
    from torchmd_b200.charmm import CharmmPrmForceField, load_molecule, read_psf
    from torchmd_b200.ff_yaml import yaml_parameters

    path = str(tmp_path / "ala.psf")
    write_psf(path, ["C", "NH1", "CT1", "C", "NH1"], [0, 1, 2, 3, 1, 2, 3, 4])
    assert read_psf(path)["crossterms"].tolist() == [[0, 1, 2, 3, 1, 2, 3, 4]]
    mol = load_molecule(path)
    ff = CharmmPrmForceField(os.path.join(reference_inputs, C36), mol)
    par = yaml_parameters(mol, ff, terms=["cmap"])
    c = par.cmap_params
    assert c["idx"].tolist() == [[0, 1, 2, 3, 4]] and c["map_of"].tolist() == [0] and c["res"].tolist() == [24]
    assert np.array_equal(c["grids"].numpy(), ff.get_cmap(ALA_KEY).ravel())
    with pytest.warns(UserWarning, match="1 CMAP cross-terms"):
        assert yaml_parameters(mol, ff, terms=["bonds"]).cmap_params is None


def test_non_backbone_cross_term_is_refused(reference_inputs, tmp_path):
    from torchmd_b200.charmm import CharmmPrmForceField, load_molecule
    from torchmd_b200.ff_yaml import yaml_parameters

    path = str(tmp_path / "odd.psf")
    write_psf(path, ["C", "NH1", "CT1", "C", "NH1", "CT1"], [0, 1, 2, 3, 2, 3, 4, 5])
    mol = load_molecule(path)
    ff = CharmmPrmForceField(os.path.join(reference_inputs, C36), mol)
    with pytest.raises(ValueError, match="5-atom form"):
        yaml_parameters(mol, ff, terms=["cmap"])


def test_missing_map_raises(reference_inputs, tmp_path):
    from torchmd_b200.charmm import CharmmPrmForceField, load_molecule
    from torchmd_b200.ff_yaml import yaml_parameters

    path = str(tmp_path / "nomap.psf")
    write_psf(path, ["C", "NH1", "CT1", "C", "OH1"], [0, 1, 2, 3, 1, 2, 3, 4])
    mol = load_molecule(path)
    with pytest.raises(RuntimeError, match="Could not find CMAP"):
        yaml_parameters(mol, CharmmPrmForceField(os.path.join(reference_inputs, C36), mol), terms=["cmap"])


# ---- the oracle -------------------------------------------------------------------------------------------------------
def test_oracle_passes_through_the_grid():
    rng = np.random.default_rng(0)
    for n in (5, 24, 36):
        grid = rng.normal(size=(n, n))
        coef = ocmap.coefficients(grid)
        a = -math.pi + 2 * math.pi * np.arange(n) / n
        phi, psi = np.meshgrid(a, a, indexing="ij")
        E, _, _ = ocmap.map_energy(coef, phi, psi)
        assert np.abs(E - grid).max() <= 1e-12
        E2, _, _ = ocmap.map_energy(coef, phi + 2 * math.pi, psi - 2 * math.pi)  # periodic
        assert np.abs(E2 - grid).max() <= 1e-12


def test_oracle_interpolates_an_asymmetric_function_with_the_right_convention():
    coef = ocmap.coefficients(grid_of(trig, 24))
    rng = np.random.default_rng(1)
    phi, psi = rng.uniform(-math.pi, math.pi, size=(2, 2000))
    E, dphi, dpsi = ocmap.map_energy(coef, phi, psi)
    assert np.abs(E - trig(phi, psi)).max() < 2e-3
    assert np.abs(dphi - (-np.sin(phi) - 0.2 * np.sin(phi - psi))).max() < 2e-2
    assert np.abs(dpsi - (np.cos(2 * psi + 0.3) + 0.2 * np.sin(phi - psi))).max() < 2e-2
    # the mistakes this would catch: phi and psi swapped, or the grid taken to start at 0 deg
    assert np.abs(E - trig(psi, phi)).max() > 0.3
    assert np.abs(E - trig(phi + math.pi, psi + math.pi)).max() > 0.3


def test_oracle_forces_are_minus_the_gradient():
    rng = np.random.default_rng(2)
    pos = rng.normal(scale=1.5, size=(9, 3))
    idx = np.array([[0, 1, 2, 3, 4], [3, 4, 5, 6, 7], [8, 2, 1, 5, 0]])
    grids = np.concatenate([grid_of(trig, 24).ravel(), rng.normal(size=10 * 10)])
    args = (idx, [0, 1, 0], [24, 10], grids)
    _, F = ocmap.energy_forces(pos, *args)
    h = 1e-6
    fd = np.zeros_like(pos)
    for a in range(len(pos)):
        for k in range(3):
            p, m = pos.copy(), pos.copy()
            p[a, k] += h
            m[a, k] -= h
            fd[a, k] = -(ocmap.energy_forces(p, *args)[0] - ocmap.energy_forces(m, *args)[0]) / (2 * h)
    assert np.abs(F - fd).max() <= 1e-6 * max(1.0, np.abs(F).max())
    # periodic images: the same terms with atoms moved by whole boxes
    box = np.array([20.0, 21.0, 22.0])  # (every bond vector below half a box)
    shifted = pos + rng.integers(-2, 3, size=pos.shape) * box
    E1, F1 = ocmap.energy_forces(pos, *args)
    E2, F2 = ocmap.energy_forces(shifted, *args, box=box)
    assert abs(E1 - E2) < 1e-9 and np.abs(F1 - F2).max() < 1e-9

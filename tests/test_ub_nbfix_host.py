"""Urey-Bradley terms and NBFIX overrides on the host: the CHARMM .prm and AMBER prmtop readers, the builders, the
TopologyParameters tables and the numpy oracle (oracle/urey_bradley.py).  Input files: tests/golden/reference_inputs.npz."""
import math
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import urey_bradley as oub

C36 = ("data", "waterbox", "parameters.prm")
ALA2 = ("data", "prod_alanine_dipeptide_amber", "structure.prmtop")


def test_charmm36_urey_bradley_and_nbfix_lines(reference_inputs):
    from torchmd_b200 import charmm

    ff = charmm.CharmmPrmForceField(os.path.join(reference_inputs, *C36))
    assert len({(min(a, c), b, max(a, c)) for a, b, c in ff.ub}) == 496
    assert ff.get_urey_bradley("NH2", "CT1", "HB1") == (50.0, 2.14) == ff.get_urey_bradley("HB1", "CT1", "NH2")
    assert ff.get_urey_bradley("CA", "CA", "CA") == (35.0, 2.4162)
    assert ff.get_urey_bradley("CT1", "C", "O") is None  # an angle line without the two columns
    assert len({tuple(sorted(k)) for k in ff.nbfix}) == 12
    sig, eps, sig14, eps14 = ff.get_nbfix("SOD", "CLA")
    assert ff.get_nbfix("CLA", "SOD") == (sig, eps, sig14, eps14)
    assert eps == 0.083875 and sig == 3.731 * 2.0 ** (-1.0 / 6.0) and (sig14, eps14) == (sig, eps)
    assert ff.get_nbfix("SOD", "SOD") is None


PRM = """* synthetic: one 1-4 pair of types with an NBFIX line
ATOMS
MASS 1 AA 12.0
MASS 2 BB 12.0
MASS 3 DD 12.0
MASS 4 EE 12.0
BONDS
AA BB 300.0 1.5
BB BB 300.0 1.5
BB DD 300.0 1.5
BB EE 300.0 1.5
ANGLES
AA BB BB 50.0 110.0 20.0 2.5
BB BB DD 50.0 110.0
BB BB EE 50.0 110.0 0.0 2.5
DIHEDRALS
AA BB BB DD 0.2 3 0.0
AA BB BB EE 0.2 3 0.0
NONBONDED nbxmod 5 atom cdiel -
cutnb 14.0
AA 0.0 -0.10 2.00 0.0 -0.05 1.80
BB 0.0 -0.10 2.00
DD 0.0 -0.20 1.90
EE 0.0 -0.30 1.70
NBFIX
AA DD -0.50 3.60 -0.25 3.40
AA EE -0.40 3.50
END
"""


def five_atoms(tmp_path):
    """AA-BB-BB-DD with a second end EE on the middle: 1-4 pairs AA-DD (NBFIX with 14 columns), AA-EE (without)."""
    import types

    from torchmd_b200 import charmm

    path = tmp_path / "syn.prm"
    path.write_text(PRM)
    mol = types.SimpleNamespace(atomtype=np.array(["AA", "BB", "BB", "DD", "EE"], dtype=object), charge=np.zeros(5, np.float32),
                                masses=np.full(5, 12.0, np.float32), bonds=np.array([[0, 1], [1, 2], [2, 3], [2, 4]]),
                                angles=np.array([[0, 1, 2], [1, 2, 3], [1, 2, 4]]), dihedrals=np.array([[0, 1, 2, 3], [0, 1, 2, 4]]),
                                impropers=np.zeros((0, 4), np.int64))
    return mol, charmm.CharmmPrmForceField(str(path), mol)


TERMS = ["bonds", "angles", "dihedrals", "1-4", "lj"]


def test_nbfix_pairs_and_the_14_rule(tmp_path):
    from torchmd_b200.ff_yaml import yaml_parameters

    mol, ff = five_atoms(tmp_path)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # (the Urey-Bradley term left out)
        plain = yaml_parameters(mol, ff, terms=TERMS, precision=torch.float64)
        par = yaml_parameters(mol, ff, terms=TERMS + ["nbfix"], precision=torch.float64)
    assert plain.nbfix_params is None
    f6 = 2.0 ** (-1.0 / 6.0)
    uq = ["AA", "BB", "DD", "EE"]
    got = {(uq[i], uq[j]): tuple(p) for (i, j), p in zip(par.nbfix_params["idx"].tolist(), par.nbfix_params["params"].tolist())}
    assert got == {("AA", "DD"): (float(np.float32(3.60 * f6)), float(np.float32(0.50))),
                   ("AA", "EE"): (float(np.float32(3.50 * f6)), float(np.float32(0.40)))}

    def ab(sig, eps):
        s6 = sig**6
        return float(np.float32(eps * 4 * s6 * s6)), float(np.float32(eps * 4 * s6))

    rows = par.nonbonded_14_params
    prm = rows["params"].numpy()[rows["map"].numpy()[:, 1]]
    pairs = rows["idx"].numpy().tolist()
    want = {(0, 3): ab(3.40 * f6, 0.25), (0, 4): ab(3.50 * f6, 0.40)}  # 14 columns when given, else the pair's own values
    for (i, j), p in zip(pairs, prm):
        assert tuple(p[:2]) == want[(i, j)], (i, j)
    # without "nbfix" the 1-4 rows are the Lorentz-Berthelot mix of the types' 1-4 values, as before
    plain_prm = plain.nonbonded_14_params["params"].numpy()[plain.nonbonded_14_params["map"].numpy()[:, 1]]
    f2 = 2.0 * f6
    assert tuple(plain_prm[0, :2]) == ab(0.5 * (1.80 * f2 + 1.90 * f2), math.sqrt(0.05 * 0.20))


def test_get_AB_overrides_only_the_nbfix_pairs(tmp_path):
    from torchmd_b200.ff_yaml import yaml_parameters

    mol, ff = five_atoms(tmp_path)
    for prec in (torch.float32, torch.float64):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            plain = yaml_parameters(mol, ff, terms=TERMS, precision=prec)
            par = yaml_parameters(mol, ff, terms=TERMS + ["nbfix"], precision=prec)
        (A0, B0), (A1, B1) = plain.get_AB(), par.get_AB()
        assert A1.dtype == prec and torch.equal(A1, A1.T) and torch.equal(B1, B1.T)
        fixed = torch.zeros_like(A0, dtype=torch.bool)
        fixed[0, 2] = fixed[2, 0] = fixed[0, 3] = fixed[3, 0] = True
        assert torch.equal(A0[~fixed], A1[~fixed]) and torch.equal(B0[~fixed], B1[~fixed])  # bit-identical elsewhere
        assert not (A0[fixed] == A1[fixed]).any()
        s, e = par.nbfix_params["params"][0]
        assert A1[0, 2] == e * 4 * s**6 * s**6 and B1[2, 0] == e * 4 * s**6


def test_urey_bradley_terms_from_the_prm(tmp_path):
    from torchmd_b200.ff_yaml import YamlForceField, yaml_parameters

    mol, ff = five_atoms(tmp_path)
    with pytest.warns(UserWarning, match="1 angles with a Urey-Bradley term"):
        plain = yaml_parameters(mol, ff, terms=TERMS, precision=torch.float64)
    assert plain.ub_params is None
    par = yaml_parameters(mol, ff, terms=TERMS + ["ureybradley"], precision=torch.float64)
    ub = par.ub_params  # BB-BB-EE has k_ub = 0: no term
    assert ub["idx"].tolist() == [[0, 1, 2]] and ub["params"].tolist() == [[20.0, 2.5]]
    with pytest.raises(RuntimeError, match="ureybradley"):
        yaml_parameters(mol, YamlForceField({"lj": {}}), terms=["bonds", "ureybradley"])


def test_builders_without_the_new_terms_are_unchanged(reference_inputs):
    """3ions, waterbox and sodiumperiodic: the default terms give no Urey-Bradley or NBFIX entry and the same A/B."""
    import glob

    from torchmd_b200 import charmm
    from torchmd_b200.ff_yaml import yaml_parameters
    from torchmd_b200.parameters import lorentz_berthelot_AB

    for name in ("3ions", "waterbox", "sodiumperiodic"):
        folder = os.path.join(reference_inputs, "data", name)
        psf, pdb, prm = (glob.glob(os.path.join(folder, e))[0] for e in ("*.psf", "*.pdb", "*.prm"))
        mol = charmm.load_molecule(psf, pdb)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            par = yaml_parameters(mol, charmm.CharmmPrmForceField(prm, mol), precision=torch.float64)
        assert par.ub_params is None and par.nbfix_params is None
        p = par.nonbonded_params["params"]
        for a, b in zip(par.get_AB(), lorentz_berthelot_AB(p[:, 0], p[:, 1])):
            assert torch.equal(a, b)


def test_amber_nbfix_tables_equal_lorentz_berthelot(reference_inputs):
    from torchmd_b200 import amber

    s = amber.AmberSystem(os.path.join(reference_inputs, *ALA2))
    terms = ("bonds", "angles", "dihedrals", "impropers", "1-4", "lj")
    A0, B0 = amber.amber_parameters(s, terms, precision=torch.float64).get_AB()
    A1, B1 = amber.amber_parameters(s, terms + ("nbfix",), precision=torch.float64).get_AB()
    # the file holds its coefficients to 9 significant digits: the tables agree to fp32 rounding
    np.testing.assert_allclose(A1.numpy(), A0.numpy(), rtol=2.0**-23, atol=0)
    np.testing.assert_allclose(B1.numpy(), B0.numpy(), rtol=2.0**-23, atol=0)


def edited_prmtop(src, dst, ia, ib, scale):
    """Copy of a prmtop with the ACOEF/BCOEF entry of type indices (ia, ib) (0-based) multiplied by ``scale``."""
    from torchmd_b200 import amber

    p = amber.read_prmtop(src)
    nt = p["POINTERS"][1]
    e = p["NONBONDED_PARM_INDEX"][nt * ia + ib] - 1
    lines = open(src).read().split("\n")
    out, flag, k = [], None, 0
    for ln in lines:
        if ln.startswith("%FLAG"):
            flag, k = ln.split()[1], 0
        elif flag in ("LENNARD_JONES_ACOEF", "LENNARD_JONES_BCOEF") and not ln.startswith("%"):
            vals = [ln[i : i + 16] for i in range(0, len(ln), 16)]
            for j, v in enumerate(vals):
                if k + j == e:
                    vals[j] = f"{float(v) * scale:16.8E}"
            k += len(vals)
            ln = "".join(vals)
        out.append(ln)
    open(dst, "w").write("\n".join(out))


def test_amber_nbfix_keeps_an_edited_pair(reference_inputs, tmp_path):
    from torchmd_b200 import amber

    src = os.path.join(reference_inputs, *ALA2)
    s0 = amber.AmberSystem(src)
    nb = s0._nb[0]
    names = list(np.unique(s0.atomtype))
    ta, tb = "C", "O"  # one off-diagonal pair of types that no other name shares (CT and CX share one LJ type)
    ia, ib = int(nb[list(s0.atomtype).index(ta)]), int(nb[list(s0.atomtype).index(tb)])
    dst = str(tmp_path / "edited.prmtop")
    edited_prmtop(src, dst, ia, ib, 1.5)
    terms = ("lj", "nbfix")
    A0, B0 = amber.amber_parameters(s0, terms, precision=torch.float64).get_AB()
    A1, B1 = amber.amber_parameters(amber.AmberSystem(dst), terms, precision=torch.float64).get_AB()
    changed = ((A0 != A1) | (B0 != B1)).numpy()
    a, b = names.index(ta), names.index(tb)
    expect = np.zeros_like(changed)
    expect[a, b] = expect[b, a] = True
    assert np.array_equal(changed, expect)
    assert abs(float(A1[a, b] / A0[a, b]) - 1.5) < 1e-7 and abs(float(B1[a, b] / B0[a, b]) - 1.5) < 1e-7
    # without "nbfix" the edit is invisible: Lorentz-Berthelot of the diagonal
    L0 = amber.amber_parameters(s0, ("lj",), precision=torch.float64).get_AB()
    L1 = amber.amber_parameters(amber.AmberSystem(dst), ("lj",), precision=torch.float64).get_AB()
    assert all(torch.equal(x, y) for x, y in zip(L0, L1))


def test_amber_chamber_urey_bradley(reference_inputs, tmp_path):
    """The ala2 prmtop with chamber Urey-Bradley sections appended: two terms on the ends of two of its angles."""
    from torchmd_b200 import amber

    src = os.path.join(reference_inputs, *ALA2)
    s0 = amber.AmberSystem(src)
    a1, a2 = s0.angles[0], s0.angles[5]
    extra = ["%FLAG CHARMM_UREY_BRADLEY_COUNT", "%FORMAT(2I8)", f"{2:8d}{2:8d}",
             "%FLAG CHARMM_UREY_BRADLEY", "%FORMAT(10I8)",
             "".join(f"{v:8d}" for v in (a1[2] + 1, a1[0] + 1, 2, a2[0] + 1, a2[2] + 1, 1)),
             "%FLAG CHARMM_UREY_BRADLEY_FORCE_CONSTANT", "%FORMAT(5E16.8)", f"{10.0:16.8E}{20.0:16.8E}",
             "%FLAG CHARMM_UREY_BRADLEY_EQUIL_VALUE", "%FORMAT(5E16.8)", f"{2.1:16.8E}{2.4:16.8E}"]
    dst = tmp_path / "ub.prmtop"
    dst.write_text(open(src).read().rstrip("\n") + "\n" + "\n".join(extra) + "\n")
    s = amber.AmberSystem(str(dst))
    with pytest.warns(UserWarning, match="2 Urey-Bradley terms"):
        assert amber.amber_parameters(s).ub_params is None
    par = amber.amber_parameters(s, ("bonds", "angles", "ureybradley"), precision=torch.float64)
    ub = par.ub_params
    rows = ub["params"].numpy()[ub["map"].numpy()[:, 1]]
    ends = {tuple(sorted((int(i[0]), int(i[2])))): tuple(r) for i, r in zip(ub["idx"].numpy(), rows)}
    assert ends == {tuple(sorted((int(a1[0]), int(a1[2])))): (20.0, 2.4), tuple(sorted((int(a2[0]), int(a2[2])))): (10.0, 2.1)}
    for i in ub["idx"].numpy():  # whole angles of the topology, first index below last
        assert i[0] < i[2] and any((i == a).all() or (i == a[::-1]).all() for a in s.angles)


def test_oracle_forces_are_the_energy_gradient():
    rng = np.random.default_rng(3)
    pos = rng.normal(scale=2.0, size=(6, 3))
    idx = np.array([[0, 2], [1, 3], [4, 5], [0, 5]])
    k, s0 = np.array([10.0, 20.0, 5.0, 1.0]), np.array([2.0, 2.5, 1.0, 3.0])
    box = np.array([5.0, 6.0, 7.0])
    for b in (None, box):
        _, F = oub.energy_forces(pos, idx, k, s0, box=b)
        h = 1e-6
        for a in range(6):
            for d in range(3):
                p, m = pos.copy(), pos.copy()
                p[a, d] += h
                m[a, d] -= h
                g = (oub.energy_forces(p, idx, k, s0, box=b)[0] - oub.energy_forces(m, idx, k, s0, box=b)[0]) / (2 * h)
                assert abs(F[a, d] + g) < 1e-6 * max(1.0, abs(g))
    assert abs(F.sum(0)).max() < 1e-12

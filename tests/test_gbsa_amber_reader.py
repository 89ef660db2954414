"""The Generalized Born sections of AMBER prmtop files (RADII, SCREEN, RADIUS_SET) through torchmd_b200/amber.py:
the alanine-dipeptide prmtop of reference_inputs.npz against the mbondi radii and Hawkins screens its atom types
take, the committed fixture tests/golden/gb_radii.npz against the reader, and the error when the sections are
missing."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden


@pytest.fixture
def ALA(reference_inputs):
    return os.path.join(reference_inputs, "data", "prod_alanine_dipeptide_amber", "structure.prmtop")


def test_alanine_dipeptide_radii_and_screens(ALA):
    from torchmd_b200 import amber

    s = amber.AmberSystem(ALA)
    assert s.natoms == 688 and len(s.gb_radius) == 688 and len(s.gb_screen) == 688
    assert s.radius_set == "modified Bondi radii (mbondi)"
    # mbondi: water H 0.8, other H 1.2 (1.3 on N, and here on C), C 1.7, N 1.55, O 1.5; screens H 0.85, C 0.72,
    # N 0.79, O 0.85
    want_r = {"HW": 0.8, "OW": 1.5, "HC": 1.3, "H1": 1.3, "H": 1.3, "C": 1.7, "CT": 1.7, "CX": 1.7, "N": 1.55, "O": 1.5}
    want_s = {"HW": 0.85, "OW": 0.85, "HC": 0.85, "H1": 0.85, "H": 0.85, "C": 0.72, "CT": 0.72, "CX": 0.72, "N": 0.79, "O": 0.85}
    for t in np.unique(s.atomtype):
        sel = s.atomtype == t
        assert np.all(s.gb_radius[sel] == want_r[t]), t
        assert np.all(s.gb_screen[sel] == want_s[t]), t
    assert (s.atomtype == "HW").sum() == 444 and (s.atomtype == "OW").sum() == 222
    par = amber.amber_parameters(s, terms=["bonds", "gb"], precision=torch.float32)
    assert par.gb_params["radius"].dtype == torch.float64
    assert np.array_equal(par.gb_params["radius"].numpy(), s.gb_radius)
    assert np.array_equal(par.gb_params["screen"].numpy(), s.gb_screen)
    assert amber.amber_parameters(s, terms=["bonds"]).gb_params is None


def test_fixture_matches_the_reader(tmp_path):
    """gb_radii.npz holds what read_prmtop gives for the three systems; their charges and atom counts agree with the
    *_nocut / *_nobox fixtures that hold the rest of each system."""
    gb = load_golden("gb_radii")
    for name, fixture in (("thrombin", "thrombin_nobox_rf"), ("ligand", "ligand_amber_nocut"), ("benzamidine", "benzamidine_amber_nocut")):
        g = load_golden(fixture)
        r, s = gb[name + "_radii"], gb[name + "_screen"]
        assert len(r) == len(s) == len(g["par_charges"])
        assert np.all(r > 0.09) and np.all(s > 0) and np.all(np.isfinite(r)) and np.all(np.isfinite(s))
        assert len(str(gb[name + "_prmtop_sha256"])) == 64
    assert str(gb["thrombin_radius_set"]) == "H(N)-modified Bondi radii (mbondi2)"
    assert str(gb["ligand_radius_set"]) == "H(N)-modified Bondi radii (mbondi2)"
    # a prmtop written with the fixture's sections reads back to the same arrays
    from torchmd_b200 import amber

    def section(flag, vals):
        lines = [f"%FLAG {flag}", "%FORMAT(5E16.8)"]
        for k in range(0, len(vals), 5):
            lines.append("".join(f"{v:16.8E}" for v in vals[k:k + 5]))
        return lines

    r, s = gb["benzamidine_radii"], gb["benzamidine_screen"]
    text = ["%FLAG RADIUS_SET", "%FORMAT(1a80)", str(gb["benzamidine_radius_set"])] + section("RADII", r) + section("SCREEN", s)
    path = tmp_path / "gb.prmtop"
    path.write_text("\n".join(text) + "\n")
    p = amber.read_prmtop(str(path))
    assert np.array_equal(np.array(p["RADII"]), r) and np.array_equal(np.array(p["SCREEN"]), s)


def test_missing_sections_raise(ALA, tmp_path):
    from torchmd_b200 import amber

    text = open(ALA).read()
    start = text.index("%FLAG RADII")
    end = text.index("%FLAG", text.index("%FLAG SCREEN") + 1)
    path = tmp_path / "nogb.prmtop"
    path.write_text(text[:start] + text[end:])
    s = amber.AmberSystem(str(path))
    assert s.gb_radius is None and s.gb_screen is None
    amber.amber_parameters(s, terms=["bonds"])  # fine without "gb"
    with pytest.raises(ValueError, match="RADII"):
        amber.amber_parameters(s, terms=["bonds", "gb"])

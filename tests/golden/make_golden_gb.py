"""Generalized Born inputs of the three AMBER systems without a box: the RADII, SCREEN and RADIUS_SET sections of the
reference's tests/data/{thrombin-ligand-amber, ligand-amber, benzamidine-amber}/structure.prmtop, read by
torchmd_b200/amber.py (read_prmtop), and the sha256 of each prmtop.  The rest of each system (parameters, coordinates)
is in thrombin_nobox_rf.npz, ligand_amber_nocut.npz and benzamidine_amber_nocut.npz.  Data only.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_gb.py
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)

from torchmd_b200 import amber  # noqa: E402

CASES = {"thrombin": "thrombin-ligand-amber", "ligand": "ligand-amber", "benzamidine": "benzamidine-amber"}


def main():
    out = {}
    for name, folder in CASES.items():
        path = os.path.join(REF, "tests", "data", folder, "structure.prmtop")
        p = amber.read_prmtop(path)
        out[f"{name}_radii"] = np.array(p["RADII"], np.float64)
        out[f"{name}_screen"] = np.array(p["SCREEN"], np.float64)
        out[f"{name}_radius_set"] = np.array(" ".join(p["RADIUS_SET"]).strip())
        out[f"{name}_prmtop_sha256"] = np.array(hashlib.sha256(open(path, "rb").read()).hexdigest())
        print(name, len(out[f"{name}_radii"]), out[f"{name}_radius_set"])
    np.savez_compressed(os.path.join(HERE, "gb_radii.npz"), **out)


if __name__ == "__main__":
    main()

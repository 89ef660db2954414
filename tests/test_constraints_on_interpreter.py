"""The constraint GPU tests (test_gpu_constraints) on the CPU, through the host SIMT-interpreter build of the library
(tests/simt) with CPU tensors, at sizes the interpreter runs in seconds; plus the topology checks of
torchmd_b200.constraints, which need no device at all."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_mirrors_on_interpreter import _install


@pytest.fixture(params=["", "_cl"])
def hostsim_con(monkeypatch, request):
    handle = _install(monkeypatch, request.param)
    import test_gpu_constraints

    monkeypatch.setattr(test_gpu_constraints, "DEV", "cpu")
    return handle


# ---- topology ------------------------------------------------------------------------------------------------------
def _bonds_of(par):
    return par.bond_params["idx"].cpu().numpy()


@pytest.mark.parametrize("hh", [False, True])
def test_water_box_topology(hh):
    from torchmd_b200 import Constraints, testsystems

    sysd = testsystems.water_box(50, hh_bonds=hh)
    par = testsystems.water_parameters(sysd, precision=torch.float64)
    for kind in ("water", "hbonds"):
        c = Constraints(par, kind)
        assert c.nwaters == 50 and c.nclusters == 0
        np.testing.assert_allclose(c.water_d[:, 0], testsystems.WATER_BOND[1])
        dhh = testsystems.WATER_HH_BOND[1] if hh else 2 * testsystems.WATER_BOND[1] * np.sin(testsystems.WATER_ANGLE[1] / 2)
        np.testing.assert_allclose(c.water_d[:, 1], dhh, rtol=1e-12)
        assert c.ndof() == 3 * 150 - 150


@pytest.mark.parametrize("name", ["ala2_xsc_rf", "thrombin_nobox_rf"])
def test_hbond_clusters_match_the_bonds(name):
    from torchmd_b200 import Constraints, testsystems

    par = testsystems.golden_system(name, precision=torch.float64)[0]
    m = par.masses.numpy().reshape(-1)
    bonds = _bonds_of(par)
    h = m < 4.5
    c = Constraints(par, "hbonds")
    in_water = np.zeros(len(m), bool)
    in_water[c.water_idx.reshape(-1)] = True
    xh = [(int(i), int(j)) for i, j in bonds if (h[i] != h[j]) and not (in_water[i] or in_water[j])]
    assert len(c.cluster_d) == len(xh)
    heavy = {j if h[i] else i for i, j in xh}
    assert c.nclusters == len(heavy)
    sizes = np.diff(c.cluster_ptr) - 1
    for x in heavy:
        assert sizes[list(c.cluster_idx[c.cluster_ptr[:-1]]).index(x)] == sum(1 for i, j in xh if x in (i, j))
    assert c.ndof() == 3 * len(m) - 3 * c.nwaters - len(xh)
    assert Constraints(par, "water").nclusters == 0


def _par(masses, bonds, bond_params=((100.0, 1.0),), angles=None):
    from torchmd_b200 import TopologyParameters

    n = len(masses)
    b = np.asarray(bonds, np.int64).reshape(-1, 2)
    return TopologyParameters(atom_types=np.zeros(n, np.int64), type_sigma=[1.0], type_epsilon=[0.1], charges=np.zeros(n),
                              masses=masses, bonds=(b, np.stack([np.arange(len(b)), np.zeros(len(b), np.int64)], 1), list(bond_params)),
                              angles=angles, precision=torch.float64)


def test_refusals():
    from torchmd_b200 import Constraints

    with pytest.raises(ValueError, match="hydrogen 1 is bonded to 2"):
        Constraints(_par([12.0, 1.0, 12.0], [(0, 1), (1, 2)]), "hbonds")
    with pytest.raises(ValueError, match="H-H bond 1-2 outside a water"):
        Constraints(_par([12.0, 1.0, 1.0, 12.0], [(0, 1), (1, 2), (0, 3)]), "hbonds")
    with pytest.raises(ValueError, match="hydrogen masses differ"):
        Constraints(_par([16.0, 1.0, 2.0], [(0, 1), (0, 2)]), "water")
    with pytest.raises(ValueError, match="H-O-H angle has no parameters"):
        Constraints(_par([16.0, 1.0, 1.0], [(0, 1), (0, 2)]), "water")
    p = _par([12.0, 1.0, 12.0], [(0, 1), (0, 2)])
    p.bond_params["map"] = p.bond_params["map"][1:]  # the C-H bond loses its parameter row
    with pytest.raises(ValueError, match="bond 0-1 has no parameters"):
        Constraints(p, "hbonds")
    with pytest.raises(ValueError, match="spans batch groups"):
        Constraints(_par([12.0, 1.0], [(0, 1)]), "hbonds", batch=torch.tensor([0, 1]))
    with pytest.raises(ValueError, match="massless atom"):
        Constraints(_par([0.0, 1.0], [(0, 1)]), "hbonds")
    # kind="water" constrains no other hydrogen and refuses nothing about them
    assert Constraints(_par([12.0, 1.0, 12.0], [(0, 1), (1, 2)]), "water").nwaters == 0


def test_ndof_with_batch():
    from torchmd_b200 import Constraints, testsystems

    sysd = testsystems.water_box(4)
    par = testsystems.water_parameters(sysd, precision=torch.float64)
    batch = torch.tensor([0] * 3 + [1] * 9)
    c = Constraints(par, "water", batch=batch)
    np.testing.assert_array_equal(c.ndof(), [9 - 3, 27 - 9])
    assert Constraints(par, "water").ndof() == 36 - 12


def test_hydrogen_mass_repartitioning_counts_as_hydrogen():
    from torchmd_b200 import Constraints

    c = Constraints(_par([9.0, 3.0, 3.0, 3.0], [(0, 1), (0, 2), (0, 3)]), "hbonds")
    assert c.nclusters == 1 and list(c.cluster_idx) == [0, 1, 2, 3]


# ---- kernels on the interpreter ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_residuals(hostsim_con, dtype):
    import test_gpu_constraints as G

    G.test_residuals_every_step(dtype, nw=60, nsteps=5)


@pytest.mark.parametrize("name,kind,nrep", [("water60", "water", 1), ("water60", "water", 2), ("ala2_xsc_rf", "hbonds", 1),
                                            ("ala2_nobox_rf_rot", "hbonds", 1)])
def test_trajectories_f64(hostsim_con, name, kind, nrep):
    import test_gpu_constraints as G

    dp, dv, _, _ = G._trajectory_case(torch.float64, name, kind, 20, nrep)
    assert dp < 1e-9 and dv < 1e-9, (dp, dv)


@pytest.mark.parametrize("name,kind", [("water60", "water"), ("ala2_xsc_rf", "hbonds")])
def test_trajectories_f32(hostsim_con, name, kind):
    import test_gpu_constraints as G

    dp, dv, _, _ = G._trajectory_case(torch.float32, name, kind, 4)
    assert dp < 2e-5 and dv < 5e-5, (dp, dv)


def test_thrombin_hbonds(hostsim_con):
    import test_gpu_constraints as G

    dp, dv, _, _ = G._trajectory_case(torch.float64, "thrombin_nobox_rf", "hbonds", 2)
    assert dp < 1e-9 and dv < 1e-9, (dp, dv)


@pytest.mark.parametrize("name,kind", [("water60", "water"), ("ala2_xsc_rf", "hbonds")])
def test_captured_step_f32(hostsim_con, name, kind):
    import test_gpu_constraints as G

    dp, dv, _, _ = G._trajectory_case(torch.float32, name, kind, 4, thermostat=False)
    assert dp < 2e-5 and dv < 5e-5, (dp, dv)


def test_stepwise_path_and_shared_forces(hostsim_con):
    import test_gpu_constraints as G

    G.test_stepwise_path_matches_md_steps()
    G.test_integrators_sharing_one_forces()


def test_under_a_random_thread_order():
    """The kernel checks again with the interpreter's threads in a random order (SIMT_SCHEDULE is read once per process)."""
    env = dict(os.environ, SIMT_SCHEDULE="random:11")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", __file__, "-k",
                        "residuals or (trajectories and water60) or captured"],
                       cwd=os.path.dirname(os.path.abspath(__file__)), env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_decomposed_runs_refuse_constraints(hostsim_con):
    import ctypes as C

    import test_gpu_constraints as G
    from torchmd_b200 import _lib
    from torchmd_b200.domain import DecomposedIntegrator

    sysd, par, system, forces, con = G._water(20, torch.float32)
    with pytest.raises(NotImplementedError):
        DecomposedIntegrator(system, forces, 2.0, "cpu", constraints=con)
    ctx = forces._ensure_ctx(system.pos)
    con.upload(ctx)
    assert _lib.lib().tmd_set_owned_atoms(ctx, 0, 10) == -5
    assert _lib.lib().tmd_dd_create(ctx, 0, 1, (C.c_ubyte * 64)()) == -5

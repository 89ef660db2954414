"""test_gpu_cluster_systems' functions on the host SIMT-interpreter build with the cluster path on (tests/simt, tag
"_cl"): the solvated protein with RF and PME, 17 to 128 atom types, and the decision to take the full rows when the
cluster lists would not fit k_cpair's shared-memory staging."""
import numpy as np
import pytest
import torch

from test_mirrors_on_interpreter import _install


@pytest.fixture
def hostsim(monkeypatch):
    handle = _install(monkeypatch, "_cl")
    monkeypatch.setenv("TMD_B200_FX", "2")  # the full rows on k_pair_fx2, as on the GPU
    import test_gpu_cluster_systems

    monkeypatch.setattr(test_gpu_cluster_systems, "DEV", "cpu")
    return handle


def test_solvated_protein_rf(hostsim):
    import test_gpu_cluster_systems as G

    G.protein_rf("two_replicas")


def test_solvated_protein_pme(hostsim):
    import test_gpu_cluster_systems as G

    G.protein_pme("atoms_thrown")


@pytest.mark.parametrize("T", [17, 65, 128])
def test_atom_types_on_the_cluster_kernel(hostsim, T):
    """Types 65-128 fill the per-warp LJ table past 64 types; type 127 is the top of the 7-bit type field."""
    import test_gpu_cluster_systems as G

    spec = G.retyped(G.tiled_water(2), T, seed=T)
    forces, pos, box, F, E, kern = G.run(spec)
    assert kern == G.CLUSTER, kern
    G.check_fp32(spec, forces, pos, box, F, E, f"{T} types", tol=G.RETYPED_TOL)


def test_129_types_are_refused(hostsim):
    import test_gpu_cluster_systems as G
    from torchmd_b200 import _lib

    with pytest.raises(_lib.TmdError, match="128 atom types"):
        G.run(G.retyped(G.tiled_water(1), 129))


def test_dilute_gas_at_a_long_cutoff_takes_the_full_rows(hostsim):
    """3,000 argon atoms in a 240 A box at cutoff 16: the capacity estimate assumes liquid density (capped at N
    entries), which needs more than 180 KB of staging -- the full rows, with the oracle's results."""
    import test_gpu_cluster_systems as G
    from torchmd_b200 import testsystems

    sysd = testsystems.argon_box(3000, seed=0)
    par = testsystems.argon_parameters(sysd, precision=torch.float64)
    spec = G._spec_of(par, sysd["coords"], sysd["box"], ["lj"], dict(cutoff=16.0, switch_dist=14.0), sysd["name"])
    forces, pos, box, F, E, kern = G.run(spec)
    assert kern == G.FULL_ROWS, kern
    G.check_fp32(spec, forces, pos, box, F, E, "argon gas at cutoff 16")

"""test_gpu_force_convention's functions on the host SIMT-interpreter build of the kernels (tests/simt; tag "_cl" for
the cluster lists): both convention orders on the cluster kernels, the autograd surfaces after an explicit compute,
and forces as the central differences of the kernels' own energies."""
import pytest
import torch

from test_mirrors_on_interpreter import _install


def _hostsim(monkeypatch, tag):
    handle = _install(monkeypatch, tag)
    import test_gpu_cluster_systems
    import test_gpu_cmap
    import test_gpu_force_convention
    import test_gpu_ub_nbfix

    for mod in (test_gpu_cluster_systems, test_gpu_cmap, test_gpu_force_convention, test_gpu_ub_nbfix):
        monkeypatch.setattr(mod, "DEV", "cpu")
    return handle


@pytest.fixture
def hostsim(monkeypatch):
    return _hostsim(monkeypatch, "")


@pytest.fixture
def hostsim_cl(monkeypatch):
    return _hostsim(monkeypatch, "_cl")


@pytest.mark.parametrize("case", ["k4_water", "k10_water", "k4_open"])
def test_both_convention_orders_on_the_cluster_kernels(hostsim_cl, monkeypatch, case):
    import test_gpu_force_convention as FC

    FC.convention_orders(case, monkeypatch)


@pytest.mark.parametrize("case", ["k0_open", "k0_box_plain", "k2", "k3", "k5", "k8", "k9"])
def test_both_convention_orders_on_the_full_rows(hostsim, monkeypatch, case):
    import test_gpu_force_convention as FC

    FC.convention_orders(case, monkeypatch)


def test_autograd_surfaces_after_explicit_forces_on_the_cluster_kernel(hostsim_cl, monkeypatch):
    import test_gpu_force_convention as FC

    FC.autograd_surfaces_after_explicit(FC.water(2), monkeypatch, nsteps=3)


@pytest.mark.parametrize("terms", [["angles"], ["dihedrals"], ["bonds", "angles", "dihedrals", "impropers", "1-4", "lj", "electrostatics"]])
def test_forces_are_the_gradient_ala2(hostsim, terms):
    import test_gpu_force_convention as FC

    FC.ala2_gradient(terms, nsample=8)


def test_forces_are_the_gradient_pme(hostsim):
    import test_gpu_force_convention as FC

    FC.ala2_gradient(["electrostatics", "lj"], pme=True, nsample=8)


def test_forces_are_the_gradient_nbfix_and_repulsion(hostsim, tmp_path):
    import test_gpu_force_convention as FC
    import test_gpu_ub_nbfix as UB

    FC.nbfix_gradient(UB.reference_inputs_dir(tmp_path), ["lj", "electrostatics"], nsample=8)
    FC.repulsion_gradient(["lj", "repulsion", "repulsioncg"], nsample=8)


def test_forces_are_the_gradient_fp32_cluster_kernel(hostsim_cl):
    import test_gpu_force_convention as FC

    FC.cluster_gradient_fp32(nsample=4)

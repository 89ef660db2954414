"""Generalized Born implicit solvent on the CPU, through the host SIMT-interpreter build of the library (tests/simt):
the GPU tests of test_gpu_gbsa with CPU tensors on the ligand and benzamidine, in both precisions and with 2 replicas,
on the plain build (stream path) and on the build with every opt-in path as the default (the captured step, the
radii and energy passes and the bonded kernel on their own streams)."""
import pytest
import torch

from test_mirrors_on_interpreter import _install


@pytest.fixture(params=["", "_r2"])
def hostsim_gb(monkeypatch, request):
    handle = _install(monkeypatch, request.param)
    import test_gpu_gbsa

    monkeypatch.setattr(test_gpu_gbsa, "DEV", "cpu")
    return handle


@pytest.mark.parametrize("sigma", [0.0, 0.0054])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("name", ["ligand", "benzamidine"])
def test_against_the_oracle(hostsim_gb, name, dtype, sigma):
    import test_gpu_gbsa as G

    G.test_against_the_oracle(name, dtype, sigma)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_reproducibility_autograd_and_steps(hostsim_gb, dtype):
    import test_gpu_gbsa as G

    G.test_gb_forces_are_bitwise_reproducible(dtype, name="ligand")
    G.test_autograd_and_vmap(dtype, name="benzamidine")
    for constraints in (None, "hbonds"):
        G.test_native_steps_report_a_fresh_energy(dtype, constraints, name="ligand", nsteps=3)
    G.test_replica_exchange_exchanges_on_the_gb_energy(dtype, name="benzamidine")


def test_minimizer_plugin_and_refusals(hostsim_gb):
    import test_gpu_gbsa as G

    G.test_minimizer_and_external_plugin(name="benzamidine")
    G.test_refusals()

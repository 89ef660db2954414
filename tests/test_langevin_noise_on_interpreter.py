"""test_gpu_langevin_noise's draw checks on the host SIMT-interpreter build with the product's defaults compiled in
(tests/simt, tag "_cl": captured step graphs, fused prepare and step boundary, overlapped bonded kernel, cluster lists).

The interpreter compiles the unmodified kernels against the host libm, whose logf / sincosf / cosf are within an ulp,
so the draws must agree with oracle/philox.py to an ulp of max(1, |xi|) here rather than to the device bound."""
import numpy as np
import pytest
import torch

from test_mirrors_on_interpreter import _install

F32, F64 = torch.float32, torch.float64


@pytest.fixture
def hostsim(monkeypatch):
    handle = _install(monkeypatch, "_cl")
    monkeypatch.setenv("TMD_B200_FX", "2")  # the full rows on k_pair_fx2, as on the GPU
    import test_gpu_langevin_noise
    import test_gpu_step_recovery

    monkeypatch.setattr(test_gpu_langevin_noise, "DEV", "cpu")
    monkeypatch.setattr(test_gpu_step_recovery, "DEV", "cpu")
    monkeypatch.setattr(test_gpu_langevin_noise, "XI_BOUND", {np.float32: 2.0**-23, np.float64: 2.0**-52})
    return handle


PATHS = ["cluster_fused_7", "cluster_fusestep0", "cluster_overlap0", "cluster_graph0", "full_rows", "no_bonded", "stepwise",
         "single_steps", "split_3_4", "fp64", "fp64_stepwise"]


@pytest.mark.parametrize("name", PATHS)
def test_draws_on_every_path(hostsim, monkeypatch, name):
    import test_gpu_langevin_noise as G

    G.test_draws_on_every_path(monkeypatch, name)


@pytest.mark.parametrize("seed", [2**32 - 1, 2**32], ids=["2^32-1", "2^32"])
def test_draws_at_edge_seeds(hostsim, monkeypatch, seed):
    import test_gpu_langevin_noise as G

    G.test_draws_at_edge_seeds(monkeypatch, "cluster_fused_7", seed)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_step_word_carries_into_the_high_counter_word(hostsim, dtype):
    import test_gpu_langevin_noise as G

    G.test_step_word_carries_into_the_high_counter_word(dtype)


def test_recovered_call_draws_the_noise_of_its_steps(hostsim, monkeypatch):
    import test_gpu_langevin_noise as G

    G.test_recovered_call_draws_the_noise_of_its_steps(monkeypatch)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_barostat_chunks_keep_the_philox_position(hostsim, monkeypatch, dtype):
    import test_gpu_langevin_noise as G

    G.test_barostat_chunks_keep_the_philox_position(monkeypatch, dtype)

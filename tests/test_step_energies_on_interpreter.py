"""test_gpu_step_energies on the host SIMT-interpreter build with the product's defaults compiled in (tests/simt, tag
"_cl": captured step graphs, fused prepare and step boundary, overlapped bonded kernel, cluster lists): the energies a
call reports against a fresh evaluation on the full rows, the stream path, the stepwise path, fp64 and the velocity
constraint, the Monte Carlo move, and tmd_md_steps_host.  The systems are the small ones (the 688-atom alanine
dipeptide, 300 waters): the 8k-atom water box of the GPU cases is left to the GPU."""
import numpy as np
import pytest
import torch

from test_mirrors_on_interpreter import _install

F32, F64 = torch.float32, torch.float64


@pytest.fixture
def hostsim(monkeypatch):
    handle = _install(monkeypatch, "_cl")
    monkeypatch.setenv("TMD_B200_FX", "2")  # the full rows on k_pair_fx2, as on the GPU
    import test_gpu_cmap
    import test_gpu_step_energies

    monkeypatch.setattr(test_gpu_step_energies, "DEV", "cpu")
    monkeypatch.setattr(test_gpu_cmap, "DEV", "cpu")
    return handle


# (environment, system, precision, calls, stepwise): the full rows, the stream path, the same-stream bonded kernel,
# the stepwise path, fp64, fixed X-H bonds in fp32 and fp64 with CMAP
CASES = {
    "full_rows": ({}, "ala2", F32, (3, 3, 3), False),
    "graph0": ({"TMD_B200_GRAPH": "0"}, "ala2", F32, (3, 2, 3), False),
    "overlap0": ({"TMD_B200_OVERLAP": "0"}, "ala2_cmap", F32, (3, 3, 3), False),
    "stepwise": ({}, "ala2", F32, (2, 2, 2), True),
    "fp64": ({}, "ala2_cmap", F64, (3, 1, 3), False),
    "hbonds": ({}, "ala2_hbonds", F32, (3, 3, 3), False),
    "hbonds_fp64": ({}, "ala2_hbonds", F64, (3, 3, 3), False),
}


@pytest.mark.parametrize("name", list(CASES))
def test_energies_on_the_host_paths(hostsim, monkeypatch, name):
    import test_gpu_step_energies as G

    env, sysname, dtype, calls, stepwise = CASES[name]
    monkeypatch.setitem(G.PATHS, name, (env, sysname, dtype, calls, stepwise, False, None, None))
    G.energy_case(monkeypatch, name)


def test_a_one_step_shift_is_detected(hostsim, monkeypatch):
    import test_gpu_step_energies as G

    monkeypatch.setitem(G.PATHS, "full_rows", ({}, "ala2", F32, (2, 3), False, False, None, None))
    G.test_a_one_step_shift_is_detected(monkeypatch, "full_rows")


@pytest.mark.parametrize("kind", [None, "water"], ids=["flexible", "rigid"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32", "fp64"])
def test_barostat_energies_describe_the_final_state(hostsim, dtype, kind):
    import test_gpu_step_energies as G

    G.barostat_case(dtype, kind)


def test_md_steps_host_matches_md_steps(hostsim, monkeypatch):
    import test_gpu_step_energies as G

    monkeypatch.setattr(G, "water8k", lambda dtype: G.ala2(dtype))
    G.test_md_steps_host_matches_md_steps(monkeypatch)


def test_batch_groups(hostsim, monkeypatch):
    import test_gpu_step_energies as G

    monkeypatch.setattr(G, "water8k", lambda dtype, nrep=2: G.ala2(dtype, nrep=nrep))
    G.test_batch_groups(monkeypatch)

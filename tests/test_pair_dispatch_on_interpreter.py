"""test_gpu_pair_dispatch's cases on the host SIMT-interpreter build of the kernels (tests/simt): the tmd_pair_kernel id of
every call, on every row of the pair-kernel choice, in both conventions, with and without energies."""
import pytest

import test_gpu_pair_dispatch as D
from test_force_convention_on_interpreter import _hostsim


@pytest.fixture
def hostsim(monkeypatch):
    return _hostsim(monkeypatch, "")


@pytest.mark.parametrize("case", list(D.CASES))
def test_pair_kernel_of_every_call(hostsim, monkeypatch, case):
    ids, _, _ = D.run_calls(case, monkeypatch)
    assert ids == D.expected(case)[0], (case, ids)

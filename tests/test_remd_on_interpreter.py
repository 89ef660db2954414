"""Replica exchange on the host SIMT-interpreter build of the kernels (tests/simt): k_remd_exchange and k_remd_scale
against oracle/remd.py through the C entry points, the ladder row of the Langevin kernels, and the small cases of
test_gpu_replica_exchange."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import remd
from test_mirrors_on_interpreter import _install

F32, F64 = torch.float32, torch.float64


@pytest.fixture
def hostsim(monkeypatch):
    handle = _install(monkeypatch, "_cl")
    monkeypatch.setenv("TMD_B200_FX", "2")
    import test_gpu_langevin_noise
    import test_gpu_replica_exchange
    import test_gpu_step_recovery

    for mod in (test_gpu_langevin_noise, test_gpu_replica_exchange, test_gpu_step_recovery):
        monkeypatch.setattr(mod, "DEV", "cpu")
    monkeypatch.setattr(test_gpu_langevin_noise, "XI_BOUND", {np.float32: 2.0**-23, np.float64: 2.0**-52})
    return handle


def _check(L, rc):
    if rc:
        raise RuntimeError(L.tmd_last_error().decode())


@pytest.mark.parametrize("nrep", [2, 3, 8, 33])
@pytest.mark.parametrize("f64", [False, True], ids=["fp32", "fp64"])
def test_exchange_kernel_against_the_oracle(hostsim, nrep, f64):
    """Random energies (stride 9, 9 terms and stride 9, 4 terms), 40 attempts from indices around 2^32 and 2^40: the
    ladder after every attempt, the counts, and the velocities bitwise."""
    L = hostsim
    natoms = 5
    h = C.c_void_p()
    _check(L, L.tmd_create(C.byref(h), 0, natoms, nrep))
    try:
        if f64:
            _check(L, L.tmd_set_precision(h, 64))
        rng = np.random.default_rng(nrep)
        temps = np.ascontiguousarray(300.0 * 1.02 ** np.arange(nrep))
        ladder = np.ascontiguousarray(rng.permutation(nrep).astype(np.int32))
        _check(L, L.tmd_set_temperature_ladder(h, nrep, temps.ctypes.data, ladder.ctypes.data))
        dt = np.float64 if f64 else np.float32
        vel = np.ascontiguousarray(rng.normal(size=(nrep, natoms, 3)).astype(dt))
        counts = np.zeros((nrep - 1, 2), np.int64)
        want_counts = np.zeros_like(counts)
        fn = L.tmd_replica_exchange_f64 if f64 else L.tmd_replica_exchange
        seed = 2**63 + 12345
        accepted = 0
        for n, a in enumerate(list(range(2**32 - 10, 2**32 + 10)) + list(range(2**40, 2**40 + 20))):
            nterms = 9 if n % 2 else 4
            ene = np.ascontiguousarray(rng.normal(0.0, 3.0, size=(nrep, 9)))
            before, v0 = ladder.copy(), vel.copy()
            U = remd.potentials(ene, 9, nterms)
            want, factor, tried = remd.exchange(before, U, temps, seed, a)
            _check(L, fn(h, ene.ctypes.data, 9, nterms, seed, a, vel.ctypes.data, counts.ctypes.data, None))
            assert np.array_equal(ladder, want), (a, before, want, ladder, tried)
            assert np.array_equal(vel, remd.scale(v0, factor, dt)), a
            for k, _, _, ok in tried:
                want_counts[k] += (1, int(ok))
                accepted += ok
            assert np.array_equal(counts, want_counts), a
        assert 0 < accepted < want_counts[:, 0].sum()
        # refusals: no ladder, too many terms for the stride
        assert fn(h, ene.ctypes.data, 4, 9, seed, 0, vel.ctypes.data, counts.ctypes.data, None) == -1
        _check(L, L.tmd_set_temperature_ladder(h, 0, None, None))
        assert fn(h, ene.ctypes.data, 9, 9, seed, 0, vel.ctypes.data, counts.ctypes.data, None) == -3
        bad = np.ascontiguousarray(np.zeros(nrep, np.int32))
        assert L.tmd_set_temperature_ladder(h, nrep, temps.ctypes.data, bad.ctypes.data) == -1
        assert L.tmd_set_temperature_ladder(h, nrep, np.ascontiguousarray(-temps).ctypes.data, ladder.ctypes.data) == -1
    finally:
        L.tmd_destroy(h)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32_full_rows", "fp64"])
def test_equal_temperatures_are_the_scalar_run(hostsim, monkeypatch, dtype):
    import test_gpu_replica_exchange as G

    G.test_equal_temperatures_are_the_scalar_run(monkeypatch, dtype)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["fp32_full_rows", "fp64"])
def test_ladder_replica_is_the_scalar_run_at_its_temperature(hostsim, monkeypatch, dtype):
    import test_gpu_replica_exchange as G

    G.test_ladder_replica_is_the_scalar_run_at_its_temperature(monkeypatch, dtype)


@pytest.mark.parametrize("name", ["cluster_fused_7", "cluster_fusestep0", "cluster_overlap0", "full_rows", "stepwise",
                                  "fp64_stepwise"])
def test_ladder_row_on_every_path(hostsim, monkeypatch, name):
    import test_gpu_replica_exchange as G

    G.test_ladder_row_on_every_path(monkeypatch, name)


@pytest.mark.parametrize("name", ["full_rows", "fp64", "stepwise"])
def test_exchange_decisions_follow_the_oracle(hostsim, monkeypatch, name):
    import test_gpu_replica_exchange as G

    G.decision_case(monkeypatch, name)


def test_exchanges_keep_the_captured_steps(hostsim, monkeypatch):
    import test_gpu_replica_exchange as G

    G.test_exchanges_keep_the_captured_steps(monkeypatch)

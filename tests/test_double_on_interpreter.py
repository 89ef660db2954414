"""The "precision: double" GPU tests run on the CPU: test_gpu_double's functions drive the C ABI of the host SIMT-interpreter
build of the library (tests/simt) with CPU tensors, through the patching of test_mirrors_on_interpreter.  The fp64 kernels
(k_prepare_f64, k_pack_f64, k_pair_f64, k_export_pairs_f64, the fp64 bonded and integrator kernels, k_wrap<double>)
and the fp64 branches of Forces / Integrator / Wrapper run here without a GPU.  Also here: seeded random systems against
the fp64 oracle (pairs bit for bit, coordinates up to the 8192 A limit of the list build's fp32 shadow), the precision
contract of the C ABI, and FrameSink in fp64."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import refmd
from test_mirrors_on_interpreter import _install

F64 = torch.float64
ERR_STATE, ERR_UNSUPPORTED = -3, -5


@pytest.fixture
def hostsim64(monkeypatch):
    handle = _install(monkeypatch, "")
    import test_gpu_double

    monkeypatch.setattr(test_gpu_double, "DEV", "cpu")
    return handle


GOLDENS = ["water291_rf_switch", "argon100_cut", "argon100_lj_rep_mix", "chain_amber_periodic", "chain_charmm_periodic",
           "adversarial_cutoff", "charmm_2watersperiodic", "charmm_benzamidine"]


@pytest.mark.parametrize("name", GOLDENS)
def test_goldens_f64(hostsim64, name):
    import test_gpu_double as D

    D.test_golden_forces_energies_f64(name)
    if name in D.PAIR_CASES:
        D.test_golden_neighbour_pairs_f64_bit_exact(name)


def test_amber_fixture_against_fp64_oracle(hostsim64):
    import test_gpu_double as D

    D.test_amber_fixtures_against_fp64_oracle("benzamidine_amber_nocut")
    D.test_amber_fixtures_against_fp64_oracle("ala2_xsc_rf")


@pytest.mark.parametrize("periodic", [False, True])
def test_cutoff_adversaries(hostsim64, periodic):
    import test_gpu_double as D

    D.test_cutoff_adversaries_at_fp64_resolution(periodic)


def test_trajectories_autograd_determinism_errors(hostsim64):
    import test_gpu_double as D

    D.test_nve_trajectory_f64()
    D.test_langevin_injected_noise_f64()
    D.test_autograd_and_vmap_f64()
    D.test_determinism_and_equal_replicas()
    D.test_overflow_regrowth_box_change_and_errors()  # (DecomposedIntegrator refusal included)


@pytest.mark.parametrize("case", ["water", "mixed", "nobonds", "zerobox"])
def test_wrap_f64(hostsim64, case):
    import test_gpu_double as D

    D.test_wrap_f64_bit_exact(case)


# ---- seeded random systems against the fp64 oracle -------------------------------------------------------------------
def _random_system(seed, periodic, far):
    """150 charged LJ atoms in a 22 A box, a third of them moved whole boxes away; ``far``: the system translated to
    5000-8100 A from the origin, where an fp32 ulp is 2^-10 to 2^-11 A (the shadow term of the list margin)."""
    rng = np.random.default_rng(seed)
    n, L = 150, 22.0
    x = rng.random((n, 3)) * L
    x += rng.integers(-2, 3, size=(n, 3)) * (rng.random((n, 1)) < 0.33) * L
    if far:
        x += rng.uniform(5000.0, 8000.0, size=3) if not periodic else L * np.floor(rng.uniform(5000.0, 8000.0, 3) / L)
    return torch.tensor(x)[None], (torch.eye(3, dtype=F64) * (L if periodic else 0.0))[None]


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("periodic", [False, True])
@pytest.mark.parametrize("far", [False, True])
def test_random_systems_against_fp64_oracle(hostsim64, seed, periodic, far):
    from test_gpu_forces import _lj_coulomb_parameters
    from torchmd_b200 import Forces

    pos, box = _random_system(seed, periodic, far)
    n = pos.shape[1]
    terms, cfg = ["lj", "electrostatics"], dict(cutoff=7.0, rfa=True, switch_dist=6.0)
    o = refmd.OracleForces(_lj_coulomb_parameters(n, F64, "cpu"), terms, decision_dtype=None, **cfg)
    want = o.neighbour_pairs(pos[0], torch.diagonal(box[0])).numpy().astype(np.int32)
    Fo = torch.zeros_like(pos)
    Eo = o.compute(pos, box, Fo)
    f = Forces(_lj_coulomb_parameters(n, F64, "cpu"), terms=terms, **cfg)
    F = torch.zeros_like(pos)
    E = f.compute(pos, box, F, returnDetails=True)
    assert np.array_equal(f.neighbour_pairs(pos, box).numpy(), want)
    assert len(want) > 0
    assert float((F - Fo).abs().max()) <= 1e-9 * max(1.0, float(Fo.abs().max()))
    for k in terms:
        assert abs(E[0][k] - float(Eo[0][k])) <= 1e-10 * abs(float(Eo[0][k])) + 1e-9, k


# ---- the precision contract of the C ABI -----------------------------------------------------------------------------
def test_c_abi_precision_contract(hostsim64):
    L = hostsim64
    n = 4
    q64, types = np.zeros(n), np.zeros(n, np.int32)
    pos64, f64 = np.zeros((1, n, 3)), np.zeros((1, n, 3))
    pos32, f32 = np.zeros((1, n, 3), np.float32), np.zeros((1, n, 3), np.float32)
    m64, m32 = np.ones(n), np.ones(n, np.float32)
    box64, box32 = np.full(3, 10.0), np.full(3, 10.0, np.float32)

    h = C.c_void_p()
    assert L.tmd_create(C.byref(h), 0, n, 1) == 0
    try:
        assert L.tmd_set_precision(h, 48) == -1
        assert L.tmd_set_precision(h, 64) == 0
        # fp32 entry points on an fp64 context
        assert L.tmd_set_atoms(h, q64.astype(np.float32).ctypes.data, types.ctypes.data, 1, None, None) == ERR_STATE
        assert b"fp64" in L.tmd_last_error()
        assert L.tmd_set_box(h, box32.ctypes.data) == ERR_STATE
        assert L.tmd_set_bonds(h, 0, None, None) == ERR_STATE
        assert L.tmd_forces(h, pos32.ctypes.data, f32.ctypes.data, None, None) == ERR_STATE
        assert L.tmd_vv_first(h, pos32.ctypes.data, f32.ctypes.data, f32.ctypes.data, m32.ctypes.data, 0.1, None) == ERR_STATE
        assert L.tmd_kinetic_energy(h, f32.ctypes.data, m32.ctypes.data, f64.ctypes.data, None) == ERR_STATE
        assert L.tmd_md_steps(h, 1, pos32.ctypes.data, f32.ctypes.data, f32.ctypes.data, m32.ctypes.data, 0.1, -1.0, None, None,
                              0, 0, None, None, None) == ERR_STATE
        # the fp64 setters are taken; the precision is then fixed
        assert L.tmd_set_atoms_f64(h, q64.ctypes.data, types.ctypes.data, 1, None, None) == 0
        assert L.tmd_set_box_f64(h, box64.ctypes.data) == 0
        assert L.tmd_set_precision(h, 32) == ERR_STATE
        assert L.tmd_set_precision(h, 64) == ERR_STATE
        # one GPU only
        assert L.tmd_set_owned_atoms(h, 0, 2) == ERR_UNSUPPORTED
        handle = (C.c_ubyte * 64)()
        assert L.tmd_dd_create(h, 0, 1, handle) == ERR_UNSUPPORTED
        assert L.tmd_dd_connect(h, handle) == ERR_UNSUPPORTED
        assert L.tmd_dd_load(h, 0, pos32.ctypes.data, None) == ERR_UNSUPPORTED
        assert L.tmd_dd_wait(h, None) == ERR_UNSUPPORTED
    finally:
        L.tmd_destroy(h)

    h = C.c_void_p()
    assert L.tmd_create(C.byref(h), 0, n, 1) == 0
    try:  # fp64 entry points on an fp32 context
        assert L.tmd_set_atoms_f64(h, q64.ctypes.data, types.ctypes.data, 1, None, None) == ERR_STATE
        assert b"fp32" in L.tmd_last_error()
        assert L.tmd_set_box_f64(h, box64.ctypes.data) == ERR_STATE
        assert L.tmd_forces_f64(h, pos64.ctypes.data, f64.ctypes.data, None, None) == ERR_STATE
        assert L.tmd_vv_first_f64(h, pos64.ctypes.data, f64.ctypes.data, f64.ctypes.data, m64.ctypes.data, 0.1, None) == ERR_STATE
        assert L.tmd_md_steps_f64(h, 1, pos64.ctypes.data, f64.ctypes.data, f64.ctypes.data, m64.ctypes.data, 0.1, -1.0, None,
                                  None, 0, 0, None, None, None) == ERR_STATE
        assert L.tmd_set_atoms(h, q64.astype(np.float32).ctypes.data, types.ctypes.data, 1, None, None) == 0
        assert L.tmd_set_precision(h, 64) == ERR_STATE  # after a setter
    finally:
        L.tmd_destroy(h)


def test_fp64_box_limit_and_far_flag_without_cutoff(hostsim64):
    """Box lengths above 4096 A are refused on fp64 contexts (the list margin's condition); without a cutoff every pair
    is listed and coordinates beyond 8192 A are accepted."""
    from test_gpu_forces import _lj_coulomb_parameters
    from torchmd_b200 import Forces
    from torchmd_b200._lib import TmdError

    pos, _ = _random_system(0, False, False)
    n = pos.shape[1]
    f = Forces(_lj_coulomb_parameters(n, F64, "cpu"), terms=["lj"], cutoff=7.0)
    with pytest.raises(TmdError, match="4096"):
        f.compute(pos, (torch.eye(3, dtype=F64) * 5000.0)[None], torch.zeros_like(pos))
    far = pos + 2.0e4
    o = refmd.OracleForces(_lj_coulomb_parameters(n, F64, "cpu"), ["lj"])
    Fo = torch.zeros_like(far)
    o.compute(far, torch.zeros(1, 3, 3, dtype=F64), Fo)
    g = Forces(_lj_coulomb_parameters(n, F64, "cpu"), terms=["lj"])
    F = torch.zeros_like(far)
    g.compute(far, torch.zeros(1, 3, 3, dtype=F64), F)
    assert float((F - Fo).abs().max()) <= 1e-9 * max(1.0, float(Fo.abs().max()))


def test_frame_sink_f64(tmp_path):
    from torchmd_b200.trajectory import FrameSink

    n, nrep = 7, 2
    sink = FrameSink(str(tmp_path / "out"), ".npy", n, nrep, "cpu", dtype=F64)
    frames = [torch.randn(nrep, n, 3, dtype=F64) * 1e3 + 1e-9 for _ in range(3)]
    for p in frames:
        sink.snapshot(p)
    sink.close()
    for k in range(nrep):
        got = np.load(tmp_path / f"out_{k}.npy")
        assert got.dtype == np.float64
        assert np.array_equal(got, np.stack([p[k].numpy() for p in frames], axis=2))
    with pytest.raises(ValueError):
        FrameSink(str(tmp_path / "bad"), ".npy", n, nrep, "cpu", dtype=torch.float16)

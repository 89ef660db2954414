"""Particle-mesh Ewald on the CPU, through the host SIMT-interpreter build of the library (tests/simt): the line DFT
against numpy.fft for every grid size the parameter choice can give from 10 to 128, and the GPU tests of
test_gpu_pme with CPU tensors at sizes the interpreter runs in seconds -- on the plain build (k_pair, stream path) and on
the build with every opt-in path as the default (k_pair_fx, the captured step with its conditional rebuild, the bonded
kernel and the reciprocal chain on their own streams)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_mirrors_on_interpreter import _install
from test_simt_kernels import CSRC, SIMT_DIR

def _sizes_235(lo, hi):
    out = []
    for n in range(lo, hi + 1):
        k = n
        for p in (2, 3, 5):
            while k % p == 0:
                k //= p
        if k == 1:
            out.append(n)
    return out


@pytest.fixture(scope="module")
def fft_lib():
    src = os.path.join(SIMT_DIR, "pme_fft.cpp")
    out = os.path.join(SIMT_DIR, "libpme_fft.so")
    deps = [src, os.path.join(CSRC, "pme.cuh"), os.path.join(SIMT_DIR, "simt.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        cmd = ["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-U_FORTIFY_SOURCE", "-I",
               os.path.join(SIMT_DIR, "stub"), "-I", CSRC, "-o", out + ".tmp", src]
        subprocess.run(cmd, check=True)
        os.replace(out + ".tmp", out)
    h = C.CDLL(out)
    h.simt_pme_line_dft.restype = C.c_int
    h.simt_pme_line_dft.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p]
    return h


@pytest.mark.parametrize("bits", [64, 32])
def test_line_dft_against_numpy(fft_lib, bits):
    rng = np.random.default_rng(bits)
    tol = 1e-13 if bits == 64 else 2e-6
    for n in _sizes_235(10, 128):
        x = rng.normal(size=n) + 1j * rng.normal(size=n)
        if bits == 32:
            x = x.astype(np.complex64).astype(np.complex128)
        for inverse, want in ((0, np.fft.fft(x)), (1, np.fft.ifft(x) * n)):
            buf = np.ascontiguousarray(np.stack([x.real, x.imag], 1).reshape(-1))
            assert fft_lib.simt_pme_line_dft(n, bits, inverse, buf.ctypes.data) == 0
            got = buf[0::2] + 1j * buf[1::2]
            err = np.abs(got - want).max() / np.abs(want).max()
            assert err <= tol * np.log2(n), (n, bits, inverse, err)


@pytest.fixture(params=["", "_r2"])
def hostsim_pme(monkeypatch, request):
    handle = _install(monkeypatch, request.param)
    import test_gpu_pme

    monkeypatch.setattr(test_gpu_pme, "DEV", "cpu")
    return handle


@pytest.mark.parametrize("name", ["water291_rf_switch", "charmm_sodiumperiodic", "charmm_2watersperiodic", "ala2_xsc_rf"])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_fixtures_against_the_oracle(hostsim_pme, name, dtype):
    import test_gpu_pme as G

    G.test_fixtures_against_the_oracle(name, dtype)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_replicas_in_different_boxes(hostsim_pme, dtype):
    import test_gpu_pme as G

    G.test_replicas_in_different_boxes(dtype, nw=60)


def test_pair_set_autograd_reproducibility_refusals(hostsim_pme):
    import test_gpu_pme as G

    for dtype in (torch.float32, torch.float64):
        G.test_pair_set_is_the_same_with_pme(dtype)
        G.test_forces_are_bitwise_reproducible(dtype)
    G.test_refusals()


def test_pme_kernels_only_with_pme(hostsim_pme, monkeypatch):
    import test_gpu_pme as G

    G.test_pme_kernels_only_with_pme(monkeypatch)


@pytest.mark.parametrize("fx", ["0", "2"])
def test_water_sampled_atoms_each_fp32_kernel(hostsim_pme, monkeypatch, fx):
    """A 3600-atom box (the cluster lists take it at a 6 A cutoff) on the Ewald cluster kernel, and on the full rows
    with k_pair_fx2_ew (FX=2) or k_pair<MODE 2> (FX=0), against the fp64 oracle on sampled atoms."""
    import test_gpu_pme as G

    for cluster in ("1", "0"):
        monkeypatch.setenv("TMD_B200_CLUSTER", cluster)
        monkeypatch.setenv("TMD_B200_FX", fx)
        kernel, _, dF, _, _ = G._water_big(1200, torch.float32, nsample=200, cutoff=6.0)
        assert kernel == (10 if cluster == "1" else {"0": 6, "2": 9}[fx]), kernel
        assert dF <= 5e-4, dF


def test_captured_steps_and_launches(monkeypatch):
    """Captured steps against the stream path, and the launch count, on the build with the conditional node."""
    _install(monkeypatch, "_r2")
    import test_gpu_pme as G

    monkeypatch.setattr(G, "DEV", "cpu")
    G.test_captured_steps_match_step_by_step(monkeypatch, nw=40, nsteps=4)
    G.test_launches_per_step_are_fixed(nw=40)


def test_under_a_random_thread_order():
    """The force checks again with the interpreter's threads in a random order (SIMT_SCHEDULE is read once per
    process): the fixed-point spread, the line DFTs and the gather do not depend on it."""
    env = dict(os.environ, SIMT_SCHEDULE="random:7")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", __file__, "-k",
                        "(fixtures and sodium) or replicas or line_dft or reproducibility"],
                       cwd=os.path.dirname(os.path.abspath(__file__)), env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_fp32_error_is_far_below_the_method_error(hostsim_pme):
    import test_gpu_pme as G

    G.test_fp32_error_is_far_below_the_method_error()

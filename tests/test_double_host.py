"""Host checks of the "precision: double" decision arithmetic (no GPU): the reference's fp64 predicate, the fp64
helpers of physics.cuh compiled for the host without FMA contraction, and the compiled fp64 pair kernel."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from conftest import ROOT

CSRC = os.path.join(ROOT, "torchmd_b200", "csrc")

SHIM = r"""
#include "physics.cuh"
extern "C" double threshold64(double rc) { return tmd::squared_threshold64(rc); }
extern "C" double image64(double d, double L) { return tmd::min_image64(d, L); }
extern "C" double norm2_64(double x, double y, double z) { return tmd::norm2_ref(x, y, z); }
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("physics64")
    src, lib = d / "shim.cpp", d / "libshim.so"
    src.write_text(SHIM)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-I", CSRC, "-o", str(lib), str(src)],
                   check=True)
    h = C.CDLL(str(lib))
    for name, nargs in (("threshold64", 1), ("image64", 2), ("norm2_64", 3)):
        getattr(h, name).restype = C.c_double
        getattr(h, name).argtypes = [C.c_double] * nargs
    return h


def fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def test_fp64_norm_is_fma_chain():
    """torch.norm(dim=1) on (P,3) fp64 is sqrt_rn(fma(z,z,fma(y,y,x*x))): the chain k_pair_f64 decides with."""
    torch.manual_seed(3)
    v = torch.randn(4001, 3, dtype=torch.float64) * 5
    n = torch.norm(v, dim=1).numpy()
    chain = np.array([math.sqrt(fma(z, z, fma(y, y, x * x))) for x, y, z in v.numpy()])
    assert np.array_equal(chain, n)


def test_threshold64_brackets_the_cutoff(shim):
    rng = np.random.default_rng(1)
    for c in [7.3, 9.0, 12.0, 2.5, 1e-3] + list(rng.uniform(1.0, 30.0, 200)):
        s = shim.threshold64(c)
        assert math.sqrt(s) <= c
        assert math.sqrt(np.nextafter(s, np.inf)) > c


def test_min_image64_is_the_reference_formula(shim):
    """w = d - L * round(d / L) in torch fp64 (forces.py:364) on separations at and around half-integers of L and
    several boxes away."""
    rng = np.random.default_rng(2)
    Ls = [30.0, 46.62, 99.99999, 12.3456789]
    ds = []
    for L in Ls:
        for m in range(-7, 8):
            base = (m + 0.5) * L
            ds += [(np.nextafter(base, s), L) for s in (-np.inf, np.inf)] + [(base, L)]
            ds += [(base + e, L) for e in rng.normal(0, 1e-12, 5)]
        ds += [(x, L) for x in rng.uniform(-4 * L, 4 * L, 200)]
    d = torch.tensor([x for x, _ in ds], dtype=torch.float64)
    L = torch.tensor([y for _, y in ds], dtype=torch.float64)
    want = (d - L * torch.round(d / L)).numpy()
    got = np.array([shim.image64(float(a), float(b)) for a, b in ds])
    assert np.array_equal(got, want)
    v = torch.randn(500, 3, dtype=torch.float64) * 7
    sq = np.array([shim.norm2_64(*map(float, r)) for r in v])
    assert np.array_equal(np.sqrt(sq), torch.norm(v, dim=1).numpy())


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA toolkit (cuobjdump) not on PATH")
def test_fp64_pair_kernel_loop_has_no_local_memory_and_fp32_kernels_stay():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import sass_budget

    table, res = sass_budget.functions(), sass_budget.resources()
    f64 = [n for n in table if "k_pair_f64" in n]
    assert len(f64) == 4
    for name in f64:
        lo, hi = sass_budget.main_loop(table[name])
        body = [t for _, t in table[name][lo : hi + 1]]
        assert not any("STL" in t or "LDL" in t for t in body), name
    # the fp32 production kernels are still built, within the budgets test_sass_invariants states
    for needle, max_regs in (("k_pairILb0ELb1ELb1ELi1E", 40), ("k_pair_fxILb0ELi1ELb1E", 48), ("k_pair_fx2ILb0E", 64)):
        names = [n for n in table if needle in n]
        assert names and res[names[0]][0] <= max_regs, needle
    for needle in ("k_cpair", "k_cstep_boundary", "k_vv_first", "k_vv_second", "k_bonded_terms", "k_build_list"):
        assert any(needle in n for n in table), needle

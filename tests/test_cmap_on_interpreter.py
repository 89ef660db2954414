"""test_gpu_cmap's functions on the host SIMT-interpreter build of the kernels (tests/simt): the CMAP kind in
k_bonded_terms / k_bonded_sum, in the deferred k_bonded_vv_second and in the fp64 bonded kernels, against the fp64
oracle, plus tmd_set_cmap's argument checks and a world-size-2 decomposition over gloo."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from conftest import ROOT
from test_mirrors_on_interpreter import _install


def _hostsim(monkeypatch, tag):
    handle = _install(monkeypatch, tag)
    import test_gpu_cmap

    monkeypatch.setattr(test_gpu_cmap, "DEV", "cpu")
    return handle


@pytest.fixture
def hostsim(monkeypatch):
    return _hostsim(monkeypatch, "")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", ["ala2_xsc_rf", "chain_amber_vacuum", "chain_amber_periodic"])
def test_cmap_against_oracle(hostsim, name, dtype):
    import test_gpu_cmap as G

    G.cmap_only_forces(name, dtype)
    G.dihedral_slot_sums(name, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_sign_seam_and_replicas(hostsim, dtype):
    import test_gpu_cmap as G

    G.sign_check(dtype)
    G.test_replicas_and_angles_at_the_seam(dtype)


def test_invariance_and_determinism(hostsim):
    import test_gpu_cmap as G

    G.invariance_and_determinism("chain_amber_vacuum")


@pytest.mark.parametrize("env", [{"TMD_B200_OVERLAP": "0"}, {"TMD_B200_OVERLAP": "1"}])
def test_two_pass_path_with_and_without_the_side_stream(hostsim, monkeypatch, env):
    import test_gpu_cmap as G

    G.paths_agree("ala2_xsc_rf", [env], monkeypatch)


def test_cluster_paths_deferred_and_folded(monkeypatch):
    """The cluster build: TMD_B200_OVERLAP=0 takes the deferred k_bonded_vv_second inside the captured steps, =1 the
    side stream folded into the half-kick."""
    import test_gpu_cmap as G

    _hostsim(monkeypatch, "_cl")
    G.paths_agree("ala2_xsc_rf", [{"TMD_B200_OVERLAP": "0"}, {"TMD_B200_OVERLAP": "1"}], monkeypatch)


def test_set_cmap_checks_its_arguments(hostsim):
    L = hostsim
    h = C.c_void_p()
    assert L.tmd_create(C.byref(h), 0, 6, 1) == 0
    try:
        res = np.array([4], np.int32)
        grid = np.zeros(16)
        idx = np.array([[0, 1, 2, 3, 4]], np.int32)
        m = np.zeros(1, np.int32)

        def call(res=res, grid=grid, idx=idx, m=m, nmaps=1, n=1):
            return L.tmd_set_cmap(h, nmaps, res.ctypes.data, grid.ctypes.data, n, idx.ctypes.data, m.ctypes.data)

        assert call() == 0
        assert call(res=np.array([3], np.int32), grid=np.zeros(9)) == -1 and b"resolution" in L.tmd_last_error()
        assert call(grid=np.full(16, np.nan)) == -1 and b"finite" in L.tmd_last_error()
        assert call(idx=np.array([[0, 1, 2, 3, 6]], np.int32)) == -1 and b"atom index" in L.tmd_last_error()
        assert call(m=np.ones(1, np.int32)) == -1 and b"map index" in L.tmd_last_error()
        assert call(nmaps=0) == -1
        assert L.tmd_set_cmap(h, 0, None, None, 0, None, None) == 0  # clears
    finally:
        L.tmd_destroy(h)


def _worker(rank, world, port, out):
    """DecomposedIntegrator (owned atom ranges, gloo all-gather) with CMAP terms against the single-process run."""
    import sys

    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    import test_gpu_cmap as G
    import test_simt_kernels as T
    from conftest import golden_cfg, golden_system_tensors, load_golden
    from torchmd_b200 import Forces, Integrator, System, _lib
    from torchmd_b200.domain import DecomposedIntegrator

    class _Stream:
        cuda_stream = None

    _lib._lib = T.load(os.path.join(T.SIMT_DIR, "libtmd_simt.so"))  # (built by the parent)
    _lib.on_device = lambda t: True
    torch.cuda.current_stream = lambda *a, **k: _Stream()
    torch.cuda.current_device = lambda: 0
    torch.cuda.synchronize = lambda *a, **k: None
    G.DEV = "cpu"

    name = "chain_amber_periodic"
    g = load_golden(name)
    terms = [str(t) for t in g["terms"]]

    def make():
        pos, box = golden_system_tensors(g, torch.float32)
        s = System(pos.shape[1], 1, torch.float32, "cpu")
        s.set_positions(pos[0].numpy())
        s.set_box(torch.diagonal(box[0]).numpy())
        f = Forces(G.make_params(g, name, torch.float32), terms=terms, **golden_cfg(g))
        f.compute(s.pos, s.box, s.forces)
        return s, f

    s1, f1 = make()
    single = Integrator(s1, f1, 0.5, "cpu")
    s2, f2 = make()
    dec = DecomposedIntegrator(s2, f2, 0.5, "cpu", use_graph=False)
    lo, hi = dec.dec.lo, dec.dec.hi
    ok = torch.equal(s1.forces[:, lo:hi], s2.forces[:, lo:hi])
    single.step(3)
    dec.step(3)
    ok = ok and torch.equal(s1.pos, s2.pos) and torch.equal(s1.forces[:, lo:hi], s2.forces[:, lo:hi])
    out.put((rank, bool(ok)))
    dist.destroy_process_group()


def test_decomposed_run_gloo():
    import socket

    import test_simt_kernels as T

    T.build_simt()
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    world = 2
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    results = dict(out.get(timeout=10) for _ in range(world))
    assert results == {0: True, 1: True}

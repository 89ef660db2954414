"""The real kernel sources executed on the CPU by the SIMT interpreter of tests/simt (fibers with
warp/block collectives; see tests/simt/simt.h) and driven through the C ABI with numpy arrays.

Purpose: check the LOGIC of the kernels -- cell binning, sorting, tile staging, chunk culling, list
rows, decision band, packed two-partner evaluation, masks, double buffering -- without a GPU.  The
arithmetic runs as the host alternatives of physics.cuh / ptx.cuh (exactly rounded where the device
uses approximations + Newton), so force values agree with the GPU to rounding, not bit for bit.
Test infrastructure only: torchmd_b200/_lib.py refuses to load this build.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT, golden_cfg, golden_system_tensors, load_golden, params_from_golden

SIMT_DIR = os.path.join(ROOT, "tests", "simt")
CSRC = os.path.join(ROOT, "torchmd_b200", "csrc")


VARIANTS = {  # tag -> defines; every interpreter build the tests use (built together, in parallel, when stale)
    "": [],
    # every opt-in path as the default
    "_r2": ["TMD_DEFAULT_FX=2", "TMD_DEFAULT_OVERLAP=1", "TMD_DEFAULT_FUSEPREP=1", "TMD_DEFAULT_GRAPH=1", "TMD_DEFAULT_CLUSTER=1"],
    "_cl": ["TMD_DEFAULT_CLUSTER=1", "TMD_DEFAULT_GRAPH=1", "TMD_DEFAULT_FUSEPREP=1", "TMD_DEFAULT_OVERLAP=1"],  # the cluster half-list path (cluster.cuh) over the plain kernels
    "_t2": ["FX_SMALLT_MAX_N=2"],
}


def _simt_command(out, defines):
    cmd = ["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-U_FORTIFY_SOURCE", "-I", os.path.join(SIMT_DIR, "stub"), "-I", CSRC]
    if "TMD_SIMT_ASAN=1" in defines:  # scripts/asan_interpreter.py
        cmd += ["-fsanitize=address", "-fno-omit-frame-pointer", "-g", "-DSIMT_UCONTEXT_ONLY"]
    # the interpreter builds start from the plain kernels (every opt-in path off) so that a variant is compared
    # with the same baseline whatever the product's defaults are; a variant's own defines come later and win
    keys = {d.split("=")[0] for d in defines}
    base = [d for d in ("TMD_DEFAULT_FX=0", "TMD_DEFAULT_OVERLAP=0", "TMD_DEFAULT_FUSEPREP=0", "TMD_DEFAULT_CLUSTER=0", "TMD_DEFAULT_GRAPH=0")
            if d.split("=")[0] not in keys]
    return cmd + [f"-D{d}" for d in base + list(defines)] + ["-o", out, os.path.join(SIMT_DIR, "simt_lib.cpp")]


def _simt_stale(out):
    srcs = [os.path.join(SIMT_DIR, f) for f in ("simt_lib.cpp", "simt.h", os.path.join("stub", "cuda_runtime.h"))]
    srcs += [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    return not os.path.exists(out) or any(os.path.getmtime(s) > os.path.getmtime(out) for s in srcs)


def build_simt(tag="", defines=()):
    out = os.path.join(SIMT_DIR, f"libtmd_simt{tag}.so")
    if _simt_stale(out):
        jobs = {tag: (out, list(defines))}
        if tag in VARIANTS:  # one of the suite's builds is stale: the others are too -- compile them side by side
            for t, d in VARIANTS.items():
                o = os.path.join(SIMT_DIR, f"libtmd_simt{t}.so")
                if t != tag and _simt_stale(o):
                    jobs[t] = (o, d)
        procs = [(o, subprocess.Popen(_simt_command(o + ".tmp", d), cwd=ROOT)) for o, d in jobs.values()]
        for o, pr in procs:
            if pr.wait() != 0:
                raise RuntimeError(f"building {o} failed")
            os.replace(o + ".tmp", o)
    return out


def load(path):
    from torchmd_b200 import _lib

    h = C.CDLL(path)
    for name, (res, args) in _lib._SIGNATURES.items():
        fn = getattr(h, name)
        fn.restype, fn.argtypes = res, args
    assert h.tmd_version() == -100
    return h


@pytest.fixture(scope="module")
def simt():
    return load(build_simt())


class Ctx:
    """A context of the interpreter build configured like Forces._ensure_ctx does for the CUDA library."""

    def __init__(self, L, g, env=None, terms=None, **kw):
        from torchmd_b200 import Forces, _lib

        self.L, self.g = L, g
        self.check = lambda rc: (_ for _ in ()).throw(RuntimeError(L.tmd_last_error().decode())) if rc else None
        cfg = golden_cfg(g)
        cfg.update(kw)
        self.terms = terms or [str(t) for t in g["terms"]]
        self.f = Forces(params_from_golden(g, precision=torch.float32), terms=self.terms, **cfg)
        pos, box = golden_system_tensors(g, torch.float32)
        self.pos = np.ascontiguousarray(pos.numpy())
        self.nrep, self.natoms = self.pos.shape[:2]
        self.box = np.ascontiguousarray(torch.diagonal(box, dim1=1, dim2=2).numpy().astype(np.float32))
        self.h = C.c_void_p()
        self.check(L.tmd_create(C.byref(self.h), 0, self.natoms, self.nrep))
        self.f._configure(L, self.h, self.check)
        self.check(L.tmd_set_box(self.h, self.box.ctypes.data))
        self.env = dict(env or {})

    def forces(self, energies=True, pos=None):
        from torchmd_b200 import _lib

        pos = self.pos if pos is None else pos
        F = np.full_like(pos, 7.0)
        E = np.zeros((self.nrep, _lib.NUM_ENERGIES))
        old = {k: os.environ.get(k) for k in self.env}
        os.environ.update(self.env)
        try:
            for _ in range(4):
                self.check(self.L.tmd_forces(self.h, pos.ctypes.data, F.ctypes.data, E.ctypes.data if energies else None, None))
                st = _lib.Stats()
                rc = self.L.tmd_get_stats(self.h, C.byref(st), None)
                if rc == 0:
                    break
                if rc != _lib.ERR_OVERFLOW:
                    self.check(rc)
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        self.stats = st
        return F, {t: E[:, _lib.ENERGY_SLOTS.index(t)] for t in self.terms}

    def pairs(self, pos=None):
        pos = self.pos if pos is None else pos
        cap = 4_000_000
        buf = np.zeros((cap, 2), np.int32)
        cnt = np.zeros(1, np.int64)
        self.check(self.L.tmd_export_pairs(self.h, pos.ctypes.data, 0, buf.ctypes.data, cap, cnt.ctypes.data, None))
        out = buf[: int(cnt[0])]
        return out[np.lexsort((out[:, 1], out[:, 0]))]

    def close(self):
        self.L.tmd_destroy(self.h)


def check_against_golden(c, F, E, tol=1e-4):
    g = c.g
    ref = g["forces_f64"]
    scale = max(1.0, float(np.abs(ref).max()) / 100.0)
    dev = np.abs(g["forces_f32"].astype(np.float64) - ref).max()
    err = np.abs(F.astype(np.float64) - ref).max()
    assert err < max(tol * scale, 1.2 * dev), err
    keys = [str(k) for k in g["energy_keys"]]
    for r in range(c.nrep):
        for col, k in enumerate(keys):
            if k in E:
                e_ref = g["energies_f64"][r, col]
                assert abs(E[k][r] - e_ref) <= 1e-5 * abs(e_ref) + 2e-3, (k, E[k][r], e_ref)
    return err


@pytest.mark.parametrize("name", ["water291_rf_switch", "argon100_cut", "chain_amber_periodic", "chain_amber_vacuum", "adversarial_cutoff"])
def test_interpreter_reproduces_the_gpu_validated_default_path(simt, name):
    """Validates the interpreter itself: the default kernels are parity-green on the GPU."""
    g = load_golden(name)
    c = Ctx(simt, g)
    F, E = c.forces()
    check_against_golden(c, F, E)
    if "pairs_f32" in g:
        assert np.array_equal(c.pairs(), g["pairs_f32"])
    assert c.stats.rebuilds >= 1 and not c.stats.overflow
    c.close()


FX_CASES = ["argon100_cut", "chain_amber_periodic", "chain_charmm_periodic", "adversarial_cutoff", "water999_eq"]


@pytest.mark.parametrize("mode", ["1", "2"])
@pytest.mark.parametrize("name", FX_CASES)
def test_fixed_point_and_packed_pair_kernels(simt, name, mode):
    """k_pair_fx (TMD_B200_FX=1) and k_pair_fx2 (=2): energies pass and force-only pass against the golden
    vectors; the exported pair set (reference predicate) is unchanged; both agree closely with the float kernel."""
    g = load_golden(name)
    # the 21.5 A box of the 999-atom fixture only meets the guard-free image condition
    # (cutoff + 2 skin < 0.45 L) with a thin skin
    kw = {"skin": 0.2} if name == "water999_eq" else {}
    c = Ctx(simt, g, env={"TMD_B200_FX": mode}, **kw)
    F, E = c.forces()
    assert simt.tmd_pair_kernel(c.h) == int(mode), "the fixed-point / packed kernel did not run"
    err = check_against_golden(c, F, E)
    F2, _ = c.forces(energies=False)
    assert simt.tmd_pair_kernel(c.h) == int(mode)
    err2 = check_against_golden(c, F2, {})
    assert np.abs(F - F2).max() < 2e-5 * max(1.0, np.abs(F).max() / 100)
    if "pairs_f32" in g:
        assert np.array_equal(c.pairs(), g["pairs_f32"])
    c0 = Ctx(simt, g, **kw)
    F0, _ = c0.forces()
    assert np.abs(F - F0).max() < 1e-4 * max(1.0, np.abs(F0).max() / 100)
    print(f"{name} FX={mode}: err {err:.2e} / {err2:.2e} (force-only)")
    c.close()
    c0.close()


@pytest.mark.parametrize("name", ["chain_amber_vacuum", "argon100_nocut", "ala2_nobox_rf", "benzamidine_amber_nocut", "ligand_amber_nocut"])
def test_packed_kernel_without_a_box(simt, name):
    g = load_golden(name)
    c = Ctx(simt, g, env={"TMD_B200_FX": "2"})
    F, E = c.forces()
    # (argon100_nocut has a box but no cutoff: periodic all-pairs, the float kernel by design)
    assert simt.tmd_pair_kernel(c.h) == (3 if not np.any(g["box"]) else 0)
    check_against_golden(c, F, E)
    F2, _ = c.forces(energies=False)
    check_against_golden(c, F2, {})
    if "pairs_f32" in g:
        assert np.array_equal(c.pairs(), g["pairs_f32"])
    c.close()


@pytest.mark.parametrize("name", ["water291_rf_switch", "argon100_cut", "chain_amber_periodic", "chain_amber_vacuum", "water999_eq", "ala2_nobox_rf"])
def test_list_build_gives_the_reference_pair_set(simt, name):
    """Chunk culling, run-wise tile fill and the two-atom chunk loop must leave no pair of the reference out of the
    rows: the exported pair set equals the reference's, and the forces summed over the rows match the goldens."""
    from oracle import refmd

    g = load_golden(name)
    c = Ctx(simt, g)
    F, E = c.forces()
    check_against_golden(c, F, E)
    assert not c.stats.overflow
    if "pairs_f32" in g:
        ref_pairs = g["pairs_f32"]
    else:  # no stored pair set: the fp32 oracle's, as oracle_check takes it
        of32 = refmd.OracleForces(params_from_golden(g, precision=torch.float32), c.terms, **golden_cfg(g))
        ref_pairs = of32.neighbour_pairs(torch.tensor(c.pos[0]), torch.tensor(g["box"])).numpy().astype(np.int32)
    assert np.array_equal(c.pairs(), ref_pairs)
    c.close()


def test_bonded_overlap_is_bit_identical(simt):
    g = load_golden("chain_amber_periodic")
    a, b = Ctx(simt, g), Ctx(simt, g, env={"TMD_B200_OVERLAP": "1"})
    Fa, Ea = a.forces()
    Fb, Eb = b.forces()
    assert np.array_equal(Fa, Fb)
    assert b.stats.kernel_launches == a.stats.kernel_launches + 1  # the overlapped path really ran: k_add_bonded
    for k in Ea:
        assert np.allclose(Ea[k], Eb[k], rtol=1e-12, atol=1e-9)
    a.close()
    b.close()


def test_exact_gradient_convention(simt):
    """tmd_set_force_convention(1): the reference's autograd forces (water291_autograd.npz)."""
    g, ga = load_golden("water291_rf_switch"), load_golden("water291_autograd")
    c = Ctx(simt, g)
    c.check(simt.tmd_set_force_convention(c.h, 1))
    F, E = c.forces()
    assert np.abs(F.astype(np.float64) - ga["forces_autograd_f64"]).max() < 1e-4
    c.check(simt.tmd_set_force_convention(c.h, 0))
    F, E = c.forces()
    assert np.abs(F.astype(np.float64) - g["forces_f64"]).max() < 1e-4
    c.close()


def test_fixed_point_kernels_with_drifted_molecules(simt):
    """Molecules up to 3 boxes away: fixed-point separations stay exact where the float path loses 1e-3."""
    from oracle import refmd

    g = load_golden("water999_eq")
    cfg = golden_cfg(g)
    rng = np.random.default_rng(7)
    box = g["box"].astype(np.float64)
    shift = rng.integers(-3, 4, (len(g["coords"]) // 3, 3)).repeat(3, axis=0)
    coords = (g["coords"].astype(np.float64) + shift * box).astype(np.float32)
    terms = [str(t) for t in g["terms"]]
    of = refmd.OracleForces(params_from_golden(g, precision=torch.float64), terms, decision_dtype=torch.float32, **cfg)
    pos_t = torch.tensor(coords)[None]
    f64 = torch.zeros(1, len(coords), 3, dtype=torch.float64)
    of.compute(pos_t.double(), torch.diag(torch.tensor(g["box"]))[None].double(), f64)
    of32 = refmd.OracleForces(params_from_golden(g, precision=torch.float32), terms, **cfg)
    pairs_ref = of32.neighbour_pairs(pos_t[0], torch.tensor(g["box"])).numpy().astype(np.int32)
    pos = np.ascontiguousarray(coords[None])
    for mode in ("1", "2"):
        c = Ctx(simt, g, env={"TMD_B200_FX": mode}, skin=0.2)
        F, _ = c.forces(pos=pos)
        assert simt.tmd_pair_kernel(c.h) == int(mode)
        err = np.abs(F.astype(np.float64) - f64.numpy()).max()
        assert err < 1e-4, (mode, err)
        assert np.array_equal(c.pairs(pos=pos), pairs_ref)
        c.close()


@pytest.mark.parametrize("name", ["water", "mixed", "nobonds", "zerobox"])
def test_wrap_kernel(simt, name):
    from torchmd_b200.wrapper import Wrapper

    g = load_golden("wrap_cases")
    bonds = g[name + "_bonds"]
    natoms = int(g[name + "_natoms"])
    w = Wrapper(natoms, bonds if len(bonds) else None, "cpu")
    pos = np.ascontiguousarray(g[name + "_pos"], np.float32).copy()
    box = np.ascontiguousarray(g[name + "_box"], np.float32)
    h = C.c_void_p()
    assert simt.tmd_wrapper_create(C.byref(h), 0, natoms, len(w._ptr) - 1, w._ptr.ctypes.data, w._atoms.ctypes.data) == 0
    assert simt.tmd_wrapper_wrap(h, pos.ctypes.data, box.ctypes.data, pos.shape[0], None) == 0
    assert np.array_equal(pos, g[name + "_after"])
    simt.tmd_wrapper_destroy(h)


# ---- integration: fused steps, injected-noise Langevin, peer-to-peer exchange with one rank ---------------
TIMEFACTOR, BOLTZMAN = 48.88821, 0.001987191  # reference integrator.py:4-5


def md_setup(simt, env=None):
    from torchmd_b200 import _lib

    g, t = load_golden("water291_rf_switch"), load_golden("water291_traj")
    c = Ctx(simt, g, env=env)
    c.vel = np.ascontiguousarray(t["vel0_f32"]).copy()
    c.posw = c.pos.copy()
    c.F, _ = c.forces(pos=c.posw)  # forces of the start configuration, like Integrator users do (run.py:259)
    c.masses = np.ascontiguousarray(g["par_masses"].astype(np.float32))
    c.dt = 1.0 / TIMEFACTOR
    c.ene = np.zeros((c.nrep, _lib.NUM_ENERGIES))
    c.ke = np.zeros(c.nrep)
    return g, t, c


def md_steps(simt, c, niter, gamma=-1.0, vcoeff=None, noise=None, seed=1234):
    c.check(simt.tmd_md_steps(c.h, niter, c.posw.ctypes.data, c.vel.ctypes.data, c.F.ctypes.data, c.masses.ctypes.data, c.dt, gamma,
                              None if vcoeff is None else vcoeff.ctypes.data, None if noise is None else noise.ctypes.data, seed, 0,
                              c.ene.ctypes.data, c.ke.ctypes.data, None))


def test_fused_md_steps_follow_the_reference_trajectories(simt):
    g, t, c = md_setup(simt)
    md_steps(simt, c, 1)
    assert np.abs(c.posw - t["nve_pos1_f64"]).max() < 2e-6
    md_steps(simt, c, 9)
    assert np.abs(c.posw - t["nve_pos10_f32"]).max() < 2e-5 and np.abs(c.vel - t["nve_vel10_f32"]).max() < 5e-5
    np.testing.assert_allclose(c.ke, t["nve_ekin10_f32"], rtol=5e-5)
    c.close()
    # Langevin with the reference's own noise
    g, t, c = md_setup(simt)
    gamma = 0.1 / (1000.0 / TIMEFACTOR)
    vcoeff = np.sqrt(2.0 * gamma / c.masses.astype(np.float64) * BOLTZMAN * 300.0 * c.dt).astype(np.float32)
    noise = np.ascontiguousarray(t["lan_noise_f32"])
    md_steps(simt, c, 4, gamma=gamma, vcoeff=vcoeff, noise=noise)
    assert np.abs(c.posw - t["lan_pos4_f32"]).max() < 2e-5 and np.abs(c.vel - t["lan_vel4_f32"]).max() < 5e-5
    c.close()


@pytest.mark.parametrize("extra", [{}, {"TMD_B200_OVERLAP": "1", "TMD_B200_FX": "2"}])
def test_integrate_and_prepare_in_one_kernel_is_bit_identical(simt, extra):
    """TMD_B200_FUSEPREP=1: k_vv_first_prepare (move the atoms, check the list, refresh the sorted records) against
    k_vv_first followed by k_prepare -- same trajectory to the last bit across list rebuilds, one launch fewer per
    step; a plain force call after fused steps still prepares for itself."""
    from torchmd_b200 import _lib

    g, t, a = md_setup(simt, env=dict(extra))
    _, _, b = md_setup(simt, env=dict(extra, TMD_B200_FUSEPREP="1"))
    gamma = 0.1 / (1000.0 / TIMEFACTOR)
    vcoeff = np.sqrt(2.0 * gamma / a.masses.astype(np.float64) * BOLTZMAN * 300.0 * a.dt).astype(np.float32)
    st = [_lib.Stats(), _lib.Stats()]
    for k, c in enumerate((a, b)):
        assert simt.tmd_get_stats(c.h, C.byref(st[k]), None) == 0
    l0 = [s.kernel_launches for s in st]
    total = 0
    for niter in (1, 2, 17):
        for c in (a, b):
            md_steps(simt, c, niter, gamma=gamma, vcoeff=vcoeff, seed=5)
        total += niter
        assert np.array_equal(a.posw, b.posw) and np.array_equal(a.vel, b.vel) and np.array_equal(a.F, b.F)
        # (energies are block-wise fp64 atomic sums: equal up to the order of the additions)
        assert np.allclose(a.ene, b.ene, rtol=1e-12, atol=1e-9) and np.allclose(a.ke, b.ke, rtol=1e-12, atol=1e-9)
    for k, c in enumerate((a, b)):
        assert simt.tmd_get_stats(c.h, C.byref(st[k]), None) == 0
    assert st[0].rebuilds == st[1].rebuilds and st[0].rebuilds >= 2  # the list is rebuilt on the way
    # one launch fewer per step (k_prepare), two with the overlapped bonded kernel (k_add_bonded folded into k_vv_second)
    assert (st[0].kernel_launches - l0[0]) - (st[1].kernel_launches - l0[1]) == total * (2 if "TMD_B200_OVERLAP" in extra else 1)
    Fa, Ea = a.forces(pos=a.posw)
    Fb, Eb = b.forces(pos=b.posw)
    assert np.array_equal(Fa, Fb) and repr(Ea) == repr(Eb)
    a.close()
    b.close()


@pytest.mark.parametrize("extra", [{}, {"TMD_B200_OVERLAP": "1", "TMD_B200_FX": "2", "TMD_B200_FUSEPREP": "1"}])
def test_captured_step_with_conditional_rebuild_replays_the_stream_path(simt, extra):
    """TMD_B200_GRAPH=1 (the interpreter's record-and-replay model of stream capture, tests/simt/stub): tmd_md_steps
    captures one step twice (with / without energy outputs), the rebuild kernels go into the body of an IF node that
    the preparing kernel switches on, and replaying gives the trajectory of the plain stream path bit for bit -- with
    the rebuild kernels launched only on the steps that rebuild."""
    from torchmd_b200 import _lib

    g, t, a = md_setup(simt, env=dict(extra))
    _, _, b = md_setup(simt, env=dict(extra, TMD_B200_GRAPH="1"))
    gamma = 0.1 / (1000.0 / TIMEFACTOR)
    vcoeff = np.sqrt(2.0 * gamma / a.masses.astype(np.float64) * BOLTZMAN * 300.0 * a.dt).astype(np.float32)
    st = [_lib.Stats(), _lib.Stats()]
    for k, c in enumerate((a, b)):
        assert simt.tmd_get_stats(c.h, C.byref(st[k]), None) == 0
    l0, r0 = [s.kernel_launches for s in st], [s.rebuilds for s in st]
    before = (C.c_longlong * 3)()
    simt.simt_graph_counters(before)  # (the model's counters are per process: other tests replay graphs too)
    total = 0
    for niter in (1, 2, 17):
        for c in (a, b):
            md_steps(simt, c, niter, gamma=gamma, vcoeff=vcoeff, seed=5)
        total += niter
        assert np.array_equal(a.posw, b.posw) and np.array_equal(a.vel, b.vel) and np.array_equal(a.F, b.F)
        # (energies are block-wise fp64 atomic sums: equal up to the order of the additions)
        assert np.allclose(a.ene, b.ene, rtol=1e-12, atol=1e-9) and np.allclose(a.ke, b.ke, rtol=1e-12, atol=1e-9)
    for k, c in enumerate((a, b)):
        assert simt.tmd_get_stats(c.h, C.byref(st[k]), None) == 0
    rebuilds = st[0].rebuilds - r0[0]
    assert st[1].rebuilds - r0[1] == rebuilds and 2 <= rebuilds < total
    after = (C.c_longlong * 3)()
    simt.simt_graph_counters(after)
    replays, ran, skipped = (after[k] - before[k] for k in range(3))
    assert replays == total and ran + skipped == total  # every step was a replay and met its IF node ...
    assert ran == rebuilds                               # ... whose body ran exactly on the steps that rebuilt
    # a step that keeps its list launches none of the five rebuild kernels: the library's launch count is the captured
    # step's node count (body included), so the check is on what actually ran -- the rebuild counter -- and on the results
    Fa, Ea = a.forces(pos=a.posw)
    Fb, Eb = b.forces(pos=b.posw)
    assert np.array_equal(Fa, Fb) and repr(Ea) == repr(Eb)
    a.close()
    b.close()


@pytest.mark.parametrize("thermostat", [False, True])
def test_peer_to_peer_exchange_with_one_rank_equals_fused_steps(simt, thermostat):
    """tmd_dd_* (double-buffered positions, push kernel, flag wait) with world size 1 against tmd_md_steps:
    identical arithmetic, so positions and velocities must agree bit for bit -- odd and even step counts,
    in-kernel Philox noise included."""
    g, t, a = md_setup(simt)
    _, _, b = md_setup(simt)
    gamma = 0.1 / (1000.0 / TIMEFACTOR) if thermostat else -1.0
    vcoeff = np.sqrt(2.0 * gamma / a.masses.astype(np.float64) * BOLTZMAN * 300.0 * a.dt).astype(np.float32) if thermostat else None
    handle = (C.c_ubyte * 64)()
    # single replica contexts only: use replica 0 of the fixture in a one-replica context
    a.close()
    b.close()
    g1 = dict(g)
    g1["cfg_nrep"] = np.int64(1)
    ga = Ctx(simt, g1)
    gb = Ctx(simt, g1)
    from torchmd_b200 import _lib

    for c in (ga, gb):
        c.vel = np.ascontiguousarray(t["vel0_f32"][:1]).copy()
        c.posw = c.pos.copy()
        c.F, _ = c.forces(pos=c.posw)
        c.masses = np.ascontiguousarray(g["par_masses"].astype(np.float32))
        c.dt = 1.0 / TIMEFACTOR
        c.ene = np.zeros((1, _lib.NUM_ENERGIES))
        c.ke = np.zeros(1)
    gb.check(simt.tmd_dd_create(gb.h, 0, 1, handle))
    gb.check(simt.tmd_dd_connect(gb.h, handle))
    parity = 0
    for niter in (1, 2, 5):
        md_steps(simt, ga, niter, gamma=gamma, vcoeff=vcoeff, seed=77)
        gb.check(simt.tmd_dd_load(gb.h, parity, gb.posw.ctypes.data, None))
        for it in range(niter):
            last = it == niter - 1
            gb.check(simt.tmd_dd_vv_first_push(gb.h, parity, gb.vel.ctypes.data, gb.F.ctypes.data, gb.masses.ctypes.data, gb.dt, None))
            gb.check(simt.tmd_dd_wait(gb.h, None))
            gb.check(simt.tmd_dd_forces(gb.h, 1 - parity, gb.F.ctypes.data, gb.ene.ctypes.data if last else None, None))
            gb.check(simt.tmd_vv_second(gb.h, gb.vel.ctypes.data, gb.F.ctypes.data, gb.masses.ctypes.data, gb.dt, gamma,
                                        None if vcoeff is None else vcoeff.ctypes.data, None, 77, 0, gb.ke.ctypes.data if last else None, None))
            parity ^= 1
        gb.check(simt.tmd_dd_store(gb.h, parity, gb.posw.ctypes.data, None))
        assert np.array_equal(ga.posw, gb.posw) and np.array_equal(ga.vel, gb.vel) and np.array_equal(ga.F, gb.F)
        assert np.allclose(ga.ke, gb.ke, rtol=1e-12) and np.allclose(ga.ene, gb.ene, rtol=1e-12, atol=1e-9)
    st = _lib.Stats()
    assert simt.tmd_get_stats(gb.h, C.byref(st), None) == 0  # (a timed-out flag wait would be reported here)
    ga.close()
    gb.close()


def test_fixed_point_kernels_across_rebuilds(simt):
    """A dozen NVE steps of the 999-atom box with a thin skin (several list rebuilds): the packed fixed-point
    kernel works on stale-but-valid lists with per-step refreshed records; trajectory stays with the float
    kernel's and the final forces / pair set match the oracle."""
    from oracle import refmd
    from torchmd_b200 import _lib

    g = load_golden("water999_eq")
    cfg = golden_cfg(g)
    out = {}
    for mode in ("0", "2"):
        c = Ctx(simt, g, env={"TMD_B200_FX": mode}, skin=0.2)
        c.vel = np.ascontiguousarray(g["vel"][None].astype(np.float32)).copy()
        c.posw = c.pos.copy()
        c.F, _ = c.forces(pos=c.posw)
        c.masses = np.ascontiguousarray(g["par_masses"].astype(np.float32))
        c.dt = 1.0 / TIMEFACTOR
        c.ene = np.zeros((1, _lib.NUM_ENERGIES))
        c.ke = np.zeros(1)
        os.environ["TMD_B200_FX"] = mode
        try:
            md_steps(simt, c, 12)
        finally:
            os.environ.pop("TMD_B200_FX", None)
        assert simt.tmd_pair_kernel(c.h) == int(mode)
        st = _lib.Stats()
        assert simt.tmd_get_stats(c.h, C.byref(st), None) == 0
        out[mode] = (c.posw.copy(), c.vel.copy(), c.F.copy(), st.rebuilds, c)
    assert out["2"][3] >= 3, "the thin skin should have forced several rebuilds"
    assert np.abs(out["0"][0] - out["2"][0]).max() < 2e-5 and np.abs(out["0"][1] - out["2"][1]).max() < 1e-4
    # final state against the oracle: forces of the last step belong to the final positions
    posf, c = out["2"][0], out["2"][4]
    terms = [str(t) for t in g["terms"]]
    of = refmd.OracleForces(params_from_golden(g, precision=torch.float64), terms, decision_dtype=torch.float32, **cfg)
    f64 = torch.zeros(1, c.natoms, 3, dtype=torch.float64)
    of.compute(torch.tensor(posf).double(), torch.diag(torch.tensor(g["box"]))[None].double(), f64)
    assert np.abs(out["2"][2].astype(np.float64) - f64.numpy()).max() < 1e-4
    of32 = refmd.OracleForces(params_from_golden(g, precision=torch.float32), terms, **cfg)
    ref_pairs = of32.neighbour_pairs(torch.tensor(posf[0]), torch.tensor(g["box"])).numpy().astype(np.int32)
    os.environ["TMD_B200_FX"] = "2"
    try:
        assert np.array_equal(c.pairs(pos=posf), ref_pairs)
    finally:
        os.environ.pop("TMD_B200_FX", None)
    for m in out:
        out[m][4].close()


def test_replicas_are_independent_in_the_packed_kernel(simt):
    g = dict(load_golden("chain_amber_periodic"))
    g["cfg_nrep"] = np.int64(2)
    c = Ctx(simt, g, env={"TMD_B200_FX": "2"})
    rng = np.random.default_rng(3)
    pos = c.pos.copy()
    pos[1] += rng.normal(scale=0.02, size=pos[1].shape).astype(np.float32)
    F, E = c.forces(pos=pos)
    assert simt.tmd_pair_kernel(c.h) == 2
    g1 = dict(g)
    g1["cfg_nrep"] = np.int64(1)
    for r in range(2):
        s = Ctx(simt, g1, env={"TMD_B200_FX": "2"})
        Fr, Er = s.forces(pos=np.ascontiguousarray(pos[r : r + 1]))
        assert np.array_equal(F[r], Fr[0])
        for k in E:
            assert abs(E[k][r] - Er[k][0]) <= 1e-9 * max(1.0, abs(Er[k][0]))
        s.close()
    c.close()


@pytest.mark.parametrize("variant", ["default", "packed"])
def test_owned_atom_range_forces_match_the_full_evaluation(simt, variant):
    """Decomposed runs (tmd_set_owned_atoms): rows, forces and bonded terms of an owned sub-range equal the same
    atoms' values in the full evaluation, bit for bit, in every kernel variant."""
    env = {"TMD_B200_FX": "2"} if variant == "packed" else None
    g = load_golden("chain_amber_periodic")
    full = Ctx(simt, g, env=env)
    Ff, Ef = full.forces()
    part = Ctx(simt, g, env=env)
    n = part.natoms
    lo, cnt = n // 3, n // 2
    part.check(simt.tmd_set_owned_atoms(part.h, lo, cnt))
    Fp, Ep = part.forces()
    assert np.array_equal(Fp[0, lo : lo + cnt], Ff[0, lo : lo + cnt])
    assert 0 < abs(Ep["lj"][0]) < abs(Ef["lj"][0]) * 1.0001 + 1.0
    full.close()
    part.close()


def test_the_package_refuses_the_interpreter_build(simt):
    """The interpreter library is a unit-test tool: torchmd_b200 must not accept it as its native library."""
    code = "import torchmd_b200._lib as l; l.lib()"
    env = dict(os.environ, TMD_B200_LIB=os.path.join(SIMT_DIR, "libtmd_simt.so"), PYTHONPATH=ROOT)
    r = subprocess.run(["python", "-c", code], capture_output=True, text=True, env=env)
    assert r.returncode != 0 and "SIMT-interpreter build" in r.stderr


@pytest.mark.parametrize("world", [2, 3])
def test_peer_to_peer_exchange_between_ranks_in_one_process(simt, world):
    """Several contexts play the ranks of a decomposed run inside one process (the interpreter's IPC handles
    carry plain pointers): every rank pushes its owned atoms into all ranks' write buffers and flags them, then
    every rank waits, evaluates its owned forces and finishes the step.  Gathered positions and velocities must
    equal the single-context trajectory bit for bit (full neighbour rows: no force reduction needed)."""
    from torchmd_b200 import _lib
    from torchmd_b200.domain import SlabDecomposition

    g, t = dict(load_golden("water291_rf_switch")), load_golden("water291_traj")
    g["cfg_nrep"] = np.int64(1)
    masses = np.ascontiguousarray(g["par_masses"].astype(np.float32))
    dt = 1.0 / TIMEFACTOR
    gamma = 0.1 / (1000.0 / TIMEFACTOR)
    vcoeff = np.sqrt(2.0 * gamma / masses.astype(np.float64) * BOLTZMAN * 300.0 * dt).astype(np.float32)

    def fresh():
        c = Ctx(simt, g)
        c.vel = np.ascontiguousarray(t["vel0_f32"][:1]).copy()
        c.posw = c.pos.copy()
        c.F, _ = c.forces(pos=c.posw)
        c.masses, c.dt = masses, dt
        c.ene, c.ke = np.zeros((1, _lib.NUM_ENERGIES)), np.zeros(1)
        return c

    ref = fresh()
    ranks = [fresh() for _ in range(world)]
    n = ref.natoms
    handles = (C.c_ubyte * (64 * world))()
    for r, c in enumerate(ranks):
        dec = SlabDecomposition(n, world, r)
        c.lo, c.cnt = dec.lo, dec.count
        c.check(simt.tmd_set_owned_atoms(c.h, c.lo, c.cnt))
        c.F, _ = c.forces(pos=c.posw)  # owned forces of the start configuration
        h = (C.c_ubyte * 64)()
        c.check(simt.tmd_dd_create(c.h, r, world, h))
        handles[64 * r : 64 * (r + 1)] = list(h)
    for c in ranks:
        c.check(simt.tmd_dd_connect(c.h, handles))
    parity, nsteps = 0, 5
    md_steps(simt, ref, nsteps, gamma=gamma, vcoeff=vcoeff, seed=99)
    for c in ranks:
        c.check(simt.tmd_dd_load(c.h, parity, c.posw.ctypes.data, None))
    for it in range(nsteps):
        for c in ranks:  # phase 1 on every rank: integrate the owned atoms, push, flag
            c.check(simt.tmd_dd_vv_first_push(c.h, parity, c.vel.ctypes.data, c.F.ctypes.data, masses.ctypes.data, dt, None))
        for c in ranks:  # phase 2: every rank finds all flags of this step
            c.check(simt.tmd_dd_wait(c.h, None))
            c.check(simt.tmd_dd_forces(c.h, 1 - parity, c.F.ctypes.data, None, None))
            c.check(simt.tmd_vv_second(c.h, c.vel.ctypes.data, c.F.ctypes.data, masses.ctypes.data, dt, gamma, vcoeff.ctypes.data, None, 99, 0,
                                       None, None))
        parity ^= 1
    for c in ranks:
        c.check(simt.tmd_dd_store(c.h, parity, c.posw.ctypes.data, None))
        assert np.array_equal(c.posw, ref.posw), "every rank must hold all final positions"
        sl = slice(c.lo, c.lo + c.cnt)
        assert np.array_equal(c.vel[0, sl], ref.vel[0, sl]) and np.array_equal(c.F[0, sl], ref.F[0, sl])
        st = _lib.Stats()
        assert simt.tmd_get_stats(c.h, C.byref(st), None) == 0
    ref.close()
    for c in ranks:
        c.close()


def test_packed_kernel_and_culled_build_on_a_3000_atom_box(simt):
    """A generated 1000-water box (L = 31 A, 6x6x6 cells, default skin): culled build + packed fixed-point kernel
    against the oracle -- forces, energies and the bit-exact pair set."""
    from oracle import refmd
    from torchmd_b200 import testsystems

    sysd = testsystems.water_box(1000, seed=1)
    terms = ["lj", "electrostatics", "bonds", "angles"]
    cfg = dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    par64 = testsystems.water_parameters(sysd, precision=torch.float64)
    g = {"coords": sysd["coords"].astype(np.float32), "box": np.asarray(sysd["box"], np.float32), "cfg_nrep": np.int64(1),
         "cfg_cutoff": np.float64(9.0), "cfg_rfa": np.bool_(True), "cfg_switch_dist": np.float64(7.5), "terms": np.array(terms)}

    class C2(Ctx):
        def __init__(self, L, env):
            from torchmd_b200 import Forces

            self.L, self.g, self.terms, self.env = L, g, terms, dict(env)
            self.check = lambda rc: (_ for _ in ()).throw(RuntimeError(L.tmd_last_error().decode())) if rc else None
            self.f = Forces(testsystems.water_parameters(sysd, precision=torch.float32), terms=terms, **cfg)
            self.pos = np.ascontiguousarray(g["coords"][None])
            self.nrep, self.natoms = 1, self.pos.shape[1]
            self.box = np.ascontiguousarray(g["box"][None])
            self.h = C.c_void_p()
            self.check(L.tmd_create(C.byref(self.h), 0, self.natoms, 1))
            self.f._configure(L, self.h, self.check)
            self.check(L.tmd_set_box(self.h, self.box.ctypes.data))

    c = C2(simt, {"TMD_B200_FX": "2"})
    F, E = c.forces()
    assert simt.tmd_pair_kernel(c.h) == 2
    of = refmd.OracleForces(par64, terms, decision_dtype=torch.float32, **cfg)
    pos_t = torch.tensor(c.pos)
    box_t = torch.diag(torch.tensor(g["box"]))[None]
    f64 = torch.zeros(c.pos.shape, dtype=torch.float64)
    e_ref = of.compute(pos_t.double(), box_t.double(), f64)[0]
    err = np.abs(F.astype(np.float64) - f64.numpy()).max()
    assert err < 1e-4 * max(1.0, f64.abs().max().item() / 100.0), err
    for k in terms:
        assert abs(E[k][0] - float(e_ref[k])) <= 2e-5 * max(1.0, abs(float(e_ref[k]))) + 2e-3, k
    of32 = refmd.OracleForces(testsystems.water_parameters(sysd, precision=torch.float32), terms, **cfg)
    ref_pairs = of32.neighbour_pairs(pos_t[0], torch.tensor(g["box"])).numpy().astype(np.int32)
    os.environ["TMD_B200_FX"] = "2"
    try:
        assert np.array_equal(c.pairs(), ref_pairs)
    finally:
        os.environ.pop("TMD_B200_FX", None)
    c.close()


@pytest.fixture(scope="module")
def simt_smalltable():
    """A build whose staged-table limit is 2 atom types: the 10-type alanine dipeptide and the 4-type chain then
    take the packed kernels' global-table path (used for real with more than 16 types, e.g. thrombin's 45)."""
    return load(build_simt("_t2", ["FX_SMALLT_MAX_N=2"]))


@pytest.mark.parametrize("name,kernel", [("ala2_nobox_rf", 3), ("chain_amber_periodic", 2)])
def test_packed_kernels_with_the_table_in_global_memory(simt_smalltable, name, kernel):
    g = load_golden(name)
    assert len(np.unique(g["par_types"])) > 2
    c = Ctx(simt_smalltable, g, env={"TMD_B200_FX": "2"})
    F, E = c.forces()
    assert simt_smalltable.tmd_pair_kernel(c.h) == kernel
    check_against_golden(c, F, E)
    F2, _ = c.forces(energies=False)
    check_against_golden(c, F2, {})
    c.close()


# ---- edge cases of the list machinery (synthetic systems against the oracle) -------------------------------
def synthetic(natoms, coords, box, bonds=None, seed=0, sigma=3.4, eps=0.238):
    from torchmd_b200.parameters import TopologyParameters

    rng = np.random.default_rng(seed)
    kw = {}
    if bonds is not None and len(bonds):
        b = np.asarray(bonds, np.int64)
        kw["bonds"] = (b, np.stack([np.arange(len(b)), np.zeros(len(b), np.int64)], 1), np.array([[100.0, 1.5]]))

    def make(precision):
        return TopologyParameters(atom_types=np.zeros(natoms, np.int64), type_sigma=[sigma], type_epsilon=[eps],
                                  charges=np.linspace(-0.3, 0.3, natoms), masses=np.full(natoms, 12.0), precision=precision, **kw)

    return make, np.ascontiguousarray(coords, np.float32), np.asarray(box, np.float32)


class SynCtx(Ctx):
    def __init__(self, L, make, coords, box, terms, env=None, **cfg):
        from torchmd_b200 import Forces

        self.L, self.terms, self.env = L, terms, dict(env or {})
        self.check = lambda rc: (_ for _ in ()).throw(RuntimeError(L.tmd_last_error().decode())) if rc else None
        self.f = Forces(make(torch.float32), terms=terms, **cfg)
        self.pos = np.ascontiguousarray(coords[None])
        self.nrep, self.natoms = 1, coords.shape[0]
        self.box = np.ascontiguousarray(box[None])
        self.h = C.c_void_p()
        self.check(L.tmd_create(C.byref(self.h), 0, self.natoms, 1))
        self.f._configure(L, self.h, self.check)
        self.check(L.tmd_set_box(self.h, self.box.ctypes.data))


def oracle_check(c, make, coords, box, terms, cfg, F, tol=1e-4):
    from oracle import refmd

    of = refmd.OracleForces(make(torch.float64), terms, decision_dtype=torch.float32, **cfg)
    pos_t = torch.tensor(coords)[None]
    box_t = torch.diag(torch.tensor(box))[None]
    f64 = torch.zeros(pos_t.shape, dtype=torch.float64)
    of.compute(pos_t.double(), box_t.double(), f64)
    scale = max(1.0, f64.abs().max().item() / 100.0)
    assert np.abs(F.astype(np.float64) - f64.numpy()).max() < tol * scale
    of32 = refmd.OracleForces(make(torch.float32), terms, **cfg)
    return of32.neighbour_pairs(pos_t[0], torch.tensor(box)).numpy().astype(np.int32)


def test_row_overflow_grows_the_rows_and_recovers(simt):
    """200 atoms inside a 17 A ball of a 77 A box: the density-based row capacity (64) is far too small; the
    overflow protocol (flag -> TMD_ERR_OVERFLOW -> grown rows -> rebuild) must end in the right answer."""
    rng = np.random.default_rng(4)
    pts = []
    while len(pts) < 200:  # min distance 2.2 A inside the ball
        p = rng.uniform(-8.5, 8.5, 3)
        if np.linalg.norm(p) < 8.5 and (not pts or np.min(np.linalg.norm(np.array(pts) - p, axis=1)) > 2.2):
            pts.append(p)
    coords = np.array(pts) + 38.0
    make, coords, box = synthetic(200, coords, [77.0, 77.0, 77.0])
    terms, cfg = ["lj", "electrostatics"], dict(cutoff=9.0, rfa=True, switch_dist=7.5)
    for env in ({}, {"TMD_B200_FX": "2"}):
        c = SynCtx(simt, make, coords, box, terms, env=env, **cfg)
        F, E = c.forces()
        assert c.stats.row_capacity >= c.stats.max_neighbours > 64 and not c.stats.overflow
        # (atoms 2.2 A apart with sigma 3.4: |F| ~ 1000 from ~200 large terms of both signs -- fp32 summation error)
        ref_pairs = oracle_check(c, make, coords, box, terms, cfg, F, tol=3e-4)
        os.environ.update(env)
        try:
            assert np.array_equal(c.pairs(), ref_pairs)
        finally:
            for k in env:
                os.environ.pop(k, None)
        c.close()


def test_more_than_32_exclusions_per_atom(simt):
    """A hub atom bonded to 40 others (its exclusion list no longer fits one per lane)."""
    rng = np.random.default_rng(5)
    n = 120
    coords = rng.uniform(2.0, 22.0, (n, 3))
    hub = 7
    leaves = [i for i in range(n) if i != hub][:40]
    for k, i in enumerate(leaves):  # put the bonded atoms around the hub
        d = rng.normal(size=3)
        coords[i] = coords[hub] + 1.5 * d / np.linalg.norm(d) + 0.05 * k * np.array([1, 0, 0])
    bonds = [(hub, i) for i in leaves]
    make, coords, box = synthetic(n, coords, [24.0, 24.0, 24.0], bonds=bonds)
    terms, cfg = ["lj", "electrostatics", "bonds"], dict(cutoff=5.0, rfa=True, switch_dist=4.0)
    c = SynCtx(simt, make, coords, box, terms, skin=0.4, **cfg)
    F, E = c.forces()
    ref_pairs = oracle_check(c, make, coords, box, terms, cfg, F, tol=2e-4)
    got = c.pairs()
    assert np.array_equal(got, ref_pairs)
    assert not any((min(hub, i), max(hub, i)) in set(map(tuple, got.tolist())) for i in leaves)
    c.close()


def test_tiny_systems(simt):
    for n in (1, 2, 3):
        coords = np.array([[1.0, 1.0, 1.0], [3.5, 1.2, 0.8], [2.0, 4.0, 1.0]])[:n]
        make, coords, box = synthetic(n, coords, [30.0, 30.0, 30.0])
        terms, cfg = ["lj", "electrostatics"], dict(cutoff=9.0, rfa=True, switch_dist=7.5)
        for env in ({}, {"TMD_B200_FX": "1"}, {"TMD_B200_FX": "2"}):
            c = SynCtx(simt, make, coords, box, terms, env=env, **cfg)
            F, E = c.forces()
            if n == 1:
                assert np.array_equal(F, np.zeros_like(F))
            else:
                oracle_check(c, make, coords, box, terms, cfg, F)
            c.close()

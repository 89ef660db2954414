"""Which pair kernel each force call runs, on every row of the choice (tmd_b200.cu, pair_kernel_of): fp32 and fp64, with
and without particle-mesh Ewald, under TMD_B200_FX 0/1/2 and TMD_B200_CLUSTER 0/1, on an open system, on periodic boxes
with and without the guard-free minimum image, and on a box large enough for the cluster lists.  Each context makes a
call with energies and one without in the explicit convention, the same in the exact-gradient convention, and again
in the explicit one, switching the convention on the same context.  On the GPU each call's pair kernel is checked down
to its template arguments (the demangled name torch.profiler reports), because a wrong flag there can still give the
right forces.  tests/test_pair_dispatch_on_interpreter.py checks the ids on the host interpreter build.
"""
import re

import pytest
import torch

import test_gpu_force_convention as FC
from torchmd_b200._lib import (PAIR_CLUSTER, PAIR_EWALD, PAIR_EWALD_CLUSTER, PAIR_EWALD_F64, PAIR_EWALD_FX,
                               PAIR_EWALD_FX2, PAIR_F64, PAIR_OPEN_FX2, PAIR_ROWS, PAIR_ROWS_FX, PAIR_ROWS_FX2)

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"

# (exact-gradient convention, energies) of the calls each context makes, in order
CALLS = [(False, True), (False, False), (True, True), (True, False), (False, True), (False, False)]

# (case, system, precision, PME, TMD_B200_FX, TMD_B200_CLUSTER): (id of an explicit call, its kernel, id of an
# exact-gradient call, its kernel); E stands for the energies flag of the call.  The systems: ala2_nobox_rf has no box;
# chain_amber_periodic (30 A box, cutoff 9) has the guard-free image and is too small for the cluster lists;
# chain_plain is it with plain cut-off Coulomb; chain_unsafe is it with a 2.5 A skin, which breaks the guard-free image;
# water_x2 is the 2x2x2 tiled water box (43 A, cutoff 5) on the cluster lists.  Every system has at most 16 atom types.
CASES = {c[0]: (c[1:], want) for c, want in {
    ("ala2_nobox_rf-f32-fx0-cl0", "ala2_nobox_rf", 32, False, 0, 0): (PAIR_ROWS, "k_pair<E, false, false, 1>", PAIR_ROWS, "k_pair<E, false, false, 0>"),
    ("ala2_nobox_rf-f32-fx0-cl1", "ala2_nobox_rf", 32, False, 0, 1): (PAIR_CLUSTER, "k_cpair<E, false>", PAIR_CLUSTER, "k_cpair_grad<E, false>"),
    ("ala2_nobox_rf-f32-fx1-cl0", "ala2_nobox_rf", 32, False, 1, 0): (PAIR_ROWS, "k_pair<E, false, false, 1>", PAIR_ROWS, "k_pair<E, false, false, 0>"),
    ("ala2_nobox_rf-f32-fx1-cl1", "ala2_nobox_rf", 32, False, 1, 1): (PAIR_CLUSTER, "k_cpair<E, false>", PAIR_CLUSTER, "k_cpair_grad<E, false>"),
    ("ala2_nobox_rf-f32-fx2-cl0", "ala2_nobox_rf", 32, False, 2, 0): (PAIR_OPEN_FX2, "k_pair2_open<E, true>", PAIR_ROWS, "k_pair<E, false, false, 0>"),
    ("ala2_nobox_rf-f32-fx2-cl1", "ala2_nobox_rf", 32, False, 2, 1): (PAIR_CLUSTER, "k_cpair<E, false>", PAIR_CLUSTER, "k_cpair_grad<E, false>"),
    ("ala2_nobox_rf-f64", "ala2_nobox_rf", 64, False, None, None): (PAIR_F64, "k_pair_f64<E, false>", PAIR_F64, "k_pair_f64<E, false>"),
    ("chain_amber_periodic-f32-fx0-cl0", "chain_amber_periodic", 32, False, 0, 0): (PAIR_ROWS, "k_pair<E, true, true, 1>", PAIR_ROWS, "k_pair<E, true, true, 0>"),
    ("chain_amber_periodic-f32-fx0-cl1", "chain_amber_periodic", 32, False, 0, 1): (PAIR_ROWS, "k_pair<E, true, true, 1>", PAIR_ROWS, "k_pair<E, true, true, 0>"),
    ("chain_amber_periodic-f32-fx1-cl0", "chain_amber_periodic", 32, False, 1, 0): (PAIR_ROWS_FX, "k_pair_fx<E, 1, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_amber_periodic-f32-fx1-cl1", "chain_amber_periodic", 32, False, 1, 1): (PAIR_ROWS_FX, "k_pair_fx<E, 1, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_amber_periodic-f32-fx2-cl0", "chain_amber_periodic", 32, False, 2, 0): (PAIR_ROWS_FX2, "k_pair_fx2<E, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_amber_periodic-f32-fx2-cl1", "chain_amber_periodic", 32, False, 2, 1): (PAIR_ROWS_FX2, "k_pair_fx2<E, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_amber_periodic-f64", "chain_amber_periodic", 64, False, None, None): (PAIR_F64, "k_pair_f64<E, true>", PAIR_F64, "k_pair_f64<E, true>"),
    ("chain_amber_periodic-f32-pme-fx0-cl0", "chain_amber_periodic", 32, True, 0, 0): (PAIR_EWALD, "k_pair<E, true, true, 2>", PAIR_EWALD, "k_pair<E, true, true, 2>"),
    ("chain_amber_periodic-f32-pme-fx0-cl1", "chain_amber_periodic", 32, True, 0, 1): (PAIR_EWALD, "k_pair<E, true, true, 2>", PAIR_EWALD, "k_pair<E, true, true, 2>"),
    ("chain_amber_periodic-f32-pme-fx1-cl0", "chain_amber_periodic", 32, True, 1, 0): (PAIR_EWALD_FX, "k_pair_fx<E, 2, true>", PAIR_EWALD_FX, "k_pair_fx<E, 2, true>"),
    ("chain_amber_periodic-f32-pme-fx1-cl1", "chain_amber_periodic", 32, True, 1, 1): (PAIR_EWALD_FX, "k_pair_fx<E, 2, true>", PAIR_EWALD_FX, "k_pair_fx<E, 2, true>"),
    ("chain_amber_periodic-f32-pme-fx2-cl0", "chain_amber_periodic", 32, True, 2, 0): (PAIR_EWALD_FX2, "k_pair_fx2_ew<E, true>", PAIR_EWALD_FX, "k_pair_fx<E, 2, true>"),
    ("chain_amber_periodic-f32-pme-fx2-cl1", "chain_amber_periodic", 32, True, 2, 1): (PAIR_EWALD_FX2, "k_pair_fx2_ew<E, true>", PAIR_EWALD_FX, "k_pair_fx<E, 2, true>"),
    ("chain_amber_periodic-f64-pme", "chain_amber_periodic", 64, True, None, None): (PAIR_EWALD_F64, "k_ewpair64<E>", PAIR_EWALD_F64, "k_ewpair64<E>"),
    ("chain_plain-f32-fx0-cl0", "chain_plain", 32, False, 0, 0): (PAIR_ROWS, "k_pair<E, true, true, 0>", PAIR_ROWS, "k_pair<E, true, true, 0>"),
    ("chain_plain-f32-fx0-cl1", "chain_plain", 32, False, 0, 1): (PAIR_ROWS, "k_pair<E, true, true, 0>", PAIR_ROWS, "k_pair<E, true, true, 0>"),
    ("chain_plain-f32-fx1-cl0", "chain_plain", 32, False, 1, 0): (PAIR_ROWS_FX, "k_pair_fx<E, 0, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_plain-f32-fx1-cl1", "chain_plain", 32, False, 1, 1): (PAIR_ROWS_FX, "k_pair_fx<E, 0, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_plain-f32-fx2-cl0", "chain_plain", 32, False, 2, 0): (PAIR_ROWS_FX2, "k_pair_fx2<E, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_plain-f32-fx2-cl1", "chain_plain", 32, False, 2, 1): (PAIR_ROWS_FX2, "k_pair_fx2<E, true>", PAIR_ROWS_FX, "k_pair_fx<E, 0, true>"),
    ("chain_plain-f64", "chain_plain", 64, False, None, None): (PAIR_F64, "k_pair_f64<E, true>", PAIR_F64, "k_pair_f64<E, true>"),
    ("chain_unsafe-f32-fx0-cl0", "chain_unsafe", 32, False, 0, 0): (PAIR_ROWS, "k_pair<E, true, false, 1>", PAIR_ROWS, "k_pair<E, true, false, 0>"),
    ("chain_unsafe-f32-fx0-cl1", "chain_unsafe", 32, False, 0, 1): (PAIR_ROWS, "k_pair<E, true, false, 1>", PAIR_ROWS, "k_pair<E, true, false, 0>"),
    ("chain_unsafe-f32-fx1-cl0", "chain_unsafe", 32, False, 1, 0): (PAIR_ROWS, "k_pair<E, true, false, 1>", PAIR_ROWS, "k_pair<E, true, false, 0>"),
    ("chain_unsafe-f32-fx1-cl1", "chain_unsafe", 32, False, 1, 1): (PAIR_ROWS, "k_pair<E, true, false, 1>", PAIR_ROWS, "k_pair<E, true, false, 0>"),
    ("chain_unsafe-f32-fx2-cl0", "chain_unsafe", 32, False, 2, 0): (PAIR_ROWS, "k_pair<E, true, false, 1>", PAIR_ROWS, "k_pair<E, true, false, 0>"),
    ("chain_unsafe-f32-fx2-cl1", "chain_unsafe", 32, False, 2, 1): (PAIR_ROWS, "k_pair<E, true, false, 1>", PAIR_ROWS, "k_pair<E, true, false, 0>"),
    ("chain_unsafe-f64", "chain_unsafe", 64, False, None, None): (PAIR_F64, "k_pair_f64<E, true>", PAIR_F64, "k_pair_f64<E, true>"),
    ("chain_unsafe-f32-pme-fx0-cl0", "chain_unsafe", 32, True, 0, 0): (PAIR_EWALD, "k_pair<E, true, false, 2>", PAIR_EWALD, "k_pair<E, true, false, 2>"),
    ("chain_unsafe-f32-pme-fx0-cl1", "chain_unsafe", 32, True, 0, 1): (PAIR_EWALD, "k_pair<E, true, false, 2>", PAIR_EWALD, "k_pair<E, true, false, 2>"),
    ("chain_unsafe-f32-pme-fx1-cl0", "chain_unsafe", 32, True, 1, 0): (PAIR_EWALD, "k_pair<E, true, false, 2>", PAIR_EWALD, "k_pair<E, true, false, 2>"),
    ("chain_unsafe-f32-pme-fx1-cl1", "chain_unsafe", 32, True, 1, 1): (PAIR_EWALD, "k_pair<E, true, false, 2>", PAIR_EWALD, "k_pair<E, true, false, 2>"),
    ("chain_unsafe-f32-pme-fx2-cl0", "chain_unsafe", 32, True, 2, 0): (PAIR_EWALD, "k_pair<E, true, false, 2>", PAIR_EWALD, "k_pair<E, true, false, 2>"),
    ("chain_unsafe-f32-pme-fx2-cl1", "chain_unsafe", 32, True, 2, 1): (PAIR_EWALD, "k_pair<E, true, false, 2>", PAIR_EWALD, "k_pair<E, true, false, 2>"),
    ("chain_unsafe-f64-pme", "chain_unsafe", 64, True, None, None): (PAIR_EWALD_F64, "k_ewpair64<E>", PAIR_EWALD_F64, "k_ewpair64<E>"),
    ("water_x2-f32-fx2-cl1", "water_x2", 32, False, 2, 1): (PAIR_CLUSTER, "k_cpair<E, true>", PAIR_CLUSTER, "k_cpair_grad<E, true>"),
    ("water_x2-f32-pme-fx2-cl1", "water_x2", 32, True, 2, 1): (PAIR_EWALD_CLUSTER, "k_cpair_ew<E>", PAIR_EWALD_CLUSTER, "k_cpair_ew_grad<E>"),
}.items()}


def system(key):
    if key == "chain_unsafe":  # cutoff + 2 skin >= 0.45 L: the full-row kernels keep the guarded minimum image
        spec = FC.system_of("chain_amber_periodic")
        spec["cfg"]["skin"] = 2.5
        return spec
    return FC.system_of(key)


def run_calls(case, monkeypatch):
    """Sets the case up on one Forces and makes the calls of CALLS on its context through the C ABI; returns the
    tmd_pair_kernel id after each call and a function that repeats the calls."""
    from torchmd_b200 import Forces, _lib

    (key, bits, pme, fx, cluster), _ = CASES[case]
    for name, value in (("TMD_B200_FX", fx), ("TMD_B200_CLUSTER", cluster)):
        if value is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(value))
    spec = system(key)
    dtype = torch.float64 if bits == 64 else torch.float32
    cfg = dict(spec["cfg"])
    if pme:
        cfg.pop("rfa", None)
    pos = torch.tensor(spec["coords"][None], dtype=dtype, device=FC.DEV)
    box = torch.diag_embed(torch.tensor(spec["box"][None], dtype=dtype, device=FC.DEV))
    forces = Forces(FC.G.params(spec, dtype, FC.DEV), terms=spec["terms"], pme=pme, **cfg)
    F = torch.zeros_like(pos)
    forces.compute(pos, box, F)  # finalises the context (and grows its lists if they overflow)
    L, ctx = _lib.lib(), forces._ctx
    fn = L.tmd_forces_f64 if bits == 64 else L.tmd_forces
    ene = torch.zeros((1, _lib.NUM_ENERGIES), dtype=torch.float64, device=FC.DEV)
    stream = torch.cuda.current_stream(pos.device).cuda_stream

    def calls():
        ids = []
        for exact, energies in CALLS:
            _lib.check(L.tmd_set_force_convention(ctx, int(exact)))
            _lib.check(fn(ctx, pos.data_ptr(), F.data_ptr(), ene.data_ptr() if energies else None, stream))
            ids.append(L.tmd_pair_kernel(ctx))
        return ids

    return calls(), calls, forces


def expected(case):
    _, (k_explicit, n_explicit, k_exact, n_exact) = CASES[case]
    ids = [k_exact if exact else k_explicit for exact, _ in CALLS]
    names = [(n_exact if exact else n_explicit).replace("E", "true" if e else "false", 1) for exact, e in CALLS]
    return ids, names


PAIR_KERNEL = re.compile(r"(?<!\w)(k_c?pair\w*|k_ewpair64)<[^>]*>")


@pytest.mark.parametrize("case", list(CASES))
def test_pair_kernel_of_every_call(case, monkeypatch):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    want_ids, want_names = expected(case)
    ids, calls, forces = run_calls(case, monkeypatch)
    assert ids == want_ids, (case, ids)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        assert calls() == want_ids
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)
    names = [m.group(0) for m in (PAIR_KERNEL.search(e.name) for e in kernels) if m]
    assert names == want_names, (case, names)

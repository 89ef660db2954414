#!/usr/bin/env python
"""Run the kernel sources in the SIMT interpreter of tests/simt under AddressSanitizer (no GPU involved).

    python scripts/asan_interpreter.py            # builds tests/simt/libtmd_simt_asan.so, re-executes under libasan

Device memory is host memory in that build, so an out-of-bounds index in a kernel (global or shared) is an ASan
report and a non-zero exit.  Covers the default, fixed-point, packed and no-box pair kernels, the list build,
row overflow and regrowth, >32 exclusions, the wrap kernel, fused MD steps, the bonded overlap, the exact-gradient
convention, owned-atom ranges, the in-process peer-to-peer exchange with three ranks, and (cluster_cases) the cluster
half-list path.  Takes about half an hour.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)


def main():
    import test_simt_kernels as T
    from conftest import load_golden

    L = T.load(T.build_simt("_asan", ["TMD_SIMT_ASAN=1"]))
    for name, env, kw in (
        ("chain_amber_periodic", {"TMD_B200_FX": "2"}, {}),
        ("water291_rf_switch", {}, {}),
        ("ala2_nobox_rf", {"TMD_B200_FX": "2"}, {}),
        ("water999_eq", {"TMD_B200_FX": "1"}, {"skin": 0.2}),
    ):
        c = T.Ctx(L, load_golden(name), env=env, **kw)
        F, E = c.forces()
        T.check_against_golden(c, F, E)
        c.forces(energies=False)
        c.pairs()
        print(f"{name}: pair kernel {L.tmd_pair_kernel(c.h)} clean", flush=True)
        c.close()
    T.test_peer_to_peer_exchange_between_ranks_in_one_process(L, 3)
    for n in ("water", "mixed", "nobonds", "zerobox"):
        T.test_wrap_kernel(L, n)
    T.test_fused_md_steps_follow_the_reference_trajectories(L)
    T.test_row_overflow_grows_the_rows_and_recovers(L)
    T.test_more_than_32_exclusions_per_atom(L)
    T.test_bonded_overlap_is_bit_identical(L)
    T.test_exact_gradient_convention(L)
    T.test_owned_atom_range_forces_match_the_full_evaluation(L, "packed")
    T.test_tiny_systems(L)
    cluster_cases()
    print("asan: no report")


def cluster_cases():
    """The cluster half-list path under ASan: the tests of tests/test_simt_cluster.py on an ASan build with the
    cluster path as the default -- list build and pair kernel in a periodic box (atoms thrown boxes away), band pairs,
    systems without a box, capacity growth and the fall-back, fused MD steps with the step boundary kernel (issued
    eagerly and as captured steps), the term-parallel bonded kernels, owned-atom ranges."""
    import torch
    from _pytest.monkeypatch import MonkeyPatch

    import test_simt_cluster as TC
    import test_simt_kernels as T
    from torchmd_b200 import _lib

    lib = T.load(T.build_simt("_asan_cl", list(T.VARIANTS["_cl"]) + ["TMD_SIMT_ASAN=1"]))

    class _Stream:
        cuda_stream = None

    mp = MonkeyPatch()
    try:
        mp.setattr(_lib, "_lib", lib)
        mp.setattr(_lib, "on_device", lambda t: True)
        mp.setattr(torch.cuda, "current_stream", lambda *a, **k: _Stream())
        mp.setattr(torch.cuda, "current_device", lambda: 0)
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        for thrown in (0, 3):
            TC.test_cluster_path_periodic_water(lib, thrown)
        print("cluster: periodic water clean", flush=True)
        TC.test_cluster_exact_pass_decides_band_pairs(lib)
        for name in ("ala2_nobox_rf", "thrombin_nobox_rf"):
            TC.test_cluster_path_without_a_box(lib, name)
        print("cluster: band pairs, no-box systems clean", flush=True)
        def with_env(fn, *args):  # the tests set environment switches through their monkeypatch fixture: undo per test
            env = MonkeyPatch()
            try:
                fn(lib, env, *args)
            finally:
                env.undo()

        with_env(TC.test_cluster_list_capacity_grows_and_lattice_falls_back)
        with_env(TC.test_cluster_md_steps_follow_the_full_list_trajectory)
        for graph in ("0", "1"):
            with_env(TC.test_step_boundary_kernel_reproduces_the_two_kernel_sequence, graph)
        print("cluster: capacity growth, MD steps, step boundary clean", flush=True)
        TC.test_cluster_path_with_owned_atom_ranges(lib)
        print("cluster: owned ranges clean", flush=True)
    finally:
        mp.undo()


if __name__ == "__main__":
    if os.environ.get("TMD_ASAN_CHILD") != "1":
        asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True, check=True).stdout.strip()
        env = dict(os.environ, TMD_ASAN_CHILD="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
        sys.exit(subprocess.run([sys.executable, os.path.abspath(__file__)], env=env).returncode)
    main()

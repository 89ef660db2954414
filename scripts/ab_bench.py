"""A/B timing of library variants in ONE process (one system generation, one torch start-up): for tuning sweeps where
bench.py's full contract (JSON line, end-to-end loop, CPU baseline, clock sampling) per variant would waste box time.

    python scripts/ab_bench.py --steps 1000 "default" "FX=2|TMD_B200_FX=2" "other+FX=2|TMD_B200_FX=2|/tmp/var/libtmd_b200.so"

A variant is "label|ENV=VALUE,ENV=VALUE|library path" (the last two optional); the pseudo-variable SKIN=<A> sets the
Verlet skin of that variant.  Every variant starts from the same
equilibrated state and runs the same number of steps with the same noise seed; prints steps/s, ms/step, the mean
pair-kernel time, launches per step and the final temperature.  The numbers to publish come from bench.py.
"""
import argparse
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEVICE = None  # tests/test_mirrors_on_interpreter.py dry-runs main() on the host interpreter build with "cpu"


def main(argv=None):
    import torch

    import bench as B
    from torchmd_b200 import Forces, Integrator, System, _lib, maxwell_boltzmann, testsystems

    ap = argparse.ArgumentParser()
    ap.add_argument("variants", nargs="+")
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--equil", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--skin", type=float, default=None)
    args = ap.parse_args(argv)
    dev = DEVICE or "cuda:0"

    sysd = testsystems.water_box(B.N_WATERS, seed=0)
    n = len(sysd["coords"])
    par = testsystems.water_parameters(sysd, device=dev)
    default_lib = _lib.LIB_PATH

    def fresh(variant_env):
        variant_env = dict(variant_env)
        skin = float(variant_env.pop("SKIN")) if "SKIN" in variant_env else args.skin
        system = System(n, 1, torch.float32, dev)
        system.set_positions(sysd["coords"])
        system.set_box(sysd["box"])
        torch.manual_seed(1)
        system.set_velocities(maxwell_boltzmann(par.masses, B.TEMPERATURE, 1))
        old = {k: os.environ.get(k) for k in variant_env}
        os.environ.update(variant_env)
        try:  # the switches are read when the context is finalised: at the first force call
            forces = Forces(par, terms=B.TERMS, skin=skin, **B.CFG)
            forces.compute(system.pos, system.box, system.forces)
        finally:
            for k, v in old.items():
                os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
        return system, forces

    print("%-44s %9s %9s %9s %8s %7s" % ("variant", "steps/s", "ms/step", "pair ms", "launches", "T [K]"), flush=True)
    for spec in args.variants:
        f = spec.split("|")
        label = f[0]
        env = dict(kv.split("=", 1) for kv in f[1].split(",") if kv) if len(f) > 1 else {}
        lib = f[2] if len(f) > 2 and f[2] else default_lib
        if DEVICE is None and lib != _lib.LIB_PATH:
            _lib.LIB_PATH, _lib._lib = lib, None  # another build of the library in the same process
        try:
            system, forces = fresh(env)
            eq = Integrator(system, forces, B.TIMESTEP_FS, dev, gamma=10.0, T=B.TEMPERATURE)
            torch.manual_seed(2)
            eq.step(niter=args.equil)
            integ = Integrator(system, forces, B.TIMESTEP_FS, dev, gamma=B.GAMMA_PS, T=B.TEMPERATURE)
            integ.seed = 12345
            integ.step(niter=args.warmup)
            L = _lib.lib()
            stream = torch.cuda.current_stream().cuda_stream
            st0 = forces.stats()
            torch.cuda.synchronize()
            _lib.check(L.tmd_profile_begin(forces._ctx, args.steps))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ekin, pot, T = integ.step(niter=args.steps)
            e1.record()
            torch.cuda.synchronize()
            pair_ms, pair_n = C.c_double(), C.c_int()
            _lib.check(L.tmd_profile_end(forces._ctx, C.byref(pair_ms), C.byref(pair_n), stream))
            st1 = forces.stats()
            ms = e0.elapsed_time(e1) / args.steps
            print("%-44s %9.0f %9.4f %9.4f %8.1f %7.1f   [pair kernel %d, %d rebuilds]" % (
                label, 1e3 / ms, ms, pair_ms.value / max(1, pair_n.value), (st1["kernel_launches"] - st0["kernel_launches"]) / args.steps,
                float(T[0]), L.tmd_pair_kernel(forces._ctx), st1["rebuilds"] - st0["rebuilds"]), flush=True)
            # the context goes with the library build that made it (the next variant may load another build)
            L.tmd_destroy(forces._ctx)
            forces._ctx = None
            del integ, eq, forces, system
        except Exception as err:  # one broken variant must not cost the others their measurement
            print("%-44s failed: %s" % (label, err), flush=True)


if __name__ == "__main__":
    main()

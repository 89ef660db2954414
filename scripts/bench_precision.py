"""Device-resident MD steps/s of "precision: double" against fp32, on water10k and water100k (BASELINE config 4
settings: LJ with switch 7.5 + reaction-field electrostatics, cutoff 9 A, flexible bonds and angles, Langevin 300 K,
gamma 0.1/ps, dt 1 fs, one replica), for three runs of the same start state:

  fp64           Forces / Integrator on float64 state (full neighbour rows, k_pair_f64)
  fp32_rows      float32 state on the full rows (TMD_B200_CLUSTER=0)
  fp32_default   float32 state with the default pair path

and the time of the fp64 and fp32 full-row pair kernels alone (CUDA events, tmd_profile_*).  The start state is the
lattice start relaxed on the fp32 full rows, so every run starts from the same bits.  Prints one JSON line.

  python scripts/bench_precision.py [--steps K] [--warmup W] [--workloads water10k,water100k]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--relax", type=int, default=1000, help="fp32 full-row steps that relax the lattice start")
    ap.add_argument("--workloads", default="water10k,water100k")
    ap.add_argument("--profile-steps", type=int, default=50)
    args = ap.parse_args()

    import torch

    import bench
    from torchmd_b200 import Forces, Integrator, System, _lib, maxwell_boltzmann

    dev = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_precision.py measures on a CUDA device; none found")

    def run(name, coords, vel, box, dtype, cluster, steps, warmup, profile=0):
        os.environ["TMD_B200_CLUSTER"] = "1" if cluster else "0"
        par, _, _, terms, cfg, nrep, _ = bench.build_workload(name, dev, precision=dtype)
        forces = Forces(par, terms=terms, **cfg)
        system = System(coords.shape[0], 1, dtype, dev)
        system.set_positions(coords)
        system.set_box(box)
        system.set_velocities(vel.to(dtype))
        forces.compute(system.pos, system.box, system.forces)
        torch.manual_seed(0)
        integ = Integrator(system, forces, 1.0, dev, gamma=0.1, T=300.0)
        if warmup:
            integ.step(niter=warmup)
        torch.cuda.synchronize()
        rate = None
        if steps:
            t0 = time.perf_counter()
            integ.step(niter=steps)
            torch.cuda.synchronize()
            rate = steps / (time.perf_counter() - t0)
        pair_ms = None
        if profile:
            L = _lib.lib()
            ctx = forces._ctx
            _lib.check(L.tmd_profile_begin(ctx, profile))
            integ.step(niter=profile)
            tot, n = C.c_double(), C.c_int()
            _lib.check(L.tmd_profile_end(ctx, C.byref(tot), C.byref(n), torch.cuda.current_stream().cuda_stream))
            pair_ms = tot.value / max(1, n.value)
        return system, rate, pair_ms, _lib.lib().tmd_pair_kernel(forces._ctx)

    result = {"metric": "MD steps/s, device resident, fp64 vs fp32", "gpu": gpu_info(), "steps": args.steps,
              "warmup": args.warmup, "workloads": {}}
    sampler = bench.ClockSampler(0)
    for name in args.workloads.split(","):
        _, coords, box, *_ = bench.build_workload(name, "cpu")
        torch.manual_seed(1)
        par, *_ = bench.build_workload(name, "cpu")
        vel0 = maxwell_boltzmann(par.masses.float(), 300.0, 1)
        relaxed, _, _, _ = run(name, coords, vel0, box, torch.float32, False, 0, args.relax)
        start = relaxed.pos[0].cpu().numpy()
        vel = relaxed.vel.cpu()
        del relaxed
        row = {"natoms": int(coords.shape[0])}
        for label, dtype, cluster in (("fp64", torch.float64, False), ("fp32_rows", torch.float32, False),
                                      ("fp32_default", torch.float32, True)):
            prof = args.profile_steps if label != "fp32_default" else 0
            _, rate, pair_ms, kernel = run(name, start, vel, box, dtype, cluster, args.steps, args.warmup, prof)
            row[label] = {"steps_per_s": round(rate, 1), "pair_kernel": kernel}
            if pair_ms is not None:
                row[label]["pair_kernel_ms"] = round(pair_ms, 4)
            torch.cuda.empty_cache()
        row["fp64_over_fp32_rows_time"] = round(row["fp32_rows"]["steps_per_s"] / row["fp64"]["steps_per_s"], 2)
        result["workloads"][name] = row
    result["clocks"] = sampler.stop()
    print(json.dumps(result))


if __name__ == "__main__":
    main()

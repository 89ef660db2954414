"""Particle-mesh Ewald against the reaction field: rigid water (Constraints(kind="water")) at 2 fs with Langevin (300 K,
gamma 0.1/ps), LJ with switch 7.5 A, cutoff 9 A, bonds and angles, one replica, default pair path, on water10k and
water100k in fp32 and on water10k in fp64.  The arms differ only in the electrostatics: rfa=True against pme=True at
the default tolerance 5e-4.  Every run starts from the same lattice start relaxed on the fp32 full rows.  Reports
steps/s, simulated ns/day, kernel launches and list rebuilds per step, alpha and the grid, the device time of each
PME kernel (torch.profiler over eager force calls, a separate pass), with the card's name, power limit and clocks read
in the same call, as one JSON line.

  python scripts/bench_pme.py [--steps K] [--warmup W] [--workloads water10k,water100k] [--f64-workloads water10k]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

PME_KERNELS = ("k_pme_spread", "k_pme_fft", "k_pme_gather")


def kernel_times(forces, system, calls):
    """Mean device time per force call of each PME kernel (and of the pair kernel) over eager force calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        forces.compute(system.pos, system.box, system.forces)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            forces.compute(system.pos, system.box, system.forces)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        label = next((k for k in PME_KERNELS if k in name), None)
        if label is None and ("k_pair" in name or "k_cpair" in name or "k_ewpair64" in name):
            label = "pair_kernel"
        if label is None:
            continue
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        out[label] = round(out.get(label, 0.0) + t / calls, 2)  # microseconds per force call (summed over launches)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--relax", type=int, default=1000, help="fp32 full-row steps at 1 fs that relax the lattice start")
    ap.add_argument("--workloads", default="water10k,water100k")
    ap.add_argument("--f64-workloads", default="water10k")
    ap.add_argument("--profile-calls", type=int, default=50)
    args = ap.parse_args()

    import torch

    import bench
    from bench_precision import gpu_info
    from torchmd_b200 import Constraints, Forces, Integrator, System, maxwell_boltzmann

    dev = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_pme.py measures on a CUDA device; none found")

    def run(name, coords, vel, box, dt_fs, pme, steps, warmup, dtype=torch.float32, rigid=True, cluster=True, profile=False):
        os.environ["TMD_B200_CLUSTER"] = "1" if cluster else "0"
        par, _, _, terms, cfg, _, _ = bench.build_workload(name, dev, precision=dtype)
        if pme:
            cfg = dict(cfg, rfa=False)
        forces = Forces(par, terms=terms, pme=pme, **cfg)
        system = System(coords.shape[0], 1, dtype, dev)
        system.set_positions(coords)
        system.set_box(box)
        system.set_velocities(vel.to(dtype))
        forces.compute(system.pos, system.box, system.forces)
        torch.manual_seed(0)
        integ = Integrator(system, forces, dt_fs, dev, gamma=0.1, T=300.0, constraints=Constraints(par, "water") if rigid else None)
        if warmup:
            integ.step(niter=warmup)
        torch.cuda.synchronize()
        if not steps:
            return system, None
        st0 = forces.stats()
        t0 = time.perf_counter()
        _, _, T = integ.step(niter=steps)
        torch.cuda.synchronize()
        rate = steps / (time.perf_counter() - t0)
        st1 = forces.stats()
        row = {"steps_per_s": round(rate, 1), "ns_per_day": round(rate * dt_fs * 1e-6 * 86400, 2),
               "kernel_launches_per_step": (st1["kernel_launches"] - st0["kernel_launches"]) / steps,
               "rebuilds_per_step": round((st1["rebuilds"] - st0["rebuilds"]) / steps, 4), "T_end": round(float(T[0]), 1)}
        if pme:
            alpha, grid = forces.pme_parameters()
            row["alpha"] = round(alpha, 6)
            row["grid"] = list(grid)
        if profile:
            row["kernel_us_per_call"] = kernel_times(forces, system, args.profile_calls)
        return system, row

    result = {"metric": "rigid water 2 fs + Langevin: reaction field vs particle-mesh Ewald (tolerance 5e-4)",
              "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "workloads": {}}
    f64 = set(w for w in args.f64_workloads.split(",") if w)
    for name in args.workloads.split(","):
        _, coords, box, *_ = bench.build_workload(name, "cpu")
        torch.manual_seed(1)
        par, *_ = bench.build_workload(name, "cpu")
        vel0 = maxwell_boltzmann(par.masses.float(), 300.0, 1)
        relaxed, _ = run(name, coords, vel0, box, 1.0, False, 0, args.relax, rigid=False, cluster=False)
        start, vel = relaxed.pos[0].cpu().numpy(), relaxed.vel.cpu()
        del relaxed
        row = {"natoms": int(coords.shape[0])}
        precisions = [("fp32", torch.float32)] + ([("fp64", torch.float64)] if name in f64 else [])
        for plabel, dtype in precisions:
            steps = args.steps if dtype == torch.float32 else max(args.steps // 4, 1)
            for label, pme in (("reaction_field", False), ("pme", True)):
                row[f"{plabel}_{label}"] = run(name, start, vel, box, 2.0, pme, steps, args.warmup, dtype=dtype, profile=pme)[1]
                torch.cuda.empty_cache()
            row[f"{plabel}_pme_step_time_ratio"] = round(row[f"{plabel}_reaction_field"]["steps_per_s"] / row[f"{plabel}_pme"]["steps_per_s"], 2)
        result["workloads"][name] = row
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()

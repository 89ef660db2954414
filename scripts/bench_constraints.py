"""Simulated time per wall-clock time with rigid water: flexible water at 1 fs against ``Constraints(kind="water")``
at 2 fs, on water10k and water100k (BASELINE config 4 settings: LJ with switch 7.5 + reaction-field electrostatics,
cutoff 9 A, bonds and angles, Langevin 300 K, gamma 0.1/ps, one replica, fp32, default pair path).  Both runs start
from the lattice start relaxed on the fp32 full rows.  Reports steps/s, simulated ns/day and kernel launches per
step and neighbour-list rebuilds per step, with the card's name and power limit, as one JSON line.

  python scripts/bench_constraints.py [--steps K] [--warmup W] [--workloads water10k,water100k]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--relax", type=int, default=1000, help="fp32 full-row steps at 1 fs that relax the lattice start")
    ap.add_argument("--workloads", default="water10k,water100k")
    args = ap.parse_args()

    import torch

    import bench
    from bench_precision import gpu_info
    from torchmd_b200 import Constraints, Forces, Integrator, System, maxwell_boltzmann

    dev = "cuda:0"
    if not torch.cuda.is_available():
        raise SystemExit("bench_constraints.py measures on a CUDA device; none found")

    def run(name, coords, vel, box, dt_fs, rigid, steps, warmup, cluster=True):
        os.environ["TMD_B200_CLUSTER"] = "1" if cluster else "0"
        par, _, _, terms, cfg, _, _ = bench.build_workload(name, dev, precision=torch.float32)
        forces = Forces(par, terms=terms, **cfg)
        system = System(coords.shape[0], 1, torch.float32, dev)
        system.set_positions(coords)
        system.set_box(box)
        system.set_velocities(vel)
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
        return system, {"dt_fs": dt_fs, "steps_per_s": round(rate, 1), "ns_per_day": round(rate * dt_fs * 1e-6 * 86400, 2),
                        "kernel_launches_per_step": (st1["kernel_launches"] - st0["kernel_launches"]) / steps,
                        "rebuilds_per_step": round((st1["rebuilds"] - st0["rebuilds"]) / steps, 4),
                        "T_end": round(float(T[0]), 1)}

    result = {"metric": "simulated ns/day, flexible 1 fs vs rigid water 2 fs", "gpu": gpu_info(), "steps": args.steps,
              "warmup": args.warmup, "workloads": {}}
    for name in args.workloads.split(","):
        _, coords, box, *_ = bench.build_workload(name, "cpu")
        torch.manual_seed(1)
        par, *_ = bench.build_workload(name, "cpu")
        vel0 = maxwell_boltzmann(par.masses.float(), 300.0, 1)
        relaxed, _ = run(name, coords, vel0, box, 1.0, False, 0, args.relax, cluster=False)
        start, vel = relaxed.pos[0].cpu().numpy(), relaxed.vel.cpu()
        del relaxed
        row = {"natoms": int(coords.shape[0])}
        for label, dt, rigid in (("flexible_1fs", 1.0, False), ("rigid_water_2fs", 2.0, True)):
            row[label] = run(name, start, vel, box, dt, rigid, args.steps, args.warmup)[1]
            torch.cuda.empty_cache()
        row["ns_per_day_gain"] = round(row["rigid_water_2fs"]["ns_per_day"] / row["flexible_1fs"]["ns_per_day"], 2)
        result["workloads"][name] = row
    print(json.dumps(result))


if __name__ == "__main__":
    main()

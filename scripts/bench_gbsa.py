"""Generalized Born implicit solvent (OBC2) against vacuum on thrombin-ligand (4676 atoms, no box, no cutoff): Langevin
at 1 fs (300 K, gamma 1/ps), all AMBER terms, in fp32 and fp64 with 1 and 16 replicas, first without and then with
Forces(..., implicit_solvent="obc2", surface_tension=0.0054).  Reports steps/s, the device time per call of each k_gb_*
kernel (torch.profiler over eager force calls, a separate pass), pair evaluations per second of the GB passes (counted
here: N(N-1) + N^2 + N(N-1) per replica and force call), and the card's name, power limit and SM clock read in the
same call, as one JSON line.

  python scripts/bench_gbsa.py [--steps K] [--warmup W] [--replicas 1,16]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

GB_KERNELS = ("k_gb_radii", "k_gb_energy", "k_gb_forces")


def gpu_info():
    import subprocess

    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def kernel_times(forces, system, calls):
    """Mean device time per force call (microseconds) of each GB kernel and of the pair kernel, over eager calls."""
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
        label = next((k for k in GB_KERNELS if k in ev.key), None)
        if label is None and ("k_pair" in ev.key):
            label = "pair_kernel"
        if label is None:
            continue
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        out[label] = round(out.get(label, 0.0) + t / calls, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--replicas", default="1,16")
    ap.add_argument("--profile-calls", type=int, default=50)
    args = ap.parse_args()

    import numpy as np
    import torch

    from conftest import load_golden, params_from_golden
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann

    if not torch.cuda.is_available():
        raise SystemExit("bench_gbsa.py measures on a CUDA device; none found")
    dev = "cuda:0"
    g, gb = load_golden("thrombin_nobox_rf"), load_golden("gb_radii")
    n = len(g["coords"])
    terms = ["bonds", "angles", "dihedrals", "impropers", "1-4", "lj", "electrostatics"]
    result = {"metric": "thrombin-ligand (4676 atoms, no box, no cutoff), Langevin 1 fs: vacuum vs OBC2 implicit solvent",
              "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "runs": {}}
    for plabel, dtype in (("fp32", torch.float32), ("fp64", torch.float64)):
        for nrep in (int(r) for r in args.replicas.split(",")):
            steps = args.steps if dtype == torch.float32 else max(args.steps // 4, 1)
            for label, solvent in (("vacuum", None), ("obc2", "obc2")):
                par = params_from_golden(g, precision=dtype, device=dev)
                par.gb_params = {"radius": torch.tensor(gb["thrombin_radii"]), "screen": torch.tensor(gb["thrombin_screen"])}
                system = System(n, nrep, dtype, dev)
                system.set_positions(np.repeat(np.asarray(g["coords"], np.float64)[:, :, None], nrep, 2))
                torch.manual_seed(1)
                system.set_velocities(maxwell_boltzmann(par.masses, 300.0, nrep))
                kw = dict(implicit_solvent=solvent, surface_tension=0.0054) if solvent else {}
                forces = Forces(par, terms=terms, cutoff=None, rfa=False, **kw)
                integ = Integrator(system, forces, 1.0, dev, gamma=1.0, T=300.0)
                integ.step(args.warmup)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ekin, pot, _ = integ.step(steps)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                row = {"steps_per_s": round(steps / dt, 1), "pot0": round(float(pot[0]), 3)}
                if solvent:
                    pairs = (2 * n * (n - 1) + n * n) * nrep
                    row["gb_pair_evals_per_s"] = float(f"{pairs * steps / dt:.4g}")
                    row["kernel_us_per_call"] = kernel_times(forces, system, args.profile_calls)
                    row["gb_us_per_call"] = round(sum(v for k, v in row["kernel_us_per_call"].items() if k.startswith("k_gb")), 2)
                result["runs"][f"{plabel}_R{nrep}_{label}"] = row
                del integ, forces, system
                torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()

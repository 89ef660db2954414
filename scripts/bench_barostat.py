"""NVT against NPT (MonteCarloBarostat, a move every 25 steps) for rigid water at 2 fs with Langevin and PME, on
water100k fp32 and water10k fp64.  Prints one JSON line: steps/s and ns/day of both, the barostat's moves and box
changes, the time of one move split into its parts, the k_scale_molecules and k_pme_influence kernel times from
torch.profiler, the mean volume, and the GPU's name, power limit and SM clock read in the same run.

    python scripts/bench_barostat.py [--steps 2000] [--warmup 200]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, sm_clock=clock)
    except Exception as e:  # (the timing still stands; the line says what could not be read)
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unread: {e}", sm_clock="unread")


def setup(nw, dtype, npt, seed=0):
    from torchmd_b200 import Constraints, Forces, Integrator, MonteCarloBarostat, System, maxwell_boltzmann, testsystems

    torch.manual_seed(seed)
    sysd = testsystems.water_box(nw, seed=seed)
    par = testsystems.water_parameters(sysd, precision=dtype, device="cuda:0")
    s = System(len(sysd["coords"]), 1, dtype, "cuda:0")
    s.set_positions(np.asarray(sysd["coords"])[:, :, None])
    s.set_box(np.asarray(sysd["box"]).reshape(3, 1))
    s.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    f = Forces(par, terms=["lj", "electrostatics", "bonds", "angles"], cutoff=9.0, switch_dist=7.5, pme=True)
    bar = MonteCarloBarostat(pressure=1.0, frequency=25) if npt else None
    integ = Integrator(s, f, 2.0, "cuda:0", gamma=1.0, T=300.0, constraints=Constraints(par, "water"), barostat=bar)
    return s, f, bar, integ


def rate(integ, steps, chunk=100):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps // chunk):
        integ.step(chunk)
    torch.cuda.synchronize()
    return (steps // chunk) * chunk / (time.perf_counter() - t0)


def move_parts(s, f, bar, integ, n=20):
    """The move's parts, each timed to a device synchronise: scale kernel, rescale, trial force call, read-back."""
    from torchmd_b200 import _lib

    L = _lib.lib()
    ctx = f._ctx
    stream = torch.cuda.current_stream().cuda_stream
    sfx = "_f64" if s.pos.dtype == torch.float64 else ""
    npd = np.float64 if sfx else np.float32
    diag = torch.diagonal(s.box, dim1=1, dim2=2).cpu().numpy().astype(np.float64)
    t = dict(scale=0.0, rescale=0.0, force=0.0, readback=0.0)
    pos0 = s.pos.clone()
    scratch = torch.empty_like(s.pos)
    ene = torch.empty((1, _lib.NUM_ENERGIES), dtype=torch.float64, device="cuda:0")
    for k in range(n):
        new = (diag * (1.0 + (0.001 if k % 2 == 0 else 0.0))).astype(npd)
        scale = torch.tensor(new.astype(np.float64) / diag, dtype=torch.float64, device="cuda:0")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _lib.check(getattr(L, "tmd_scale_molecules" + sfx)(ctx, s.pos.data_ptr(), scale.data_ptr(), stream))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        _lib.check(getattr(L, "tmd_rescale_box" + sfx)(ctx, np.ascontiguousarray(new).ctypes.data, stream))
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        _lib.check(getattr(L, "tmd_forces" + sfx)(ctx, s.pos.data_ptr(), scratch.data_ptr(), ene.data_ptr(), stream))
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        ene.cpu()
        t4 = time.perf_counter()
        t["scale"] += t1 - t0
        t["rescale"] += t2 - t1
        t["force"] += t3 - t2
        t["readback"] += t4 - t3
        s.pos.copy_(pos0)
        _lib.check(getattr(L, "tmd_rescale_box" + sfx)(ctx, np.ascontiguousarray(diag.astype(npd)).ctypes.data, stream))
    f.compute(s.pos, s.box, s.forces)
    return {k: round(v / n * 1e3, 4) for k, v in t.items()}


def kernel_times(s, f, bar, integ):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        integ.step(250)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("k_scale_molecules", "k_pme_influence"):
            if name in ev.key:
                out[name + "_us"] = round(ev.device_time_total / max(ev.count, 1), 2)
    return out


def arm(nw, dtype, steps, warmup):
    res = {}
    for npt in (False, True):
        s, f, bar, integ = setup(nw, dtype, npt)
        integ.step(warmup)
        r = rate(integ, steps)
        key = "npt" if npt else "nvt"
        res[key + "_steps_per_s"] = round(r, 1)
        res[key + "_ns_per_day"] = round(r * 2e-6 * 86400, 2)
        if npt:
            V = []
            for _ in range(10):
                integ.step(100)
                V.append(float(torch.prod(torch.diagonal(s.box[0])).item()))
            b = bar.stats()[0]
            res.update(moves_attempted=b["attempted"], moves_accepted=b["accepted"], fast_box_changes=b["fast_box_changes"],
                       full_box_changes=b["full_box_changes"], volume_mean_A3=round(float(np.mean(V)), 1))
            res["move_ms"] = move_parts(s, f, bar, integ)
            res.update(kernel_times(s, f, bar, integ))
        del integ, f, s
        torch.cuda.empty_cache()
    res["npt_over_nvt"] = round(res["npt_steps_per_s"] / res["nvt_steps_per_s"], 3)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_barostat needs a CUDA device")
    import __graft_entry__ as g

    g.build()
    line = dict(bench="barostat", frequency=25, steps=a.steps, **gpu_info())
    line["water100k_fp32"] = arm(33333, torch.float32, a.steps, a.warmup)
    line["water10k_fp64"] = arm(3333, torch.float64, a.steps // 4, a.warmup // 4)
    line.update({"after_" + k: v for k, v in gpu_info().items() if k != "gpu"})
    print(json.dumps(line))


if __name__ == "__main__":
    main()

"""Parallel tempering on thrombin (golden_system("thrombin_nobox_rf")): 16 replicas, fp32, Langevin 1/ps, 1 fs, a
geometric ladder from 300 to 450 K.  Four arms: a scalar T, the ladder without exchanges, an exchange every 1000
steps and an exchange every 100 steps.  Prints one JSON line: steps/s of each arm, the device time of one
tmd_replica_exchange call (CUDA events around 200 calls), the acceptance of each neighbour pair in the last arm, and
the GPU's name, power limit and SM clock read in the same run.

    python scripts/bench_remd.py [--steps 6000] [--warmup 1000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
R = 16
TEMPS = [300.0 * 1.5 ** (k / (R - 1)) for k in range(R)]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, sm_clock=clock)
    except Exception as e:  # (the timing still stands; the line says what could not be read)
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unread: {e}", sm_clock="unread")


def setup(T, frequency=None):
    from torchmd_b200 import Forces, Integrator, ReplicaExchange, System, maxwell_boltzmann, testsystems

    torch.manual_seed(0)
    par, coords, box, terms, cfg = testsystems.golden_system("thrombin_nobox_rf", device="cuda:0")
    s = System(len(coords), R, torch.float32, "cuda:0")
    s.set_positions(np.repeat(np.asarray(coords)[:, :, None], R, 2))
    s.set_box(np.repeat(np.asarray(box, np.float64).reshape(3, -1)[:, :1], R, 1))
    s.set_velocities(maxwell_boltzmann(par.masses, T, R))
    f = Forces(par, terms=terms, **cfg)
    f.compute(s.pos, s.box, s.forces)
    rex = ReplicaExchange(frequency=frequency, seed=1) if frequency else None
    integ = Integrator(s, f, 1.0, "cuda:0", gamma=1.0, T=T, replica_exchange=rex)
    return s, f, rex, integ


def rate(integ, steps, chunk=1000):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps // chunk):
        integ.step(chunk)
    torch.cuda.synchronize()
    return (steps // chunk) * chunk / (time.perf_counter() - t0)


def attempt_us(s, f, rex, integ, n=200):
    from torchmd_b200 import _lib

    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    ene = integ._out[1]
    args = (f._ctx, ene.data_ptr(), _lib.NUM_ENERGIES, _lib.NUM_ENERGIES, rex.seed)
    counts = torch.zeros((R - 1, 2), dtype=torch.int64, device="cuda:0")
    for a in range(20):  # warm-up
        _lib.check(L.tmd_replica_exchange(*args, a, s.vel.data_ptr(), counts.data_ptr(), stream))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for a in range(n):
        _lib.check(L.tmd_replica_exchange(*args, a, s.vel.data_ptr(), counts.data_ptr(), stream))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6000)
    ap.add_argument("--warmup", type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_remd.py needs a CUDA GPU")
    res = dict(system="thrombin_nobox_rf", replicas=R, precision="fp32", dt_fs=1.0, gamma_ps=1.0,
               ladder_K=[round(t, 2) for t in TEMPS], steps=a.steps, warmup=a.warmup)
    arms = [("scalar_T", 300.0, None), ("ladder_no_exchange", TEMPS, None), ("exchange_every_1000", TEMPS, 1000),
            ("exchange_every_100", TEMPS, 100)]
    for name, T, freq in arms:
        s, f, rex, integ = setup(T, freq)
        rate(integ, a.warmup)
        res[name + "_steps_per_s"] = round(rate(integ, a.steps), 1)
        res[name + "_pair_kernel"] = int(__import__("torchmd_b200")._lib.lib().tmd_pair_kernel(f._ctx))
        if rex is not None:
            res[name + "_attempts"] = rex.attempts
        if freq == 100:
            res["acceptance_per_pair"] = [round(float(x), 3) for x in rex.acceptance()]
            res["us_per_attempt"] = round(attempt_us(s, f, rex, integ), 2)
        del s, f, rex, integ
        torch.cuda.empty_cache()
    base = res["scalar_T_steps_per_s"]
    for name in ("ladder_no_exchange", "exchange_every_1000", "exchange_every_100"):
        res[name + "_vs_scalar"] = round(res[name + "_steps_per_s"] / base, 4)
    res.update(gpu_info())
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Cost of the CMAP correction maps: thrombin (tests/golden/thrombin_nobox_rf, the fixture's own settings, Langevin at
300 K, 1 fs) with 1 and 16 replicas, fp32 and fp64, without and with backbone-like CMAP terms (138, picked by the
rule in tests/test_gpu_cmap.py, two 24x24 maps).  For each: steps/s of Integrator.step, the
k_bonded_terms (fp64: k_bonded_terms_f64) time per call from torch.profiler in a run of its own, and the kernel launches
per step.  Prints the GPU's name and power limit read in the same run, and one JSON line.

    python scripts/bench_cmap.py [--steps 2000] [--warmup 200]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_barostat import gpu_info  # noqa: E402


def setup(nrep, dtype, with_cmap):
    import test_gpu_cmap as G
    from conftest import golden_cfg, load_golden
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann

    name = "thrombin_nobox_rf"
    g = load_golden(name)
    G.DEV = "cuda:0"
    par = G.make_params(g, name, dtype, with_cmap=with_cmap)
    rng = np.random.default_rng(0)
    coords = np.stack([g["coords"] + (rng.normal(scale=0.01, size=g["coords"].shape) if r else 0) for r in range(nrep)])
    s = System(coords.shape[1], nrep, dtype, "cuda:0")
    s.set_positions(np.ascontiguousarray(coords.transpose(1, 2, 0)))
    s.set_box(np.zeros((3, nrep)))
    torch.manual_seed(0)
    s.set_velocities(maxwell_boltzmann(par.masses, 300.0, nrep))
    f = Forces(par, terms=[str(t) for t in g["terms"]], **golden_cfg(g))
    f.compute(s.pos, s.box, s.forces)
    return f, Integrator(s, f, 1.0, "cuda:0", gamma=1.0, T=300.0), (0 if par.cmap_params is None else len(par.cmap_params["idx"]))


def arm(nrep, dtype, with_cmap, steps, warmup, chunk=100):
    from torch.profiler import ProfilerActivity, profile

    f, integ, nterms = setup(nrep, dtype, with_cmap)
    integ.step(warmup)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps // chunk):
        integ.step(chunk)
    torch.cuda.synchronize()
    rate = (steps // chunk) * chunk / (time.perf_counter() - t0)
    n0 = f.stats()["kernel_launches"]
    integ.step(chunk)
    launches = (f.stats()["kernel_launches"] - n0) / chunk
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        integ.step(200)
        torch.cuda.synchronize()
    us = None
    for ev in prof.key_averages():
        if "k_bonded_terms" in ev.key:
            us = round(ev.device_time_total / max(ev.count, 1), 2)
    return dict(cmap_terms=nterms, steps_per_s=round(rate, 1), k_bonded_terms_us=us, launches_per_step=launches)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_cmap needs a CUDA device")
    import __graft_entry__ as g

    g.build()
    info = gpu_info()
    print(f"[bench_cmap] {info['gpu']}, power limit {info['power_limit']}", flush=True)
    line = dict(bench="cmap", workload="thrombin_nobox_rf", steps=a.steps, **info)
    for nrep in (1, 16):
        for dtype, tag in ((torch.float32, "fp32"), (torch.float64, "fp64")):
            for with_cmap in (False, True):
                key = f"r{nrep}_{tag}_{'cmap' if with_cmap else 'plain'}"
                line[key] = arm(nrep, dtype, with_cmap, a.steps, a.warmup)
                print(f"[bench_cmap] {key}: {line[key]}", flush=True)
                torch.cuda.empty_cache()
    print(json.dumps(line))


if __name__ == "__main__":
    main()

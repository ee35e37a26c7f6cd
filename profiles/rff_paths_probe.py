"""Timing probe of the kernel-matched random features and the sample-function evaluator (cmoe_gp_sample_rff_optima_ex,
cmoe_rff_evaluate; DESIGN.md K14 addendum).

1. Matched against reference mode at K14's shapes (those of profiles/rff_probe.py, on Matern-5/2 GPs), P = 200 and
   G = 10^4: the whole call (host clock ending in a synchronise, median of 9 after a warm-up) in each mode, and the
   features kernel's device time in each mode from torch.profiler.
2. The evaluator's throughput in cosine evaluations per second (P X F per call) for shared and per-function points, with
   and without gradients, from torch.profiler device times, next to the grid stage of the same sample functions.
3. NumPy on the host evaluating the same functions at the same points (one function at a time, as the reference's
   wrapper does), for the ratio.
The card's name, power limit and SM clock are read in the same run.  Prints one JSON line per row; writes a file only
when --out names one."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "cornell-moe_b200"), os.path.join(ROOT, "tests")]

from synth import make_problem  # noqa: E402

SHAPES = [(20, 2, 0), (150, 2, 2), (500, 8, 0)]
FS = [256, 1000, 4096]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=False).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(f, reps=9):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def device_ms(f, names, runs=3):
    """Device time per run (ms) of the kernels whose names contain any of `names`."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    f()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            f()
        torch.cuda.synchronize()
    t = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and any(nm in e.name for nm in names):
            t += e.device_time_total * 1e-3 / runs
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--numpy-max-cos", type=float, default=2e9, help="skip the host NumPy arm above this P X F")
    a = ap.parse_args()
    from cornell_moe_b200 import capi
    rows = []
    print(json.dumps({"card": card()}), flush=True)

    def emit(row):
        rows.append(row)
        print(json.dumps(row), flush=True)

    P, G = 200, 10000
    for n, d, g in SHAPES:
        pr = make_problem(n, d, tuple(range(g)), seed=0, noise=1e-2, length=0.3)
        gp = capi.GaussianProcess(capi.MATERN_NU_2P5, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"],
                                  pr["derivs"])
        grid = np.random.default_rng(1).uniform(size=(G, d))
        bounds = np.array([[0.0, 1.0]] * d)
        for F in FS:
            row = dict(part="modes", n=n, d=d, g=g, M=n * (1 + g), F=F, P=P, G=G)
            for name, sp in (("reference", capi.RFF_SPECTRAL_REFERENCE), ("kernel", capi.RFF_SPECTRAL_KERNEL)):
                call = lambda: gp.sample_rff_optima(F, P, bounds, grid, seed=7, spectral=sp)  # noqa: E731
                row[f"{name}_call_ms"] = timed(call) * 1e3
                row[f"{name}_features_ms"] = device_ms(call, ("rff_features_kernel",))
                row[f"{name}_grid_ms"] = device_ms(call, ("rff_grid_kernel",))
            emit(row)

    # the evaluator against the grid stage of the same functions, and NumPy
    for d, F, P, X in ((2, 1000, 200, 10000), (8, 4096, 200, 10000), (8, 4096, 16, 100000)):
        pr = make_problem(500, d, (), seed=0, noise=1e-2, length=0.3)
        gp = capi.GaussianProcess(capi.MATERN_NU_2P5, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"])
        fun = gp.sample_rff_functions(F, P, seed=3, spectral=capi.RFF_SPECTRAL_KERNEL)
        x = np.random.default_rng(2).uniform(size=(X, d))
        xp = np.random.default_rng(3).uniform(size=(P, X, d))
        cos = P * X * F
        row = dict(part="evaluator", d=d, F=F, P=P, X=X, cos=cos)
        for name, pts, grads in (("shared", x, False), ("shared_grad", x, True), ("per_function", xp, False)):
            f = lambda: capi.rff_evaluate(fun.omega, fun.b, fun.theta, fun.c, pts, grads=grads)  # noqa: E731
            kms = device_ms(f, ("rff_eval_kernel",))
            row[f"{name}_kernel_ms"] = kms
            row[f"{name}_gcos_per_s"] = cos / (kms * 1e-3) / 1e9 if kms else None
            row[f"{name}_call_ms"] = timed(f, reps=3) * 1e3
        bounds = np.array([[0.0, 1.0]] * d)
        opt = lambda: gp.sample_rff_optima(F, P, bounds, x, seed=3, spectral=capi.RFF_SPECTRAL_KERNEL)  # noqa: E731
        gms = device_ms(opt, ("rff_grid_kernel",), runs=1)
        row["grid_stage_ms"] = gms
        row["grid_stage_gcos_per_s"] = cos / (gms * 1e-3) / 1e9 if gms else None
        if cos <= a.numpy_max_cos:
            t0 = time.perf_counter()
            for p in range(P):
                fun.c * np.cos(x @ fun.omega[p].T + fun.b[p]) @ fun.theta[p]
            row["numpy_shared_s"] = time.perf_counter() - t0
            row["numpy_over_call"] = row["numpy_shared_s"] / (row["shared_call_ms"] * 1e-3)
        emit(row)
    print(json.dumps({"card_after": card()}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1, default=str)


if __name__ == "__main__":
    main()

"""Timing probe of the random-feature sampler (cmoe_gp_sample_rff_optima, DESIGN.md K14) on SquareExponential GPs.

Shapes: (n, d, g) in {(20, 2, 0), (150, 2, 2), (500, 8, 0)}, F in {256, 1000, 4096} (M = n (1 + g) < F takes the
Woodbury branch; F = 256 puts the last two shapes on the Cholesky branch), P in {16, 200, 1024}, G in {1e3, 1e4,
1e5}; a shape is timed only when P G F <= --max-cos (the grid stage alone is P G F FP64 cosines).  For each: the whole
device call (host clock ending in a synchronise, median, min and max of 9 after a warm-up).  For P = 200, G = 1e4 a
separate torch.profiler run gives each stage's device time (features + design, Gram, factor, theta, grid, optimiser),
the Gram stage's FP64 rate (its Q(Q+1)/2 K multiply-adds, 2 FLOP each, per sample) against the DMMA peak that
cmoe_bench_fp64_peaks measures in the same run, and the grid stage's cosine evaluations per second.  The card's name,
power limit and SM clock are read in the same run.  Prints one JSON line per shape; writes a file only when --out names
one.  `--reference` (development host only; it reads the reference checkout) times the reference's per-sample routine
instead."""
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
FS, PS, GS = [256, 1000, 4096], [16, 200, 1024], [1000, 10000, 100000]
STAGES = {"design": ("rff_features_kernel", "rff_design_kernel"), "gram": ("rff_gram_kernel",),
          "factor": ("chol_panel_kernel", "chol_update_kernel", "chol_diag_writeback_kernel"),
          "theta": ("rff_theta_kernel",), "grid": ("rff_grid_kernel", "best_of_parts_kernel"), "opt": ("rff_opt_kernel",)}


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
    return statistics.median(ts), min(ts), max(ts)


def problem(n, d, g):
    derivs = tuple(range(g))
    pr = make_problem(n, d, derivs, seed=0, noise=1e-2, length=0.3)
    grid_rng = np.random.default_rng(1)
    return pr, grid_rng


def stage_seconds(gp, args, runs=2):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            gp.sample_rff_optima(*args)
        torch.cuda.synchronize()
    out = {k: 0.0 for k in STAGES}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for k, names in STAGES.items():
            if any(nm in e.name for nm in names):
                out[k] += e.device_time_total * 1e-6 / runs
    return out


def device_probe(a):
    from cornell_moe_b200 import capi
    peaks = capi.fp64_peaks()
    print(json.dumps({"card": card(), "fp64_peaks": peaks}, default=str), flush=True)
    rows = []
    for n, d, g in SHAPES:
        pr, rng = problem(n, d, g)
        gp = capi.GaussianProcess(capi.SQUARE_EXPONENTIAL, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"],
                                  pr["derivs"])
        bounds = np.array([[0.0, 1.0]] * d)
        M = n * (1 + g)
        for F in a.features:
            for G in GS:
                grid = rng.uniform(size=(G, d))
                for P in PS:
                    if P * G * F > a.max_cos:
                        continue
                    args = (F, P, bounds, grid, 7)
                    t = timed(lambda: gp.sample_rff_optima(*args))
                    row = dict(n=n, d=d, g=g, M=M, F=F, P=P, G=G, branch="woodbury" if M < F else "cholesky",
                               call_ms=t[0] * 1e3, call_ms_min=t[1] * 1e3, call_ms_max=t[2] * 1e3)
                    if P == 200 and G == 10000:
                        st = stage_seconds(gp, args)
                        Q, K = min(F, M), max(F, M)
                        row.update({f"{k}_ms": v * 1e3 for k, v in st.items()})
                        row["gram_tflops"] = P * Q * (Q + 1) / 2 * K * 2 / st["gram"] / 1e12 if st["gram"] else None
                        row["grid_gcos_per_s"] = P * G * F / st["grid"] / 1e9 if st["grid"] else None
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "fp64_peaks": peaks, "rows": rows}, f, indent=1, default=str)


def reference_probe(a):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_rff_golden as mk
    rf = mk._load_reference()
    for n, d, g in SHAPES:
        pr, rng = problem(n, d, g)
        Y = pr["y"].reshape(n, 1 + g)
        gp = mk.StubGP(pr["X"], Y, pr["noise"], list(range(g)), pr["alpha"], pr["lengths"])
        for F in a.features:
            grid = rng.uniform(size=(1000, d))
            t0 = time.perf_counter()
            rf.sample_from_global_optima(gp, F, [[0.0, 1.0]] * d, grid, 2)
            print(json.dumps(dict(n=n, d=d, g=g, F=F, G=1000, reference_s_per_sample=(time.perf_counter() - t0) / 2)),
                  flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--max-cos", type=float, default=2e11, help="skip shapes with P G F above this")
    ap.add_argument("--features", type=int, nargs="+", default=FS)
    ap.add_argument("--reference", action="store_true", help="time the reference routine (development host only)")
    a = ap.parse_args()
    reference_probe(a) if a.reference else device_probe(a)


if __name__ == "__main__":
    main()

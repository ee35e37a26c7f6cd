"""Timing probe of the LCB batch selection (cmoe_lcb_select, DESIGN.md K13) on Matern-5/2 GPs.

For (N, d) in {(50, 2), (500, 8), (2000, 10)}, C in {1e3, 1e4, 1e5} and q in {1, 4, 16}: the whole device call (host
clock ending in a synchronise, median, min and max of 9 after a warm-up), the screen's FP64 rate C n^2 over the summed
device time of its kernels (mix_cov_kernel, trsm_kernel, post_mean_only_kernel, lcb_screen_kernel; a separate
torch.profiler run of 3 q = 1 calls), and the
reference routine's pattern on the drop-in GPP module (one compute_cholesky_variance_of_points call per candidate and
a refit per round), timed on a subset of candidates and scaled.  Prints one JSON line per shape and the card's name
and power limit; writes a file only when --out names one."""
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

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402
from synth import make_problem  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=False).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(f, reps=9):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), min(ts), max(ts)


SCREEN_KERNELS = ("mix_cov_kernel", "trsm_kernel", "post_mean_only_kernel", "lcb_screen_kernel")


def screen_kernel_seconds(gp, cand, runs=3):
    """Summed device time per call of the screen's kernels, from torch.profiler (CUDA activities only)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            gp.lower_confidence_bound(cand, 1)
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and any(k in e.name for k in SCREEN_KERNELS):
            total += e.device_time_total * 1e-6
    return total / runs


def reference_pattern(pr, cand, q, nsat, subset=50):
    """Seconds for the front end's loop through GPP: C + (q - 1) C' single-candidate calls and q - 1 refits."""
    N, d = pr["X"].shape
    gp = C_GP.GaussianProcess([pr["alpha"], list(pr["lengths"])], list(pr["X"].ravel()), list(pr["y"]),
                              list(pr["noise"]), [], 0, d, N)
    pts = [list(c) for c in cand[:subset]]
    gp.compute_cholesky_variance_of_points(pts[0], 1)
    t0 = time.perf_counter()
    for p in pts:
        gp.compute_cholesky_variance_of_points(p, 1)
    per_call = (time.perf_counter() - t0) / len(pts)
    t_refit = 0.0
    if q > 1:
        t0 = time.perf_counter()
        gp.add_sampled_points(list(cand[0]), [0.0], 1)  # one AddPointsToGP append
        t_refit = time.perf_counter() - t0
    return per_call * (len(cand) + (q - 1) * nsat) + (q - 1) * t_refit, per_call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="one small shape (a rehearsal)")
    a = ap.parse_args()
    shapes = [(50, 2), (500, 8), (2000, 10)]
    Cs, qs = [1000, 10000, 100000], [1, 4, 16]
    if a.quick:
        shapes, Cs, qs = [(50, 2)], [1000], [1, 4]
    print(json.dumps({"card": card()}), flush=True)
    rows = []
    for N, d in shapes:
        pr = make_problem(N, d, (), seed=0)
        gp = capi.GaussianProcess(capi.MATERN_NU_2P5, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"])
        for C in Cs:
            cand = np.random.default_rng(1).uniform(size=(C, d))
            t_screen = timed(lambda: gp.lower_confidence_bound(cand, 1))
            _, mean, sd = gp.lower_confidence_bound(cand, 1)
            nsat = int(np.sum(mean - sd <= np.min(mean + sd)))
            k_screen = screen_kernel_seconds(gp, cand)
            for q in qs:
                t = t_screen if q == 1 else timed(lambda: gp.lower_confidence_bound(cand, q))
                t_ref, per_call = reference_pattern(pr, cand, q, nsat)
                row = dict(N=N, d=d, C=C, q=q, num_satisfied=nsat, call_ms=t[0] * 1e3, call_ms_min=t[1] * 1e3,
                           call_ms_max=t[2] * 1e3, screen_kernel_ms=k_screen * 1e3,
                           screen_gflops=C * float(N) ** 2 / k_screen / 1e9, reference_pattern_s=t_ref,
                           reference_per_call_ms=per_call * 1e3, speedup=t_ref / t[0])
                rows.append(row)
                print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()

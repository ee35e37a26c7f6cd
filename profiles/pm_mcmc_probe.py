"""Times the ensemble posterior-mean calls of the recommendation step (cmoe_posterior_mean_mcmc and
cmoe_posterior_mean_mcmc_optimization) at M = 16 members, (N, d) = (50, 2) and (500, 8), Matern-5/2, with the parameters
of examples/main.py (1000 steps, 15 averaged, gamma 0.7, pre_mult 1.0, max_relative_change 0.02), and prints one JSON
line with the card name, power limit and SM clock read in the same run.

Device figures are host wall-clock times of whole calls (each ends in a stream synchronise), the median of --runs after
one warm-up call:
  * screening of 1e4 points;
  * the 1000-step descent from 1, 128 and 1024 starts (per-step time = one start / 1000);
  * recommend_point end to end (screen 1e4 points, descend from the best one).

For an order of magnitude, the same run times the reference's way of doing the work on the CPU: one call per point and
per member into the compiled reference (oracle/_ref, or the C oracle if that is missing), which stands for the
Boost.Python call PosteriorMeanMCMC makes per member.  The screening is timed over --cpu-points points and the descent
over --cpu-steps steps, then scaled linearly to 1e4 points and 1000 steps (the work is the same per point and per step).
This is not a like-for-like comparison: the CPU figure is one core in a Python loop.

    python profiles/pm_mcmc_probe.py [--runs 5] [--cpu-points 1000] [--cpu-steps 100]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from cornell_moe_b200 import capi  # noqa: E402

M = 16
PARAMS = capi.GDParams(1, 1000, 3, 15, 0.7, 1.0, 0.02, 1e-10)  # examples/main.py:115-121


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    line = out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in line.split(",")])) if line else {"error": out.stderr.strip()}


def timed(fn, runs):
    fn()  # warm-up
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def workload(N, d, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, d))
    y = np.sin(3 * X).sum(axis=1)
    hypers = np.column_stack([rng.uniform(0.5, 2.0, M), rng.uniform(0.2, 0.5, (M, d))])
    noises = np.full((M, 1), 1e-2)
    bounds = np.tile([0.0, 1.0], (d, 1))
    pts = rng.uniform(size=(10000, d))
    starts = rng.uniform(size=(1024, d))
    return X, y, hypers, noises, bounds, pts, starts


def cpu_reference(X, y, hypers, noises, pts, starts, n_pts, n_steps):
    import oracle as orc
    backend = orc.load_reference() if orc.have_reference() else orc.load_oracle()
    gps = [backend.gp(1, h[0], h[1:], X, y, nz)[0] for h, nz in zip(hypers, noises)]
    t0 = time.perf_counter()
    for x in pts[:n_pts]:
        v = 0.0
        for gp in gps:
            v += -float(gp.mean_additional(x)[0])
    screen_ms = (time.perf_counter() - t0) * 1e3 * (len(pts) / n_pts)
    x = starts[0].copy()
    t0 = time.perf_counter()
    for k in range(1, n_steps + 1):
        g = np.zeros(X.shape[1])
        for gp in gps:
            g += -gp.posterior(x, want=("grad_mean",))["grad_mean"]
        x = np.clip(x + (g / M) * PARAMS.pre_mult * k ** -PARAMS.gamma, 0.0, 1.0)
    descent_ms = (time.perf_counter() - t0) * 1e3 * (PARAMS.max_num_steps / n_steps)
    return {"backend": backend.name, "screen_1e4_ms": screen_ms, "descent_1000_steps_ms": descent_ms,
            "timed_points": n_pts, "timed_steps": n_steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--cpu-points", type=int, default=1000)
    ap.add_argument("--cpu-steps", type=int, default=100)
    args = ap.parse_args()
    assert capi.device_count() > 0, "no CUDA device"
    out = {"card": card(), "M": M, "params": "1000 steps, 15 averaged, gamma 0.7, pre_mult 1.0, mrc 0.02",
           "shapes": []}
    for N, d in ((50, 2), (500, 8)):
        X, y, hypers, noises, bounds, pts, starts = workload(N, d)
        ens = capi.GaussianProcessEnsemble(hypers, noises, X, y, kernel=capi.MATERN_NU_2P5)
        row = {"N": N, "d": d}
        row["screen_1e4_ms"] = timed(lambda: ens.posterior_mean(pts), args.runs)
        row["screen_1e4_grad_ms"] = timed(lambda: ens.posterior_mean(pts, grad=True), args.runs)
        for S in (1, 128, 1024):
            row[f"descent_{S}_starts_ms"] = timed(
                lambda S=S: ens.posterior_mean_optimization(starts[:S], PARAMS, bounds), args.runs)
        row["per_step_1_start_us"] = row["descent_1_starts_ms"] * 1e3 / PARAMS.max_num_steps
        row["recommend_point_ms"] = timed(lambda: ens.recommend_point(pts, PARAMS, bounds), args.runs)
        row["cpu_reference_loops"] = cpu_reference(X, y, hypers, noises, pts, starts, args.cpu_points, args.cpu_steps)
        out["shapes"].append(row)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

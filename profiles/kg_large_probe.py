"""Timing probe of q-KG past 32 union rows (cmoe_kg_eval_large, DESIGN.md K17).

Call times (host clock ending in a synchronise, median of --reps after a warm-up) of the value and of value + gradient:
* N = 500, d = 8, SquareExponential, EXAMPLE_INNER_GD, 64 candidates x 4096 samples, Q = q = 32, 64 and 128;
* d-KG at d = 8 with all 8 partials observed (g = 8), q + p = 4 (Q = 36), N = 100, same inner optimiser.
Each line gives sample-evaluations per second (candidates x num_mc / call time).  At Q = 32 the same inputs also run
through cmoe_kg_eval: the workload on each side of the drivers' selection at 32 rows.  `--profile` adds one
torch.profiler run (value + gradient at Q = 64) that gives each kernel's device time.  The card's name, power limit and
SM clock are read in the same run.  Prints JSON lines; writes them to --out when given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=False).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    from cornell_moe_b200 import capi
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(json.dumps(d))

    emit({"card": card()})
    nc, mc, d = 64, 4096, 8
    rng = np.random.default_rng(0)
    prob = make_problem(500, d, seed=1, noise=1e-2)
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"])
    disc = rng.uniform(size=(10, d))
    args_kg = (mc, 0.1, EXAMPLE_INNER_GD, unit_bounds(d), disc)
    for q in (32, 64, 128):
        cands = rng.uniform(size=(nc, q, d))
        tv = timed(lambda: gp.kg_large(cands, None, *args_kg, seed=1), args.reps)
        tg = timed(lambda: gp.kg_large(cands, None, *args_kg, seed=1, grad=True), args.reps)
        line = {"shape": "N=500 d=8 SE", "Q": q, "candidates": nc, "num_mc": mc, "value_s": tv, "value_grad_s": tg,
                "value_sample_evals_per_s": nc * mc / tv, "value_grad_sample_evals_per_s": nc * mc / tg}
        if q == 32:
            sv = timed(lambda: gp.kg(cands, None, *args_kg, seed=1), args.reps)
            sg = timed(lambda: gp.kg(cands, None, *args_kg, seed=1, grad=True), args.reps)
            line.update({"kg_eval_value_s": sv, "kg_eval_value_grad_s": sg})
        emit(line)
    dprob = make_problem(100, d, g_idx=tuple(range(d)), seed=2, noise=1e-2)
    dgp = capi.GaussianProcess(0, dprob["alpha"], dprob["lengths"], dprob["X"], dprob["y"], dprob["noise"],
                               dprob["derivs"])
    cands = rng.uniform(size=(nc, 2, d))
    Xp = rng.uniform(size=(2, d))
    tv = timed(lambda: dgp.kg_large(cands, Xp, *args_kg, seed=1), args.reps)
    tg = timed(lambda: dgp.kg_large(cands, Xp, *args_kg, seed=1, grad=True), args.reps)
    emit({"shape": "d-KG N=100 d=8 g=8 q=2 p=2", "Q": 36, "candidates": nc, "num_mc": mc, "value_s": tv,
          "value_grad_s": tg, "value_sample_evals_per_s": nc * mc / tv, "value_grad_sample_evals_per_s": nc * mc / tg})
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        cands = rng.uniform(size=(nc, 64, d))
        gp.kg_large(cands, None, *args_kg, seed=1, grad=True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            gp.kg_large(cands, None, *args_kg, seed=1, grad=True)
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                per[e.name] = per.get(e.name, 0.0) + e.device_time_total
        top = sorted(per.items(), key=lambda kv: -kv[1])[:15]
        emit({"profile": "N=500 d=8 Q=64 candidates=64 num_mc=4096 value+grad", "device_us": {k[:60]: v for k, v in top}})
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

"""Timing probe of the large-set q-EI (cmoe_ei_eval_large, DESIGN.md K16).

Call times (host clock ending in a synchronise, median of 5 after a warm-up) of value + gradient for U in {128, 512,
2048} x num_mc in {1e3, 1e4} x {1, 64} candidates (p = 0, n = 200 training points, d = 4, Philox normals).  For each
value-only call the forward tiles' FP64 rate from U (U + 1) / 2 num_mc multiply-adds per candidate (2 FLOP each) over
the call time (an underestimate of the tiles' own rate: the call also builds the posterior), against the DMMA peak that
cmoe_bench_fp64_peaks measures in the same run.  At U = 96 the same call against cmoe_ei_eval: the workload on each side
of the drivers' size selection.  `--profile` adds one torch.profiler run at U = 512, num_mc = 1e4, 64 candidates that
gives each kernel's device time.  The card's name, power limit and SM clock are read in the same run.  Prints JSON
lines; writes them to --out when given."""
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

from synth import make_problem  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=False).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(f, reps=5):
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
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    from cornell_moe_b200 import capi
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(json.dumps(d))

    emit({"card": card(), "fp64_peaks_tflops": capi.fp64_peaks()})
    prob = make_problem(200, 4, seed=1, length=0.4)
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"])
    best = float(prob["y"].min()) + 0.3
    rng = np.random.default_rng(0)
    for U in (128, 512, 2048):
        for mc in (1000, 10000):
            for nc in (1, 64):
                cands = rng.uniform(size=(nc, U, 4))
                tv = timed(lambda: gp.ei_large(cands, None, mc, best, seed=1))
                tg = timed(lambda: gp.ei_large(cands, None, mc, best, seed=1, grad=True))
                flops = 2.0 * U * (U + 1) / 2 * mc * nc
                emit({"U": U, "num_mc": mc, "candidates": nc, "value_s": tv, "value_grad_s": tg,
                      "forward_tflops_lower_bound": flops / tv / 1e12})
    cands = rng.uniform(size=(64, 96, 4))
    for mc in (1000, 10000):
        t_small = timed(lambda: gp.ei(cands, None, mc, best, seed=1, grad=True))
        t_large = timed(lambda: gp.ei_large(cands, None, mc, best, seed=1, grad=True))
        emit({"U": 96, "num_mc": mc, "candidates": 64, "ei_eval_s": t_small, "ei_eval_large_s": t_large})
    if args.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        cands = rng.uniform(size=(64, 512, 4))
        gp.ei_large(cands, None, 10000, best, seed=1, grad=True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            gp.ei_large(cands, None, 10000, best, seed=1, grad=True)
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                per[e.name] = per.get(e.name, 0.0) + e.device_time_total
        top = sorted(per.items(), key=lambda kv: -kv[1])[:15]
        emit({"profile": "U=512 num_mc=1e4 candidates=64 value+grad", "device_us": {k[:60]: v for k, v in top}})
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

"""Timing of joint posterior sampling on one GPU: cmoe_gp_sample_global_optima at N = 500, d = 8 (SE), the batched
Cholesky against a loop of the single-matrix Cholesky on the same device-resident matrices, and the reference's CPU time
for the work of one optimum.  Prints one JSON object.

    python profiles/sample_probe.py [--repeats 3] [--out FILE]

Host time is taken around whole calls (each ends in a device synchronise), after one warm-up call.  Two FP64 rates per
row: ``tflops_shape_count`` takes n^2 Q (triangular solve) + n Q^2 (V^T V in full) + Q^3 / 3 (Cholesky) per optimum;
``tflops_executed`` counts V^T V as computed, on the lower 64 x 64 tiles only (n 64^2 per tile, T (T+1) / 2 tiles for
T = ceil(Q / 64), about n Q^2 / 2).  The loop baseline of the Cholesky comparison calls potrf_lower once per matrix;
each call carries its own host work (scratch allocation, attribute set-up, a stream synchronise), so the ratio is
call against call, not kernel against kernel.  The reference figure is ONE timed call per shape (after one warm-up call
at the smallest shape) of what SamplePointsFromGP computes before its normals (ComputeMeanOfPoints,
ComputeVarianceOfPoints, ComputeCholeskyFactorL) through oracle/_ref, single-threaded: an order of magnitude; the
normals and the mean + L w step are not in it.  "not measured" when oracle/_ref was not built.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle as orc  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, check=True).stdout.strip().split(", ")
        return {"name": q[0], "power_limit": q[1]}
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown", "power_limit": f"not read ({e})"}


def flops(n, Q):
    return n * n * Q + n * Q * Q + Q ** 3 / 3.0


def flops_executed(n, Q):
    t = (Q + 63) // 64
    return n * n * Q + n * 64 * 64 * t * (t + 1) / 2 + Q ** 3 / 3.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    N, dim = 500, 8
    rng = np.random.default_rng(0)
    X = rng.uniform(size=(N, dim))
    y = np.sin(3 * X).sum(axis=1)
    lens = np.full(dim, 0.5)
    gp = capi.GaussianProcess(capi.SQUARE_EXPONENTIAL, 1.0, lens, X, y, [1e-2])
    bounds = np.tile([0.0, 1.0], dim)
    res = {"card": card(), "shape": {"N": N, "dim": dim, "kernel": "square_exponential"}}
    res["dmma_peak_tflops"] = capi.fp64_peaks()[1]
    rows = []
    for B in (16, 128):
        for inner in (256, 1024, 2048):
            gp.sample_global_optima(B, inner, bounds, seed=1)
            ts = []
            for r in range(a.repeats):
                t0 = time.perf_counter()
                gp.sample_global_optima(B, inner, bounds, seed=1, first_draw=r)
                ts.append(time.perf_counter() - t0)
            t = float(np.median(ts))
            rows.append({"num_optima": B, "inner_number": inner, "ms_per_call": t * 1e3,
                         "ms_per_optimum": t * 1e3 / B, "tflops_shape_count": B * flops(N, inner) / t * 1e-12,
                         "tflops_executed": B * flops_executed(N, inner) / t * 1e-12})
            print(json.dumps(rows[-1]), flush=True)
    res["global_optima"] = rows
    chol = []
    for B in (16, 128):
        for Q in (256, 1024, 2048):
            base = []
            for k in range(4):
                P = np.random.default_rng(k).uniform(size=(Q, dim))
                d2 = (((P[:, None, :] - P[None, :, :]) / 0.5) ** 2).sum(axis=2)
                base.append(np.exp(-0.5 * d2) + 1e-3 * np.eye(Q))
            mats = np.stack([base[i % 4] for i in range(B)])
            tb, tl = capi.bench_cholesky_batched(mats, repeats=a.repeats)
            chol.append({"num_mats": B, "Q": Q, "usec_batched": tb, "usec_potrf_loop": tl, "speedup": tl / tb,
                         "tflops_batched": B * Q ** 3 / 3.0 / (tb * 1e-6) * 1e-12})
            print(json.dumps(chol[-1]), flush=True)
            del mats
    res["cholesky"] = chol
    if orc.have_reference():
        ref, lm = orc.load_reference().gp(0, 1.0, lens, X, y, [1e-2])
        cpu = []
        ref.posterior(rng.uniform(size=(256, dim)), want=("mean", "var", "chol_var"))  # warm-up
        for inner in (256, 1024, 2048):
            pts = rng.uniform(size=(inner, dim))
            t0 = time.perf_counter()
            ref.posterior(pts, want=("mean", "var", "chol_var"))
            t = time.perf_counter() - t0
            cpu.append({"inner_number": inner, "ms_one_sample": t * 1e3, "samples": 1})
            print(json.dumps(cpu[-1]), flush=True)
        res["reference_cpu"] = cpu
    else:
        res["reference_cpu"] = "not measured"
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

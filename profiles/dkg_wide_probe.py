"""Times q-KG on GPs with full gradient observations past eight partials (the wide derivative-observation kernel,
kg_mc_gen_kernel<..., WIDE>) and prints one JSON line with the card name, power limit and SM clock read in the same run.

Shapes (SquareExponential, q = 1, 256 candidates x 8192 samples, the inner optimiser of the reference's examples):
  * d = 10, all 10 partials observed, N = 100 (n = 1100);
  * d = 16, all 16 partials observed, N = 60 (n = 1020).

Device figures come from the plan's own CUDA events (cmoe_kg_plan_timings): the whole plan run and the MC kernel alone,
the median of --runs runs after one warm-up run, as MC sample-evaluations per second (candidates x samples / time).

For an order of magnitude, the same run times the reference's evaluator on one host core (oracle/_ref, or the C oracle
if that is missing) over --cpu-samples samples of one candidate, scaled linearly to samples per second.  This is not a
like-for-like comparison: it is one core, value only, on a small sample.

    python profiles/dkg_wide_probe.py [--runs 3] [--cpu-samples 32]
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

INNER = [1, 6, 1, 3, 0.0, 1.0, 0.1, 1e-10]  # examples/main.py:123-130 in the reference
NC, MC, NUM_PTS = 256, 8192, 20


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    line = out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in line.split(",")])) if line else {"error": out.stderr.strip()}


def workload(N, d, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, d))
    y = np.concatenate([np.sin(3 * X).sum(axis=1, keepdims=True), 3 * np.cos(3 * X)], axis=1)
    y += 0.1 * rng.standard_normal(y.shape)
    lengths = np.full(d, 0.5 * np.sqrt(d / 8.0))
    noise = np.full(1 + d, 1e-2)
    cands = rng.uniform(size=(NC, 1, d))
    disc = rng.uniform(size=(NUM_PTS, d))
    return X, y.ravel(), lengths, noise, np.arange(d, dtype=np.int32), cands, disc


def cpu_reference(X, y, lengths, noise, derivs, cand, disc, best, samples):
    import oracle as orc
    backend = orc.load_reference() if orc.have_reference() else orc.load_oracle()
    ref, _ = backend.gp(0, 1.0, lengths, X, y, noise, derivs)
    d = X.shape[1]
    table = np.random.default_rng(1).standard_normal((samples // 2) * (1 + d))
    t0 = time.perf_counter()
    ref.kg(cand, None, samples, best, table, INNER, np.tile([0.0, 1.0], d), disc)
    dt = time.perf_counter() - t0
    return {"backend": backend.name, "timed_samples": samples, "sample_evals_per_s": samples / dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--cpu-samples", type=int, default=32)
    args = ap.parse_args()
    assert capi.device_count() > 0, "no CUDA device"
    out = {"card": card(), "candidates": NC, "num_mc": MC, "q": 1, "num_pts": NUM_PTS, "inner": INNER, "shapes": []}
    for N, d in ((100, 10), (60, 16)):
        X, y, lengths, noise, derivs, cands, disc = workload(N, d)
        gp = capi.GaussianProcess(capi.SQUARE_EXPONENTIAL, 1.0, lengths, X, y, noise, derivs)
        best = float(gp.posterior(disc[:, None, :], (), ("mean",))["mean"].min())
        plan = capi.KGPlan(gp, MC, best, INNER, np.tile([0.0, 1.0], d), disc, NC, 1, seed=7, want_grad=True)
        plan.upload(cands)
        totals, mcs = [], []
        for r in range(args.runs + 1):  # run 0 is the warm-up
            plan.run()
            plan.sync()
            kg, _, _ = plan.download()
            total, mc_ms, _ = plan.timings()
            if r:
                totals.append(total)
                mcs.append(mc_ms)
        assert np.all(np.isfinite(kg))
        t, m = float(np.median(totals)), float(np.median(mcs))
        row = {"N": N, "d": d, "g": d, "n": N * (1 + d), "plan_run_ms": t, "mc_kernel_ms": m,
               "plan_runs_ms": totals, "sample_evals_per_s_plan": NC * MC / (t * 1e-3),
               "sample_evals_per_s_mc_kernel": NC * MC / (m * 1e-3)}
        row["cpu_reference_one_core"] = cpu_reference(X, y, lengths, noise, derivs, cands[0], disc, best,
                                                      args.cpu_samples)
        out["shapes"].append(row)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

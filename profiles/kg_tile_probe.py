"""Times `kg_mc_kernel` at the bench shape (c3: N=500, d=8, q=8, num_mc=16384, 1024 candidates, SquareExponential)
through `KGPlan.timings()` for the library named by CMOE_B200_LIB (default: the in-tree build), and prints one JSON line:
kernel and step times, the per-sample round counts (point_evals, line_batches, posterior_evals and line_search_steps per
mc_sample), and the card name, power limit and SM clock read in the same run.

With --counters DIR it also evaluates every candidate on its own and writes the four integer counters per candidate to
DIR/counters.npy ([candidates, 4]: posterior_evals, line_search_steps, point_evals, line_batches).  Two libraries that
take the same accept / reject decisions in every sample give identical arrays; a flipped Armijo or step-tolerance decision
changes the counters of its candidate.

    CMOE_B200_LIB=... python profiles/kg_tile_probe.py [--runs 5] [--counters DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, INNER_GD, SEED_PHILOX, make_workload  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

KEYS = ("posterior_evals", "line_search_steps", "point_evals", "line_batches")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    line = out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in line.split(",")])) if line else {"error": out.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--counters", metavar="DIR", default=None)
    args = ap.parse_args()
    assert capi.device_count() > 0, "no CUDA device"
    w = CONFIGS["c3"]
    wl = make_workload(w)
    gp = capi.GaussianProcess(0, w["alpha"], wl["lengths"], wl["X"], wl["y"], wl["noise"], wl["derivs"])
    best = float(gp.posterior(wl["disc"][:, None, :], (), ("mean",))["mean"].min())
    cands = wl["cands"]
    plan = capi.KGPlan(gp, w["num_mc"], best, INNER_GD, wl["bounds"], wl["disc"], len(cands), w["q"], seed=SEED_PHILOX)
    plan.upload(cands)
    mc_ms, tot_ms = [], []
    for it in range(1 + args.runs):  # first run = warm-up
        plan.run()
        plan.sync()
        tot, mc, _ = plan.timings()
        if it > 0:
            mc_ms.append(mc)
            tot_ms.append(tot)
    _, _, st = plan.download()
    clocks = card()
    ns = max(1, st["mc_samples"])
    out = {"lib": capi.LIB_PATH, "shape": "N=500 d=8 q=8 num_mc=16384 candidates=1024 (bench c3, SE)",
           "kg_mc_kernel_ms": {"mean": float(np.mean(mc_ms)), "min": float(np.min(mc_ms)), "max": float(np.max(mc_ms))},
           "step_ms_mean": float(np.mean(tot_ms)), "mc_samples": st["mc_samples"],
           "per_sample": {k: st[k] / ns for k in KEYS}, "totals": {k: st[k] for k in KEYS}, "card": clocks}
    del plan
    if args.counters:
        one = capi.KGPlan(gp, w["num_mc"], best, INNER_GD, wl["bounds"], wl["disc"], 1, w["q"], seed=SEED_PHILOX)
        cnt = np.zeros((len(cands), len(KEYS)), dtype=np.int64)
        for c in range(len(cands)):
            one.upload(cands[c:c + 1])
            one.run()
            one.sync()
            _, _, s = one.download()
            cnt[c] = [s[k] for k in KEYS]
        os.makedirs(args.counters, exist_ok=True)
        np.save(os.path.join(args.counters, "counters.npy"), cnt)
        out["counters"] = os.path.join(args.counters, "counters.npy")
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Times the q-KG accumulation kernel at the bench shape (c3: N=500, d=8, q=8, num_mc=16384, 1024 candidates,
SquareExponential) for the library named by CMOE_B200_LIB (default: the in-tree build), and prints one JSON line: the
accumulation and `kg_mc_kernel` times per step, the step time, and the card name, power limit and SM clock read in the
same run.

The step and `kg_mc_kernel` times come from `KGPlan.timings()` (CUDA events) over --runs unprofiled steps after one
warm-up step.  The per-kernel times come from a separate `torch.profiler` run of --profiled-runs steps: the summed
device time of every kernel whose name contains `kg_acc` (the scalar `kg_acc_kernel` or the tile `kg_acc_tile_kernel`),
and of `kg_mc_kernel`, per step.

    CMOE_B200_LIB=... python profiles/kg_acc_probe.py [--runs 3] [--profiled-runs 2]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from bench import CONFIGS, INNER_GD, SEED_PHILOX, make_workload  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402
from kg_tile_probe import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--profiled-runs", type=int, default=2)
    args = ap.parse_args()
    assert capi.device_count() > 0, "no CUDA device"
    import torch
    from torch.profiler import ProfilerActivity, profile

    w = CONFIGS["c3"]
    wl = make_workload(w)
    gp = capi.GaussianProcess(0, w["alpha"], wl["lengths"], wl["X"], wl["y"], wl["noise"], wl["derivs"])
    best = float(gp.posterior(wl["disc"][:, None, :], (), ("mean",))["mean"].min())
    cands = wl["cands"]
    plan = capi.KGPlan(gp, w["num_mc"], best, INNER_GD, wl["bounds"], wl["disc"], len(cands), w["q"], seed=SEED_PHILOX,
                       want_grad=True)
    plan.upload(cands)
    mc_ms, tot_ms = [], []
    for it in range(1 + args.runs):  # first run = warm-up
        plan.run()
        plan.sync()
        tot, mc, _ = plan.timings()
        if it > 0:
            mc_ms.append(mc)
            tot_ms.append(tot)
    clocks = card()
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.profiled_runs):
            plan.run()
            plan.sync()
        torch.cuda.synchronize()
    per_kernel = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per_kernel[e.name] += e.device_time_total / 1e3 / args.profiled_runs
    acc = {k: v for k, v in per_kernel.items() if "kg_acc" in k}
    mck = {k: v for k, v in per_kernel.items() if "kg_mc_kernel" in k}
    top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:8]
    out = {"lib": capi.LIB_PATH, "shape": "N=500 d=8 q=8 num_mc=16384 candidates=1024 (bench c3, SE, value + gradient)",
           "kg_acc_ms_per_step": sum(acc.values()), "kg_acc_kernels": acc,
           "kg_mc_kernel_ms_per_step_profiled": sum(mck.values()),
           "kg_mc_kernel_ms_events": {"mean": float(np.mean(mc_ms)), "min": float(np.min(mc_ms)),
                                      "max": float(np.max(mc_ms))},
           "step_ms": {"mean": float(np.mean(tot_ms)), "min": float(np.min(tot_ms)), "max": float(np.max(tot_ms))},
           "top_kernels_ms_per_step": {k[:90]: round(v, 3) for k, v in top}, "card": clocks}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

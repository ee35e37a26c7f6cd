"""Accepted-trial histogram of the q-KG LINE rounds at the bench shape (c3: N=500, d=8, q=8, num_mc=16384, 1024
candidates, SquareExponential), and the cost model that sizes the tile instantiation's LINE batch (kg_line_batch,
DESIGN.md K6).

Needs a library whose kg_mc_inst_8 was compiled with -DCMOE_KG_TRIAL_HIST (the product build has no counters):

    profiles/build_variants.sh hist8 "-DCMOE_KG_TRIAL_HIST -DCMOE_LINE_BATCH_TILE=8"
    CMOE_B200_LIB=variants/libvar_hist8.so python profiles/kg_trial_hist_probe.py

It runs the c3 plan once and prints the table (rows: inner step index, columns: accepted trial index counted from a_0),
the batch, range-fallback and warp-vote counters, and one JSON line.  Cost model, per step of a warp and per 8 training
rows, in SM cycles of the FP64 pipe: a LINE round is two half-blocks of L(KB) = 391 - 16 (8 - KB) cycles (the
fp64_mix_probe figure for KB = 8, 2 cycles for each of the 8 FP64 instructions a trial adds to a half-block), a POINT
round one block of 407.  A step whose accepted index needs p batches of KB costs its lane p - 1 extra LINE rounds, each
with an idle POINT round for the rest of the warp, and the warp pays for its slowest lane: with the 32 lanes' steps
taken as independent, a warp step costs (2 L(KB) + 407) (1 + sum_m>=1 (1 - (1 - P[p > m])^32)).
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, INNER_GD, SEED_PHILOX, make_workload  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

STEPS, TRIALS = 16, 32  # kHistSteps, kHistTrials (kg_mc.cuh)
COUNTS = ("batches", "all_fail", "range_fallback", "warp_rounds", "idle_rounds", "idle_lanes")
LINE_HALF_BLOCK, POINT_BLOCK = 391.0, 407.0  # SM cycles at KB = 8 (profiles/fp64_mix_probe.cu, DESIGN.md K6)


def read_hist(reset):
    fn = capi.lib().cmoe_kg_trial_hist
    fn.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    out = np.zeros(STEPS * TRIALS + len(COUNTS), dtype=np.uint64)
    rc = fn(out.ctypes.data_as(ctypes.POINTER(ctypes.c_ulonglong)), int(reset))
    assert rc == 0, f"cmoe_kg_trial_hist: CUDA error {rc}"
    return out


def cost_model(by_index):
    tail = by_index[::-1].cumsum()[::-1] / max(1, by_index.sum())  # tail[i] = P[accepted index >= i]
    base = None
    rows = {}
    for kb in range(4, 9):
        lane = float(sum(tail[m * kb] for m in range(1, (TRIALS - 1) // kb + 1)))  # E[p - 1] of one lane
        warp = float(sum(1.0 - (1.0 - tail[m * kb]) ** 32 for m in range(1, (TRIALS - 1) // kb + 1)))
        cyc = (2 * (LINE_HALF_BLOCK - 16 * (8 - kb)) + POINT_BLOCK) * (1 + warp)
        base = cyc if kb == 8 else base
        rows[kb] = {"extra_batches_per_lane_step": lane, "extra_rounds_per_warp_step": warp,
                    "cycles_per_step_8rows": cyc}
    for kb in rows:
        rows[kb]["vs_kb8"] = rows[kb]["cycles_per_step_8rows"] / base
    return rows


def main():
    assert capi.device_count() > 0, "no CUDA device"
    if not hasattr(capi.lib(), "cmoe_kg_trial_hist"):
        sys.exit(f"{capi.LIB_PATH} has no trial histogram: build it with -DCMOE_KG_TRIAL_HIST (see the docstring)")
    w = CONFIGS["c3"]
    wl = make_workload(w)
    gp = capi.GaussianProcess(0, w["alpha"], wl["lengths"], wl["X"], wl["y"], wl["noise"], wl["derivs"])
    best = float(gp.posterior(wl["disc"][:, None, :], (), ("mean",))["mean"].min())
    cands = wl["cands"]
    plan = capi.KGPlan(gp, w["num_mc"], best, INNER_GD, wl["bounds"], wl["disc"], len(cands), w["q"], seed=SEED_PHILOX)
    plan.upload(cands)
    read_hist(reset=True)
    plan.run()
    plan.sync()
    _, _, st = plan.download()
    h = read_hist(reset=True)
    del plan
    table = h[:STEPS * TRIALS].reshape(STEPS, TRIALS).astype(np.int64)
    counts = dict(zip(COUNTS, (int(v) for v in h[STEPS * TRIALS:])))
    by_index = table.sum(axis=0)
    hi = int(np.nonzero(by_index)[0].max()) + 1 if by_index.any() else 1
    print("accepted trial index (from a_0) by inner step, bench shape c3:")
    print("step " + "".join(f"{k:>11d}" for k in range(hi)) + "      total")
    for s in range(STEPS):
        if table[s].any():
            print(f"{s:4d} " + "".join(f"{v:11d}" for v in table[s, :hi]) + f"{table[s].sum():11d}")
    tot = by_index.sum()
    print(" all " + "".join(f"{v:11d}" for v in by_index[:hi]) + f"{tot:11d}")
    print("   % " + "".join(f"{100.0 * v / max(1, tot):11.4f}" for v in by_index[:hi]))
    print("counters:", counts)
    model = cost_model(by_index)
    for kb, r in model.items():
        print(f"KB={kb}: {r['extra_batches_per_lane_step']:.3e} extra batches per lane step, "
              f"{r['extra_rounds_per_warp_step']:.3e} per warp step, "
              f"{r['cycles_per_step_8rows']:.1f} cycles per step and 8 rows ({r['vs_kb8']:.4f} x KB=8)")
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    smi = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    stats = {k: int(st[k]) for k in ("mc_samples", "posterior_evals", "line_search_steps", "point_evals", "line_batches")}
    print(json.dumps({"lib": capi.LIB_PATH, "by_step_and_index": table[:, :hi].tolist(),
                      "by_index": by_index[:hi].tolist(), "counters": counts, "stats": stats, "model": model,
                      "card": smi.stdout.strip()}))


if __name__ == "__main__":
    main()

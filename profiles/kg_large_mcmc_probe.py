"""Timing probe of the ensemble q-KG past 32 union rows (cmoe_kg_eval_mcmc on cmoe_kg_eval_large's stages, DESIGN.md
K18) at the settings of the reference's examples/main.py loop: M = 16 Matern-5/2 members, num_mc = 128, d = 6 with all
six partials observed (g = 6), q = 5 (Q = 35), N = 20 and 100, a 200-candidate value screen and a 20-candidate
value + gradient batch (the descent's batch).

Each shape is timed three ways (host clock ending in a synchronise, median of --reps after a warm-up):
* `ensemble_s`: the ensemble call, members in flight on their own streams;
* `serial_large_s`: the same members through 16 serial cmoe_kg_eval_large calls, summed on the host;
* `one_at_a_time_s`: the ensemble call with cmoe_set_option("ensemble_members_in_flight", 1).
It also checks that the three give the same bits.  The card's name and power limit are read at the start, and the SM
clock right after each shape's timed calls (`sm_clock_after`), in the same run.  The README figures come from
`python profiles/kg_large_mcmc_probe.py` (the default --reps 5).  Prints JSON lines; writes them to --out when given."""
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


def query(fields):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"],
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
    args = ap.parse_args()
    from cornell_moe_b200 import capi
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(json.dumps(d))

    emit({"card": query("name,power.limit,clocks.max.sm")})
    M, d, q, mc, num_pts = 16, 6, 5, 128, 10
    g_idx = tuple(range(d))
    rng = np.random.default_rng(0)
    for N in (20, 100):
        prob = make_problem(N, d, g_idx=g_idx, seed=N, noise=1e-2)
        hypers = np.concatenate([rng.uniform(0.8, 1.5, size=(M, 1)), rng.uniform(0.3, 0.8, size=(M, d))], axis=1)
        noises = rng.uniform(0.005, 0.02, size=(M, 1 + d))
        ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"])
        disc = rng.uniform(size=(M, num_pts, d))
        best = np.full(M, float(prob["y"][:: 1 + d].min()))
        for nc, grad in ((200, False), (20, True)):
            cands = rng.uniform(size=(nc, q, d))
            kw = dict(seed=1, grad=grad)

            def ensemble():
                return ens.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(d), disc, **kw)

            def serial():
                parts = [m.kg_large(cands, None, mc, best[i], EXAMPLE_INNER_GD, unit_bounds(d), disc[i], **kw)
                         for i, m in enumerate(ens.members)]
                return parts

            def one_at_a_time():
                capi.set_option("ensemble_members_in_flight", 1)
                try:
                    return ensemble()
                finally:
                    capi.set_option("ensemble_members_in_flight", 0)

            te = timed(ensemble, args.reps)
            ts = timed(serial, args.reps)
            to = timed(one_at_a_time, args.reps)
            clock = query("clocks.sm")
            a, b = ensemble(), one_at_a_time()
            parts = serial()
            va = a[0] if grad else a
            vs = np.zeros(nc)
            for x in parts:
                vs = vs + (x[0] if grad else x)
            same = bool(np.array_equal(va, vs / float(M)) and np.array_equal(va, b[0] if grad else b))
            emit({"shape": f"M={M} Matern52 N={N} d={d} g={d} q={q} Q={q * (1 + d)} num_mc={mc}", "candidates": nc,
                  "gradient": grad, "ensemble_s": te, "serial_large_s": ts, "one_at_a_time_s": to,
                  "ensemble_over_one_at_a_time": te / to, "identical": same, "reps": args.reps,
                  "sm_clock_after": clock})
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

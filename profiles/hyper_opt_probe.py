"""Times the hyper-parameter gradient at a list of sets (cmoe_grad_log_marginal_likelihood_list) against a loop of
single-set calls (cmoe_grad_log_marginal_likelihood) over the same sets, and the multistart hyper-parameter descent
(cmoe_hyperparameter_gradient_descent) against the reference's gradient on one host core, and prints one JSON line per
shape plus a markdown table, with the card name, power limit and SM clock read in the same run.

Shapes (N points, d dimensions, g observed partials) in {(20, 2, 0), (100, 6, 0), (50, 3, 3), (500, 8, 0)}, each with
16, 128 and 1024 sets drawn log-uniformly (alpha, lengths, noise), Matern-5/2 as the reference's Python boundary uses.
A time is the host wall clock of one whole call (list, descent) or of the whole loop (single), each of which ends in a
device synchronise; the median of --runs runs after one warm-up run.  The gradients of the two device paths are
compared as well.

The reference column is an order of magnitude only: the reference's single-set ComputeGradLogLikelihood (compiled into
oracle/_ref by __graft_entry__.build()) is timed on one host core over at most 16 of the sets, and multiplied by the
number of gradient evaluations the descent made (starts x steps x restarts, an upper bound: runs that converge stop
early).  Without oracle/_ref the column reads "not measured".

    python profiles/hyper_opt_probe.py [--runs 5] [--steps 10] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "profiles")]

import oracle as orc  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402
from lml_list_probe import NUM_SETS, SHAPES, card, timed, workload  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("hyper_opt_probe needs a CUDA device")
    ref = orc.load_reference() if orc.have_reference() else None
    info = card()
    gd = (0, a.steps, 1, 0, 0.5, 0.01, 0.2, 1e-12)  # tolerance tiny: every start takes every step
    rows = []
    for (N, d, g) in SHAPES:
        for ns in NUM_SETS:
            X, y, derivs, H = workload(N, d, g, ns)
            bounds = np.stack([H.min(axis=0) * 0.5, H.max(axis=0) * 2.0], axis=1)

            def batched():
                return capi.grad_log_marginal_likelihood_list(1, H, X, y, derivs)[1]

            def loop():
                return np.array([capi.grad_log_marginal_likelihood(1, h[0], h[1:1 + d], X, y, h[1 + d:], derivs)
                                 for h in H])

            def descent():
                return capi.hyperparameter_gradient_descent(1, gd, bounds, H, X, y, derivs)

            tb, gb = timed(batched, a.runs)
            tl, gl = timed(loop, a.runs)
            td, _ = timed(descent, a.runs)
            rel = float(np.max(np.abs(gb - gl)) / np.max(np.abs(gl)))
            tref = None
            if ref is not None:
                sub = H[:16]
                t0 = time.perf_counter()
                for h in sub:
                    ref.grad_log_marginal_likelihood(1, h[0], h[1:1 + d], X, y, h[1 + d:], derivs)
                per = (time.perf_counter() - t0) / sub.shape[0]
                tref = per * ns * a.steps
            row = dict(N=N, d=d, g=g, num_sets=ns, grad_list_ms=tb * 1e3, grad_loop_ms=tl * 1e3, speedup=tl / tb,
                       max_rel_diff=rel, descent_ms=td * 1e3, descent_steps=a.steps,
                       ref_descent_estimate_ms=None if tref is None else tref * 1e3, card=info)
            print(json.dumps(row), flush=True)
            rows.append(row)
    print(f"\n{info.get('name')}, power limit {info.get('power.limit')}, SM clock {info.get('clocks.sm')} "
          f"(max {info.get('clocks.max.sm')}); median of {a.runs} runs after a warm-up; descent: {a.steps} steps\n")
    print("| N | d | g | sets | gradient list (ms) | loop of single gradients (ms) | loop / list | descent (ms) "
          "| reference, one core (ms, order of magnitude) |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        refc = "not measured" if r["ref_descent_estimate_ms"] is None else f"~{r['ref_descent_estimate_ms']:.0f}"
        print(f"| {r['N']} | {r['d']} | {r['g']} | {r['num_sets']} | {r['grad_list_ms']:.2f} | "
              f"{r['grad_loop_ms']:.1f} | {r['speedup']:.1f}x | {r['descent_ms']:.1f} | {refc} |")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()

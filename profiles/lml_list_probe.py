"""Times the log marginal likelihood at a list of hyper-parameter sets (cmoe_log_marginal_likelihood_list) against a
loop of single-set calls (cmoe_log_marginal_likelihood) over the same sets, and prints one JSON line per shape plus a
markdown table, with the card name, power limit and SM clock read in the same run.

Shapes (N points, d dimensions, g observed partials) in {(20, 2, 0), (100, 6, 0), (50, 3, 3), (500, 8, 0)}, each with
16, 128 and 1024 sets drawn log-uniformly (alpha, lengths, noise), Matern-5/2 as the reference's Python boundary uses.
A time is the host wall clock of one whole call (list) or of the whole loop (single), both of which end in a device
synchronise; the median of --runs runs after one warm-up run.  The values of the two paths are compared as well.

    python profiles/lml_list_probe.py [--runs 5] [--json out.json]
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

SHAPES = [(20, 2, 0), (100, 6, 0), (50, 3, 3), (500, 8, 0)]
NUM_SETS = [16, 128, 1024]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    line = out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in line.split(",")])) if line else {"error": out.stderr.strip()}


def workload(N, d, g, num_sets, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, d))
    cols = [np.sin(3 * X).sum(axis=1)] + [3 * np.cos(3 * X[:, a]) for a in range(g)]
    y = np.stack(cols, axis=1) + 0.1 * rng.standard_normal((N, 1 + g))
    scale = np.sqrt(d / 8.0) if d >= 8 else 1.0
    H = np.concatenate([np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=(num_sets, 1))),
                        scale * np.exp(rng.uniform(np.log(0.2), np.log(1.5), size=(num_sets, d))),
                        np.exp(rng.uniform(np.log(1e-3), np.log(1e-1), size=(num_sets, 1 + g)))], axis=1)
    return X, y.ravel(), np.arange(g, dtype=np.int32), H


def timed(fn, runs):
    fn()  # warm-up
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("lml_list_probe needs a CUDA device")
    info = card()
    rows = []
    for (N, d, g) in SHAPES:
        for ns in NUM_SETS:
            X, y, derivs, H = workload(N, d, g, ns)

            def batched():
                return capi.log_marginal_likelihood_list(1, H, X, y, derivs)

            def loop():
                return np.array([capi.log_marginal_likelihood(1, h[0], h[1:1 + d], X, y, h[1 + d:], derivs) for h in H])

            tb, vb = timed(batched, a.runs)
            tl, vl = timed(loop, a.runs)
            fin = np.isfinite(vl)
            rel = float(np.max(np.abs(vb[fin] - vl[fin]) / np.abs(vl[fin]))) if fin.any() else 0.0
            row = dict(N=N, d=d, g=g, num_sets=ns, list_ms=tb * 1e3, loop_ms=tl * 1e3, speedup=tl / tb,
                       max_rel_diff=rel, same_inf=bool(np.array_equal(np.isinf(vb), np.isinf(vl))), card=info)
            print(json.dumps(row), flush=True)
            rows.append(row)
    print(f"\n{info.get('name')}, power limit {info.get('power.limit')}, SM clock {info.get('clocks.sm')} "
          f"(max {info.get('clocks.max.sm')}); median of {a.runs} runs after a warm-up\n")
    print("| N | d | g | sets | list call (ms) | loop of single calls (ms) | loop / list |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['N']} | {r['d']} | {r['g']} | {r['num_sets']} | {r['list_ms']:.2f} | {r['loop_ms']:.1f} | "
              f"{r['speedup']:.1f}x |")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()

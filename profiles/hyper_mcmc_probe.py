"""Whole-call timings of the hyper-parameter MCMC (cmoe_hyperparameter_mcmc, DESIGN.md K12) against the host-driven
patterns it replaces, at the re-training step of examples/main.py: max(16, 2 nh) walkers (the front end's n_chains),
2000 burn-in + 1000 chain steps,
Matern-5/2, default prior, noise-free model.  Every time ends in a device synchronise; device calls are the median of 5
after a warm-up.  Beside each device call, on the same data:
  (a) numpy stretch moves + one cmoe_log_marginal_likelihood_list call per half-step (INTEGRATION.md's pattern without
      emcee), timed over 200 steps and scaled to 3000;
  (b) one cmoe_log_marginal_likelihood call per walker per step (the unmodified front end), timed over 20 steps, scaled;
  (c) the reference's single-set likelihood on the CPU (oracle/_ref) times the walkers * 3001 calls, order of magnitude.
Run with CMOE_B200_LIB pointing at another build to compare builds in one session.  Usage:
  python profiles/hyper_mcmc_probe.py [--shapes 15,2,0 ...] [--out FILE]
Every row is printed as one JSON line; --out also writes them all to FILE."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cornell_moe_b200 import capi  # noqa: E402
import hyper_mcmc_ref as R  # noqa: E402

BURN, CHAIN = 2000, 1000
SHAPES = [(15, 2, 0), (15, 6, 0), (50, 3, 3), (100, 6, 0), (500, 8, 0)]


def smi(field):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().split("\n")[0]
    except (OSError, subprocess.CalledProcessError):
        return "not measured"


def problem(N, d, g):
    rng = np.random.default_rng(N + 10 * d + g)
    X = rng.uniform(0.0, 1.0, size=(N, d))
    derivs = np.arange(g, dtype=np.int32)
    cols = [np.sin(3.0 * X).sum(axis=1)] + [3.0 * np.cos(3.0 * X[:, a]) for a in derivs]
    y = np.stack(cols, axis=1).ravel()
    p0 = R.initial_walkers(np.random.default_rng(1), max(16, 2 * (2 + d + g)), d, g)
    return X, y, derivs, p0


def device_call(X, y, derivs, p0):
    p, _ = capi.hyperparameter_mcmc(1, p0, X, y, BURN, derivs=derivs, noisy=False, seed=5)
    return capi.hyperparameter_mcmc(1, p, X, y, CHAIN, derivs=derivs, noisy=False, seed=5, first_step=BURN)


def pattern_a(X, y, derivs, p0, steps):
    d, g = X.shape[1], derivs.size
    lml = lambda H: capi.log_marginal_likelihood_list(1, H, X, y, derivs)  # noqa: E731
    tables = R.random_state_tables(np.random.RandomState(0), steps, len(p0))
    R.stretch_chain(p0, steps, lambda P: R.log_prob(P, lml, d, g, False, True), tables)


def pattern_b(X, y, derivs, p0, steps):
    d, g = X.shape[1], derivs.size

    def lml(H):
        return [capi.log_marginal_likelihood(1, h[0], h[1:1 + d], X, y, h[1 + d:], derivs) for h in H]

    tables = R.random_state_tables(np.random.RandomState(0), steps, len(p0))
    R.stretch_chain(p0, steps, lambda P: R.log_prob(P, lml, d, g, False, True), tables)


def median_time(f, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="*", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-host", action="store_true", help="device calls only")
    args = ap.parse_args()
    shapes = [tuple(int(v) for v in s.split(",")) for s in args.shapes] if args.shapes else SHAPES
    meta = {"lib": capi.LIB_PATH, "gpu": smi("name"), "power_limit": smi("power.limit"),
            "sm_clock": smi("clocks.sm"), "steps": BURN + CHAIN}
    print(json.dumps(meta), flush=True)
    try:
        import oracle as orc
        ref = orc.load_reference() if orc.have_reference() else None
    except Exception:  # noqa: BLE001
        ref = None
    rows = []
    for N, d, g in shapes:
        X, y, derivs, p0 = problem(N, d, g)
        device_call(X, y, derivs, p0)  # warm-up
        t_dev = median_time(lambda: device_call(X, y, derivs, p0), 5)
        row = {"N": N, "d": d, "g": g, "walkers": len(p0), "device_s": t_dev,
               "device_per_step_us": 1e6 * t_dev / (BURN + CHAIN)}
        if not args.skip_host:
            sa = 200
            pattern_a(X, y, derivs, p0, 5)
            row["a_s"] = median_time(lambda: pattern_a(X, y, derivs, p0, sa), 1) * (BURN + CHAIN) / sa
            sb = 20
            row["b_s"] = median_time(lambda: pattern_b(X, y, derivs, p0, sb), 1) * (BURN + CHAIN) / sb
            if ref is not None:
                h = np.exp(p0[0])
                t0 = time.perf_counter()
                for _ in range(20):
                    ref.log_marginal_likelihood(1, h[0], h[1:1 + d], X, y, np.full(1 + g, 1e-8), derivs)
                row["c_s"] = (time.perf_counter() - t0) / 20 * len(p0) * (BURN + CHAIN + 1)
            else:
                row["c_s"] = "not measured"
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"meta": meta, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()

"""Whole-call timings of the hyper-parameter MAP fit (cmoe_hyperparameter_map, DESIGN.md K19) against the host-driven
pattern it replaces: GaussianProcessLogLikelihoodMCMC.optimize, scipy.optimize.minimize(nll, p0) (BFGS with
finite-difference gradients) over one synchronising device fit per objective call.  Matern-5/2, default prior,
noisy = True, starts drawn like DefaultPrior's samples.  Per shape and start count:
  device_s      the device call's host time, ending in a synchronise: median of 9 after a warm-up;
  rounds        the largest per-start evaluation count (every round evaluates one trial of every active start);
  iterations / evaluations   summed over the starts;
  a_s           (a) the unmodified pattern, scipy BFGS over GPP.compute_log_likelihood, run from every start (at most 16
                of them, then scaled to the start count), with its summed nfev;
  c_s           (b) one host core through the reference (oracle/_ref): one likelihood call timed, times (a)'s nfev;
                an order of magnitude.
Usage: python profiles/hyper_map_probe.py [--shapes 20,2,0 ...] [--starts 1 16 128] [--out FILE] [--skip-host]
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
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

from cornell_moe_b200 import capi  # noqa: E402
import hyper_map_ref as M  # noqa: E402
import hyper_mcmc_ref as R  # noqa: E402

SHAPES = [(20, 2, 0), (100, 6, 0), (50, 3, 3), (500, 8, 0)]
STARTS = [1, 16, 128]
HOST_STARTS = 16


def smi(field):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().split("\n")[0]
    except (OSError, subprocess.CalledProcessError):
        return "not measured"


def problem(N, d, g, S):
    rng = np.random.default_rng(N + 10 * d + g)
    X = rng.uniform(0.0, 1.0, size=(N, d))
    derivs = np.arange(g, dtype=np.int32)
    cols = [np.sin(3.0 * X).sum(axis=1)] + [3.0 * np.cos(3.0 * X[:, a]) for a in derivs]
    y = (np.stack(cols, axis=1) + 0.1 * rng.standard_normal((N, 1 + g))).ravel()
    p0 = R.initial_walkers(np.random.default_rng(1), S, d, g)
    return X, y, derivs, p0


def gpp_nll(X, y, derivs):
    import GPP as C_GP
    N, d = X.shape
    g = derivs.size
    Xl, yl, dl = list(X.ravel()), list(y), list(int(v) for v in derivs)

    def lml(h):
        try:
            return C_GP.compute_log_likelihood(Xl, yl, d, N, C_GP.LogLikelihoodTypes.log_marginal_likelihood,
                                               [float(h[0]), list(h[1:1 + d])], dl, g, list(h[1 + d:]))
        except Exception:  # noqa: BLE001  a singular fit: the reference carries on with a garbage value
            return -np.inf

    return lambda t: M.nll(t, lml, d, g, True, True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="*", default=None)
    ap.add_argument("--starts", nargs="*", type=int, default=STARTS)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-host", action="store_true", help="device calls only")
    args = ap.parse_args()
    shapes = [tuple(int(v) for v in s.split(",")) for s in args.shapes] if args.shapes else SHAPES
    meta = {"lib": capi.LIB_PATH, "gpu": smi("name"), "power_limit": smi("power.limit"), "sm_clock": smi("clocks.sm")}
    print(json.dumps(meta), flush=True)
    try:
        import oracle as orc
        ref = orc.load_reference() if orc.have_reference() else None
    except Exception:  # noqa: BLE001
        ref = None
    rows = []
    for N, d, g in shapes:
        for S in args.starts:
            X, y, derivs, p0 = problem(N, d, g, S)
            call = lambda: capi.hyperparameter_map(1, p0, X, y, derivs, noisy=True, default_prior=True)  # noqa
            r = call()  # warm-up
            ts = []
            for _ in range(9):
                t0 = time.perf_counter()
                call()
                ts.append(time.perf_counter() - t0)
            row = {"N": N, "d": d, "g": g, "starts": S, "device_s": float(np.median(ts)),
                   "rounds": int(r["evaluations"].max()), "iterations": int(r["iterations"].sum()),
                   "evaluations": int(r["evaluations"].sum()),
                   "status": {str(k): int(v) for k, v in zip(*np.unique(r["status"], return_counts=True))}}
            if not args.skip_host and S <= HOST_STARTS or (not args.skip_host and S == max(args.starts)):
                from scipy import optimize
                nll = gpp_nll(X, y, derivs)
                k = min(S, HOST_STARTS)
                nfev, t0 = 0, time.perf_counter()
                for s in range(k):
                    res = optimize.minimize(nll, p0[s])
                    nfev += res.nfev
                row["a_s"] = (time.perf_counter() - t0) * S / k
                row["a_nfev"] = int(nfev * S / k)
                if ref is not None:
                    h = np.exp(p0[0])
                    t1 = time.perf_counter()
                    for _ in range(5):
                        ref.log_marginal_likelihood(1, h[0], h[1:1 + d], X, y, h[1 + d:], derivs)
                    row["c_s"] = (time.perf_counter() - t1) / 5 * row["a_nfev"]
                else:
                    row["c_s"] = "not measured"
            rows.append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"meta": meta, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()

"""Times the discretisation step of the MCMC q-KG loop (examples/main.py:172-197 of the reference, then best_so_far per
member) two ways in one process, alternating them:
  (a) cmoe_posterior_mean_optima_mcmc: one call for all members;
  (b) the loop of single-GP calls it replaces: per member one cmoe_gp_posterior for the screen, one
      cmoe_posterior_mean_optimization, the fallback on the host, one cmoe_gp_posterior for best_so_far
      (stage 2 of profiles/suggest_probe.py).
M = 16 Matern-5/2 members; (N, d) in {(20, 2), (50, 2), (500, 8), (2000, 10)}; screens of 1e3 and 1e4 points plus the
member's sampled points, shared by the members; 10 shared discretisation points; the descent with main.py's
cpp_sgd_params_ps (6 steps, 1 restart) and a longer one (50 steps, 3 restarts).

Every figure is the host wall-clock time of a whole call ending in a device synchronise: median (min-max) of --runs
after one warm-up of each.  The two ways must return the same kept_start and optima within 1e-7, or the script fails.
After the timed passes a torch.profiler pass over (a) gives the device time of its three kernels per shape; what is
left of (a) is the upload, the download, the launches and the synchronise.  Prints one JSON line with the card name,
power limit and SM clock read in the same run.  Fails without a CUDA device.

    python profiles/pm_optima_probe.py [--runs 9]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

from cornell_moe_b200 import capi  # noqa: E402

M, NUM_SHARED = 16, 10
DESCENTS = {"6 steps x 1 restart": [1, 6, 1, 3, 0.0, 1.0, 0.1, 1e-10],   # cpp_sgd_params_ps, examples/main.py:123-130
            "50 steps x 3 restarts": [1, 50, 3, 3, 0.7, 1.0, 0.1, 1e-10]}
SHAPES = ((20, 2), (50, 2), (500, 8), (2000, 10))
SCREENS = (1000, 10000)
KERNELS = ("pm_members_screen_kernel", "pm_members_argmin_kernel", "pm_members_opt_kernel")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    line = out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in line.split(",")])) if line else {"error": out.stderr.strip()}


def workload(N, d, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, d))
    y = np.sin(3 * X).sum(axis=1) + 0.1 * rng.standard_normal(N)
    lengths = rng.uniform(0.3, 0.6, (M, d)) * (np.sqrt(d / 2.0))
    hypers = np.column_stack([rng.uniform(0.5, 2.0, M), lengths])
    ens = capi.GaussianProcessEnsemble(hypers, np.full((M, 1), 1e-2), X, y, kernel=capi.MATERN_NU_2P5)
    return ens, X, rng.uniform(size=(max(SCREENS), d)), rng.uniform(size=(NUM_SHARED, d)), np.tile([0.0, 1.0], d)


def loop_of_single_calls(ens, X, pts, shared, gd, bounds):
    optima, kept, best = np.empty((M, X.shape[1])), np.empty(M, dtype=int), np.empty(M)
    screen = np.concatenate([pts, X])
    for m, gp in enumerate(ens.members):
        mu = gp.posterior(screen[:, None, :], (), ("mean",))["mean"].ravel()
        x0 = screen[np.argmin(mu)]
        end, val, _ = capi.posterior_mean_optimization(gp, x0, gd, bounds)
        kept[m] = -val > mu.min()
        optima[m] = x0 if kept[m] else end
        disc = np.concatenate([shared, optima[m][None]])
        best[m] = gp.posterior(disc[:, None, :], (), ("mean",))["mean"].min()
    return optima, kept, best


def stats(ts):
    return {"median_ms": float(np.median(ts)) * 1e3, "min_ms": float(np.min(ts)) * 1e3, "max_ms": float(np.max(ts)) * 1e3}


def kernel_times_us(fn, repeats=5):
    """Device time per call of each of the three kernels (all launches of one call added), from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
    return {k: v / repeats for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=9)
    args = ap.parse_args()
    assert capi.device_count() > 0, "no CUDA device"
    out = {"card": card(), "M": M, "num_shared": NUM_SHARED, "runs": args.runs, "rows": []}
    calls = []
    for N, d in SHAPES:
        ens, X, all_pts, shared, bounds = workload(N, d)
        for P in SCREENS:
            pts = all_pts[:P]
            for name, gd in DESCENTS.items():
                def one(ens=ens, pts=pts, gd=gd, bounds=bounds, shared=shared):
                    return ens.posterior_mean_optima(pts, gd, bounds, 0, True, shared)

                def loop(ens=ens, X=X, pts=pts, gd=gd, bounds=bounds, shared=shared):
                    return loop_of_single_calls(ens, X, pts, shared, gd, bounds)

                a, (b_opt, b_kept, b_best) = one(), loop()  # warm-up of both, and the comparison
                assert np.array_equal(a.kept_start, b_kept), (N, d, P, name, a.kept_start, b_kept)
                diff = float(np.abs(a.optima - b_opt).max())
                assert diff <= 1e-7, (N, d, P, name, diff)
                assert np.allclose(a.best_so_far, b_best, rtol=1e-9, atol=0), (N, d, P, name)
                ta, tb = [], []
                for _ in range(args.runs):
                    t0 = time.perf_counter()
                    one()
                    t1 = time.perf_counter()
                    loop()
                    t2 = time.perf_counter()
                    ta.append(t1 - t0)
                    tb.append(t2 - t1)
                row = {"N": N, "d": d, "screen_points": P, "descent": name, "one_call": stats(ta),
                       "loop_of_3M_calls": stats(tb), "max_abs_optima_difference": diff,
                       "kept_start": int(a.kept_start.sum())}
                row["loop_over_one_call"] = row["loop_of_3M_calls"]["median_ms"] / row["one_call"]["median_ms"]
                out["rows"].append(row)
                calls.append((row, one))
    # the profiler pass, after every timed pass (tracing slows the host)
    for row, one in calls:
        row["kernel_us"] = kernel_times_us(one)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

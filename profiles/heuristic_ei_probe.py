"""Times heuristic batch EI (DESIGN.md K20) three ways at the GPP level, in one process:
  (a) GPP.heuristic_expected_improvement_optimization (Constant Liar, lie = min y): one call, one descent launch per
      round;
  (b) the loop of existing calls it replaces: per round GPP.multistart_expected_improvement_optimization with q = 1
      (its descent driven from the host, one synchronising posterior call per step), the posterior mean and variance
      at the chosen point and add_sampled_points on a copy of the GP;
  (c) for context, Monte-Carlo q-EI over the same q by multistart_expected_improvement_optimization,
      max_int_steps = 1e4.
(N, d) in {(50, 2), (500, 8), (2000, 10)} (Matern-5/2), q in {2, 4, 16}, with main.py's cpp_sgd_params_kg (200
starts, 50 steps x 2 restarts) and the reference's demo parameters (50 starts, 300 steps x 4 restarts, gamma 0.6).

Every figure is the host wall-clock time of a whole call, which returns host lists and so ends after the device work:
median (min-max) of --runs after one warm-up.  A configuration whose warm-up alone takes longer than --slow seconds is
timed --slow-runs times instead (its row says how many); once --budget seconds have passed the remaining
configurations are recorded as not measured.  Each row records the largest difference between the points of (a) and
(b).  A separate torch.profiler pass over (a) at N >= 500 gives the device time per kernel name and its share of the
call's wall time.
With --out PATH it rewrites the JSON result at PATH after every row, so a run stopped early keeps its finished rows;
it prints the result at the end, with the card name, power limit and SM clock read in the same run.  Fails without a
CUDA device.

    python profiles/heuristic_ei_probe.py [--runs 9] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "cornell-moe_b200")]

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

PARAMS = {"main.py cpp_sgd_params_kg": [200, 50, 2, 4, 0.7, 1.0, 0.5, 1.0e-10],
          "demo (50 starts, 300 x 4, gamma 0.6)": [50, 300, 4, 0, 0.6, 1.0, 1.0, 1.0e-6]}
SHAPES = ((50, 2), (500, 8), (2000, 10))
QS = (2, 4, 16)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    line = out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else ""
    return dict(zip(q.split(","), [v.strip() for v in line.split(",")])) if line else {"error": out.stderr.strip()}


def problem(N, d, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, d))
    y = np.sin(3 * X).sum(axis=1) + 0.1 * rng.standard_normal(N)
    lengths = list(np.full(d, 0.5 * np.sqrt(max(d, 2) / 2.0)))
    return X, y, lengths


def gpp_gp(X, y, lengths):
    return C_GP.GaussianProcess([1.0, lengths], list(X.ravel()), list(y), [0.01], [], 0, X.shape[1], X.shape[0])


def params_of(gd, opt=C_GP.OptimizerTypes.gradient_descent):
    return type("P", (), dict(domain_type=C_GP.DomainTypes.tensor_product, optimizer_type=opt, num_random_samples=16,
                              optimizer_parameters=C_GP.GradientDescentParameters(*gd)))


def rnd():
    r = C_GP.RandomnessSourceContainer(1)
    r.SetExplicitUniformGeneratorSeed(5)
    return r


def stats(ts):
    return {"n": len(ts), "median_ms": float(np.median(ts)) * 1e3, "min_ms": float(np.min(ts)) * 1e3,
            "max_ms": float(np.max(ts)) * 1e3}


def timed(fn, runs, slow, slow_runs):
    t0 = time.perf_counter()
    res = fn()
    warm = time.perf_counter() - t0
    ts = []
    for _ in range(runs if warm <= slow else slow_runs):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return res, stats(ts)


def kernel_breakdown(fn):
    """Device time per kernel name in one call of fn, and the call's wall time, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e6
    ker = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if t > 0:
            ker[ev.key[:80]] = float(t)
    total = sum(ker.values())
    top = dict(sorted(ker.items(), key=lambda kv: -kv[1])[:8])
    descent = sum(v for k, v in ker.items() if "hei_descent_kernel" in k)
    return {"wall_us_profiled": wall, "device_us_all_kernels": total, "hei_descent_kernel_us": descent,
            "descent_share_of_wall": descent / wall if wall > 0 else None, "top_kernels_us": top}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=9)
    ap.add_argument("--slow", type=float, default=3.0)
    ap.add_argument("--slow-runs", type=int, default=2)
    ap.add_argument("--budget", type=float, default=900.0)
    ap.add_argument("--out", default=None, help="JSON file rewritten after every row")
    args = ap.parse_args()
    assert capi.device_count() > 0, "no CUDA device"
    out = {"card": card(), "runs": args.runs, "rows": [], "profile": []}
    start = time.perf_counter()

    def save():
        if args.out:
            with open(args.out, "w") as f:
                json.dump(out, f, indent=1)

    for pname, gd in PARAMS.items():
        for N, d in SHAPES:
            X, y, lengths = problem(N, d)
            best = float(y.min())
            bounds = list(np.tile([0.0, 1.0], d))
            gp = gpp_gp(X, y, lengths)
            prm = params_of(gd)
            for q in QS:
                row = {"params": pname, "N": N, "d": d, "q": q}
                if time.perf_counter() - start > args.budget:
                    row["not_measured"] = "time budget of the probe run exhausted"
                    out["rows"].append(row)
                    continue

                def device(q=q, gp=gp, prm=prm, bounds=bounds, best=best):
                    return C_GP.heuristic_expected_improvement_optimization(
                        prm, gp, bounds, C_GP.ConstantLiarEstimationPolicy(best, 0.01), q, best, 1, rnd(), {})

                def loop(q=q, X=X, y=y, lengths=lengths, prm=prm, bounds=bounds, best=best, d=d):
                    g = gpp_gp(X, y, lengths)
                    r = rnd()
                    pts = []
                    for _ in range(q):
                        pt = C_GP.multistart_expected_improvement_optimization(prm, g, bounds, [], 1, 0, best, 1000, 1,
                                                                               False, 0, r, {})
                        g.compute_mean_of_points(pt, 1)
                        g.compute_variance_of_points(pt, 1)
                        g.add_sampled_points(pt, [best], 1)
                        pts.extend(pt)
                    return pts

                def mc(q=q, gp=gp, prm=prm, bounds=bounds, best=best):
                    return C_GP.multistart_expected_improvement_optimization(prm, gp, bounds, [], q, 0, best, 10000, 1,
                                                                             False, 0, rnd(), {})

                a, row["a_device_call"] = timed(device, args.runs, args.slow, args.slow_runs)
                b, row["b_loop_of_existing_calls"] = timed(loop, args.runs, args.slow, args.slow_runs)
                row["max_abs_point_difference"] = float(np.abs(np.array(a) - np.array(b)).max())
                row["b_over_a"] = row["b_loop_of_existing_calls"]["median_ms"] / row["a_device_call"]["median_ms"]
                if time.perf_counter() - start > args.budget:
                    row["c_mc_qei"] = "not measured: time budget of the probe run exhausted"
                else:
                    _, row["c_mc_qei"] = timed(mc, args.runs, args.slow, args.slow_runs)
                out["rows"].append(row)
                save()
                print(json.dumps(row), flush=True)
    # the profiler pass, separate from the timed passes (tracing slows the host)
    gd = PARAMS["main.py cpp_sgd_params_kg"]
    for N, d in SHAPES[1:]:
        X, y, lengths = problem(N, d)
        best = float(y.min())
        gp = gpp_gp(X, y, lengths)
        bounds = list(np.tile([0.0, 1.0], d))

        def device(gp=gp, bounds=bounds, best=best):
            return C_GP.heuristic_expected_improvement_optimization(
                params_of(gd), gp, bounds, C_GP.ConstantLiarEstimationPolicy(best, 0.01), 4, best, 1, rnd(), {})

        out["profile"].append({"params": "main.py cpp_sgd_params_kg", "N": N, "d": d, "q": 4,
                               **kernel_breakdown(device)})
        save()
    out["card_after"] = card()
    save()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Before / after probe of the q-KG start-point table at the bench shape (c3: N=500, d=8, q=8, num_mc=16384, 1024
candidates, SquareExponential).  Alternates two libraries — one built from the commit before the table (a sample's
inner descent starts with a POINT round) and the in-tree one — in separate processes (profiles/kg_tile_probe.py, which
reads the card, power limit and SM clock in the same run), and prints one JSON line per run and a summary line: the
`kg_mc_kernel` and step times, and the four counters (posterior evaluations, accepted steps, POINT rounds, LINE batches).

Build the parent library once, from a checkout of the parent commit:
    git worktree add /tmp/parent HEAD~1 && make -C /tmp/parent/cornell-moe_b200 lib
    python profiles/kg_start_probe.py --parent /tmp/parent/cornell-moe_b200/libcornell_moe_b200.so [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("posterior_evals", "line_search_steps", "point_evals", "line_batches")


def run_one(lib, runs):
    env = dict(os.environ, CMOE_B200_LIB=lib)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "profiles", "kg_tile_probe.py"), "--runs", str(runs)],
                         env=env, capture_output=True, text=True, check=True)
    return json.loads(out.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True, help="library built from the commit before the start-point table")
    ap.add_argument("--new", default=os.path.join(ROOT, "cornell-moe_b200", "libcornell_moe_b200.so"))
    ap.add_argument("--rounds", type=int, default=3, help="parent / new alternations")
    ap.add_argument("--runs", type=int, default=3, help="timed plan runs per process (after one warm-up run)")
    args = ap.parse_args()
    res = {"parent": [], "new": []}
    for r in range(args.rounds):
        for name, lib in (("parent", args.parent), ("new", args.new)):
            o = run_one(lib, args.runs)
            res[name].append(o)
            print(json.dumps({"round": r, "build": name, "kg_mc_kernel_ms": o["kg_mc_kernel_ms"]["mean"],
                              "step_ms": o["step_ms_mean"], "totals": o["totals"], "card": o["card"]}), flush=True)
    summ = {}
    for name, rs in res.items():
        mc = [o["kg_mc_kernel_ms"]["mean"] for o in rs]
        st = [o["step_ms_mean"] for o in rs]
        summ[name] = {"kg_mc_kernel_ms": {"mean": float(np.mean(mc)), "min": float(np.min(mc)), "max": float(np.max(mc))},
                      "step_ms": {"mean": float(np.mean(st)), "min": float(np.min(st)), "max": float(np.max(st))},
                      "totals": rs[-1]["totals"]}
    summ["step_gain"] = 1.0 - summ["new"]["step_ms"]["mean"] / summ["parent"]["step_ms"]["mean"]
    summ["kernel_gain"] = 1.0 - summ["new"]["kg_mc_kernel_ms"]["mean"] / summ["parent"]["kg_mc_kernel_ms"]["mean"]
    summ["counter_delta"] = {k: summ["new"]["totals"][k] - summ["parent"]["totals"][k] for k in KEYS}
    summ["card"] = res["new"][-1]["card"]
    print(json.dumps(summ))


if __name__ == "__main__":
    main()

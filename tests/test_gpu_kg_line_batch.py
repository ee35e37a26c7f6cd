"""GPU parity of the LINE batch of the tile instantiation `kg_mc_kernel<SE,8,8>`, which tries 6 step sizes per batch
(`kg_line_batch`, kg_mc.cuh) where the other instantiations try 8, against the CPU checker with table-fed normals:
- a short length scale (0.15), where most steps accept trial 6 or 7: a second LINE batch with 6 trials, rarely one
  with 8;
- initial step sizes a_0 = 128, where a_0 |p_j| reaches the range bound 512 of the batched trials (checked as a_min
  |p_j| < 512 / 2^5 with 6 trials) in about two fifths of the steps: those steps fall back to one-at-a-time trials and
  the others run batched.
The torch.profiler check confirms that both cases run the tile instantiation."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from gpu_util import checker
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

pytestmark = pytest.mark.gpu

# name: (N, length scale, inner optimiser)
CASES = {
    "short_length_scale": (200, 0.15, EXAMPLE_INNER_GD),
    "near_range_bound": (67, 0.5, [1, 5, 2, 3, 0.0, 128.0, 0.5, 1e-10]),
}


def _inputs(name):
    N, length, gd = CASES[name]
    prob = make_problem(N, 8, seed=9, noise=0.1, length=length)
    rng = np.random.default_rng(41)
    q, mc = 8, 64
    cands = rng.uniform(size=(2, q, 8))
    disc = rng.uniform(size=(5, 8))
    table = rng.standard_normal((mc // 2) * q)
    return prob, gd, cands, disc, table, mc


def _device_gp(capi, prob):
    return capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])


def kernel_names(name):
    """Names of the CUDA kernels the q-KG call of case `name` launches (torch.profiler)."""
    import torch
    from cornell_moe_b200 import capi
    from torch.profiler import ProfilerActivity, profile
    prob, gd, cands, disc, table, mc = _inputs(name)
    gp = _device_gp(capi, prob)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gp.kg(cands, None, mc, 0.0, gd, unit_bounds(8), disc, table=table, grad=True)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events()})


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


@pytest.mark.parametrize("name", sorted(CASES))
def test_tile_line_batch_matches_checker(capi, name):
    prob, gd, cands, disc, table, mc = _inputs(name)
    gp = _device_gp(capi, prob)
    ref, lm = checker().gp(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    best = float(ref.mean_additional(disc).min())
    kg, grad, st = gp.kg(cands, None, mc, best, gd, unit_bounds(8), disc, table=table, grad=True, stats=True)
    print(name, st)
    if name == "short_length_scale":
        assert st["line_batches"] >= 1.5 * st["line_search_steps"]  # a second batch for most steps
    if name == "near_range_bound":
        # trials run one at a time (POINT rounds) in the fallback steps, and in LINE batches in the others
        assert st["point_evals"] > 2 * st["line_search_steps"]
        assert st["posterior_evals"] - st["point_evals"] - st["mc_samples"] > 2 * st["line_search_steps"]
    for c in range(2):
        v, g = ref.kg(cands[c], None, mc, best, table, gd, unit_bounds(8), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("name", sorted(CASES))
def test_line_batch_cases_run_the_tile_instantiation(name):
    """The profiler runs in a child process: a profiling session leaves CUPTI state behind that makes later sessions
    of the suite miss kernel records (tests/test_gpu_amplitude.py)."""
    tests = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys, json; sys.path[:0] = [{os.path.dirname(tests)!r}, {tests!r}]; "
            f"import test_gpu_kg_line_batch as t; print(json.dumps(t.kernel_names({name!r})))")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().splitlines()[-1])
    assert any("kg_mc_kernel<0, 8, 8, " in n for n in names), names

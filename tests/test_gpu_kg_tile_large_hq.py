"""GPU parity of the q-KG tile kernels far from the exponent's origin: a length scale of 0.03 on the unit box puts the
scaled training points up to ~40 length scales from the centre (the training points' mean).  The candidates, pending
points and discrete points are put within about one length scale of the training points farthest from the centre, so
every query point has training rows with kernel values near 1 while its per-sample term hq = -|x~|^2/2 is several
hundred and the row exponents e_j + x~ . X~_j are as large before they cancel.  The BIG build of `kg_mc_kernel<SE,8,8>`
and `kg_acc_tile_kernel<8,8>` carry hq as exp2k_shifted's rounding constant and a per-lane factor (kg_mc.cuh), so the
training rows, which dominate the compared values and gradients here, go through the cancellation and the split of hq.
The torch.profiler check confirms that these two kernels ran."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from gpu_util import checker
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

pytestmark = pytest.mark.gpu

# N = 300: many 8-row blocks and two row CTAs of the accumulation kernel; q + p = 8 and 7 (a padded union column)
CASES = [(300, 8, 0, 96), (300, 5, 2, 70)]


def _inputs(N, q, p, mc):
    prob = make_problem(N, 8, seed=5000 + N + q, noise=0.05, length=0.03)
    rng = np.random.default_rng(N + 13 * q + p)
    X = prob["X"]
    far = np.argsort(-np.sum((X - X.mean(axis=0)) ** 2, axis=1))[:32]  # the training points farthest from the centre

    def near(n):  # n points within about one length scale (0.01 per coordinate) of far training points
        return np.clip(X[rng.choice(far, n)] + 0.01 * rng.standard_normal((n, 8)), 0.0, 1.0)
    cands = near(2 * q).reshape(2, q, 8)
    Xp = near(p) if p else None
    disc = near(6)
    table = rng.standard_normal((mc // 2) * (q + p))
    return prob, cands, Xp, disc, table


def _query_regime(prob, pts):
    """For each query point: the largest training-row kernel value exp(-|x~ - X~_j|^2/2) and -hq = |x~|^2/2 in the
    centred frame of the kernels."""
    X, ls = prob["X"], prob["lengths"]
    c = X.mean(axis=0)
    xs, Xs = (pts - c) / ls, (X - c) / ls
    d2 = np.sum((xs[:, None, :] - Xs[None, :, :]) ** 2, axis=2)
    return np.exp(-0.5 * d2.min(axis=1)), 0.5 * np.sum(xs * xs, axis=1)


def _device_gp(capi, prob):
    return capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])


def kernel_names(case):
    """Names of the CUDA kernels the q-KG call of `case` launches (torch.profiler)."""
    import torch
    from cornell_moe_b200 import capi
    from torch.profiler import ProfilerActivity, profile
    N, q, p, mc = case
    prob, cands, Xp, disc, table = _inputs(N, q, p, mc)
    gp = _device_gp(capi, prob)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gp.kg(cands, Xp, mc, 0.0, EXAMPLE_INNER_GD, unit_bounds(8), disc, table=table, grad=True)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events()})


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


@pytest.mark.parametrize("case", CASES, ids=[f"N{c[0]}-q{c[1]}-p{c[2]}" for c in CASES])
def test_tile_kernels_match_checker_at_large_hq(capi, case):
    N, q, p, mc = case
    prob, cands, Xp, disc, table = _inputs(N, q, p, mc)
    # the regime this case is about: every query point (the inner searches start at the union and discrete points) has
    # training rows that matter, at |hq| of several hundred
    pts = np.concatenate([cands.reshape(-1, 8), disc] + ([Xp] if p else []))
    kmax, nhq = _query_regime(prob, pts)
    assert kmax.min() > 1e-2, kmax
    assert nhq.min() > 300.0, nhq
    gp = _device_gp(capi, prob)
    ref, lm = checker().gp(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, table=table, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], Xp, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(8), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("case", CASES, ids=[f"N{c[0]}-q{c[1]}-p{c[2]}" for c in CASES])
def test_large_hq_cases_run_the_big_tile_build(case):
    """The profiler runs in a child process: a profiling session leaves CUPTI state behind that makes later sessions
    of the suite miss kernel records (tests/test_gpu_amplitude.py)."""
    tests = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys, json; sys.path[:0] = [{os.path.dirname(tests)!r}, {tests!r}]; "
            f"import test_gpu_kg_tile_large_hq as t; print(json.dumps(t.kernel_names({case!r})))")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().splitlines()[-1])
    assert any("kg_mc_kernel<0, 8, 8, true>" in n for n in names), names
    assert any("kg_acc_tile_kernel" in n for n in names), names

"""GPU tests of the first-extremum rule (device_math.cuh: beats / block_best / best_of_parts_kernel) where the selected
index is visible: exact ties across threads, warps and CTAs resolve to the first occurrence, as np.argmin does.  The
per-member screen of the posterior-mean optima is covered by test_gpu_pm_optima.py."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

from cornell_moe_b200 import capi  # noqa: E402

from synth import make_problem  # noqa: E402

pytestmark = pytest.mark.gpu


def _gp(pr):
    return capi.GaussianProcess(0, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"])


def test_rff_grid_argmin_takes_the_first_of_tied_rows():
    """With zero frequencies every sample function is constant, so all grid rows tie exactly (over many threads and
    CTAs of the grid kernel), the gradient is zero and the optimiser keeps its start: the result is the first row."""
    pr = make_problem(30, 2, (), seed=4, noise=1e-2, length=0.4)
    gp = _gp(pr)
    F, P, G = 40, 3, 5000
    grid = np.random.default_rng(1).uniform(0.0, 1.0, size=(G, 2))
    rng = np.random.default_rng(2)
    table = {"omega": np.zeros((P, F, 2)), "b": rng.uniform(0.0, 2 * np.pi, size=(P, F)), "z": rng.normal(size=(P, F)),
             "eps": np.zeros((P, 30))}
    for first in (0, 3000):
        g = np.roll(grid, -first, axis=0)
        pts, _ = gp.sample_rff_optima(F, P, np.array([[0.0, 1.0], [0.0, 1.0]]), g, table=table)
        np.testing.assert_array_equal(pts, np.tile(g[0], (P, 1)))


def test_lcb_takes_the_first_of_duplicated_candidates():
    """q = 1: a copy of the winner placed before it, or far after it (another warp and thread of the selection CTA),
    wins only when it comes first.  q = 2: the same for the round's argmax over the satisfied set."""
    pr = make_problem(40, 3, (), seed=7, noise=1e-2, length=0.5)
    gp = _gp(pr)
    cand = np.random.default_rng(3).uniform(0.0, 1.0, size=(3000, 3))
    (a,), _, _ = gp.lower_confidence_bound(cand, 1)
    late = np.insert(cand, min(a + 1500, cand.shape[0]), cand[a], axis=0)
    assert gp.lower_confidence_bound(late, 1)[0][0] == a
    early = np.insert(cand, 0, cand[a], axis=0)
    assert gp.lower_confidence_bound(early, 1)[0][0] == 0
    i0, i1 = gp.lower_confidence_bound(cand, 2)[0]
    at = min(i1 + 1500, cand.shape[0])
    late = np.insert(cand, at, cand[i1], axis=0)
    np.testing.assert_array_equal(gp.lower_confidence_bound(late, 2)[0], [i0 + (i0 >= at), i1])
    early = np.insert(cand, 0, cand[i1], axis=0)
    np.testing.assert_array_equal(gp.lower_confidence_bound(early, 2)[0], [i0 + 1, 0])

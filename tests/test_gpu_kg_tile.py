"""GPU parity of the q-KG tile path (DMMA evaluation of the training rows on the shared-memory fast path, the
SquareExponential instantiation with padded DIM = 8 and QP = 8) against the CPU checker with table-fed normals: partial
last row blocks, zero-padded coordinates and union columns, partly empty warps, the LINE round's edge paths on a problem
with several row blocks, and independence of the lane a sample runs on."""
import numpy as np
import pytest

from gpu_util import checker
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def _pair(capi, kernel, prob):
    gp = capi.GaussianProcess(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                              prob["derivs"])
    ref, lm = checker().gp(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    return gp, ref


# N = 61: seven full blocks of 8 rows and a last block of 5; the union rows (U = q + p) follow.  Every case runs the
# <SE, 8, 8> instantiation: d = 7 pads the coordinates to 8 (a zero column in the fragments), q + p = 5 to 7 pads the
# union columns to 8 (zero columns in the weight fragments).
@pytest.mark.parametrize("dim,q,p", [(8, 8, 0), (8, 5, 0), (7, 3, 3), (7, 4, 3)])
def test_tile_partial_blocks_and_padding(capi, dim, q, p):
    prob = make_problem(61, dim, seed=100 + dim + q, noise=0.05)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(dim * 31 + q)
    cands = rng.uniform(size=(2, q, dim))
    Xp = rng.uniform(size=(p, dim)) if p else None
    disc = rng.uniform(size=(6, dim))
    mc = 24  # fewer samples than lanes: the warp is partly empty
    table = rng.standard_normal((mc // 2) * (q + p))
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, table=table, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], Xp, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(dim), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("case", ["second_batch", "out_of_range_factors", "exhausted_search"])
def test_tile_line_edge_paths(capi, case):
    """The LINE round's edge paths (second batch, factors out of range, exhausted search) with N = 67 rows, d = 8,
    q = 8 (the tile instantiation)."""
    gd = {"second_batch": [1, 5, 2, 3, 0.0, 32.0, 0.5, 1e-10],
          "out_of_range_factors": [1, 5, 2, 3, 0.0, 4096.0, 0.5, 1e-10],
          "exhausted_search": [1, 3, 2, 3, 0.0, 1e12, 0.5, 1e-10]}[case]
    prob = make_problem(67, 8, seed=9, noise=0.1)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(41)
    q, mc = 8, 40
    cands = rng.uniform(size=(2, q, 8))
    disc = rng.uniform(size=(5, 8))
    table = rng.standard_normal((mc // 2) * q)
    best = float(ref.mean_additional(disc).min())
    kg, grad, st = gp.kg(cands, None, mc, best, gd, unit_bounds(8), disc, table=table, grad=True, stats=True)
    print(case, st)
    if case == "second_batch":
        assert st["line_batches"] >= 1.5 * st["line_search_steps"]  # two batches for most steps ...
        assert st["point_evals"] < st["posterior_evals"] / 3  # ... and few one-at-a-time trials
    if case == "out_of_range_factors":
        assert st["point_evals"] > 5 * st["line_search_steps"]  # the trials were evaluated one at a time
    for c in range(2):
        v, g = ref.kg(cands[c], None, mc, best, table, gd, unit_bounds(8), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


def test_tile_results_do_not_depend_on_lane(capi):
    """N = 500, d = 8, q = 8, 65536 samples: 16 candidates in one call, and in subsets of 1 and of 5, give
    bit-identical values and gradients.  The plan sizes its sample chunks (samples per CTA) from candidates x samples:
    the 16-candidate call uses larger chunks than the 1- and 5-candidate calls, so most samples start on a different
    lane of a different CTA, on top of the refill order of the lanes' shared sample counter."""
    prob = make_problem(500, 8, seed=20260924 % 1000, noise=1e-2)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(11)
    cands = rng.uniform(size=(16, 8, 8))
    disc = rng.uniform(size=(10, 8))
    best = float(ref.mean_additional(disc).min())
    mc = 65536
    kg, grad = gp.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xC0FFEE, grad=True)
    assert np.all(np.isfinite(kg)) and np.all(np.isfinite(grad))
    for size in (1, 5):
        for s in range(0, 16, size):
            k, g = gp.kg(cands[s:s + size], None, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xC0FFEE,
                         grad=True)
            np.testing.assert_array_equal(k, kg[s:s + size])
            np.testing.assert_array_equal(g, grad[s:s + size])

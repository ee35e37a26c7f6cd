"""GPU parity of the q-KG tile accumulation kernel (`kg_acc_tile_kernel`: the envelope-theorem sums of the gradient on
FP64 DMMA, the SquareExponential instantiation with padded DIM = 8 and QP = 8 on the shared-memory fast path) against
the CPU checker with table-fed normals: sample counts that are not a multiple of the 8-sample groups or of the 64-sample
shared-memory tiles, training-row counts that leave the last 16-row tile and the last row CTA partly empty, zero-padded
coordinates (d = 7) and union columns (q + p < 8), pending points (p > 0); and independence of the batch a candidate is
evaluated in."""
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


def _pair(capi, prob):
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    ref, lm = checker().gp(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    return gp, ref


# N = 61: four 16-row tiles, the last one with 13 rows; N = 300: two row CTAs of 256 rows, the second with 44 rows.
# num_mc = 100 and 70: 64-sample tiles with 36 and 6 samples left over, 8-sample groups with 4 and 6.
@pytest.mark.parametrize("N,dim,q,p,mc", [(61, 8, 8, 0, 100), (61, 7, 5, 0, 70), (300, 7, 3, 3, 100),
                                          (300, 8, 4, 3, 70), (45, 8, 6, 1, 24)])
def test_acc_tile_gradient_matches_checker(capi, N, dim, q, p, mc):
    prob = make_problem(N, dim, seed=300 + N + dim + q, noise=0.05)
    gp, ref = _pair(capi, prob)
    rng = np.random.default_rng(N * 7 + dim * 31 + q)
    cands = rng.uniform(size=(2, q, dim))
    Xp = rng.uniform(size=(p, dim)) if p else None
    disc = rng.uniform(size=(6, dim))
    table = rng.standard_normal((mc // 2) * (q + p))
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, table=table, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], Xp, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(dim), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


def test_acc_tile_results_do_not_depend_on_batch(capi):
    """N = 300, d = 8, q + p = 7, 4100 samples: 9 candidates in one call, and in subsets of 1 and of 4, give
    bit-identical values and gradients."""
    prob = make_problem(300, 8, seed=77, noise=1e-2)
    gp, ref = _pair(capi, prob)
    rng = np.random.default_rng(12)
    cands = rng.uniform(size=(9, 6, 8))
    Xp = rng.uniform(size=(1, 8))
    disc = rng.uniform(size=(10, 8))
    best = float(ref.mean_additional(disc).min())
    mc = 4100
    kg, grad = gp.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xACC, grad=True)
    assert np.all(np.isfinite(kg)) and np.all(np.isfinite(grad))
    for size in (1, 4):
        for s in range(0, 9, size):
            k, g = gp.kg(cands[s:s + size], Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xACC,
                         grad=True)
            np.testing.assert_array_equal(k, kg[s:s + size])
            np.testing.assert_array_equal(g, grad[s:s + size])

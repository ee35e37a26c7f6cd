"""GPU parity: q-KG Monte-Carlo value and envelope-theorem gradient, CUDA path through the C ABI vs the CPU checker
(the compiled reference when available) on identical inputs and identical (table-fed) normals."""
import numpy as np
import pytest

import oracle as orc
from gpu_util import checker
from synth import DISCRETE_ONLY_GD, EXAMPLE_INNER_GD, make_problem, unit_bounds

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


# the reference's own ping-test shapes (gpp_knowledge_gradient_optimization_test.cpp:536-551): (q,p) in
# {(1,0),(2,0),(1,2),(3,2)}, num_mc_iter = 16, 5 discrete points, noise 0.1
@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("q,p", [(1, 0), (2, 0), (1, 2), (3, 2)])
def test_kg_discrete_only_table_fed(capi, kernel, q, p):
    """inner max_num_steps = 0: no data-dependent path, so parity is tight (SURVEY.md 8d(i): <= 1e-8 relative)."""
    prob = make_problem(16, 3, seed=9, noise=0.1)
    gp, ref = _pair(capi, kernel, prob)
    rng = np.random.default_rng(27)
    cands = rng.uniform(size=(3, q, 3))
    Xp = rng.uniform(size=(p, 3))
    disc = rng.uniform(size=(5, 3))
    mc = 16
    table = rng.standard_normal((mc // 2) * (q + p))
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, Xp, mc, best, DISCRETE_ONLY_GD, unit_bounds(3), disc, table=table, grad=True)
    for c in range(3):
        v, g = ref.kg(cands[c], Xp, mc, best, table, DISCRETE_ONLY_GD, unit_bounds(3), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-8, atol=1e-11)
        np.testing.assert_allclose(grad[c], g, rtol=1e-6, atol=1e-9)
    kv = gp.kg(cands, Xp, mc, best, DISCRETE_ONLY_GD, unit_bounds(3), disc, table=table)
    np.testing.assert_array_equal(kv, kg)


@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("gd", [EXAMPLE_INNER_GD, [1, 20, 3, 3, 0.7, 1.0, 0.2, 1e-7], [1, 8, 1, 3, 0.0, 4.0, 1.0, 1e-10]])
@pytest.mark.parametrize("q,p", [(1, 0), (2, 0), (3, 2)])
def test_kg_inner_line_search_table_fed(capi, kernel, gd, q, p):
    prob = make_problem(16, 3, seed=9, noise=0.1)
    gp, ref = _pair(capi, kernel, prob)
    rng = np.random.default_rng(31)
    cands = rng.uniform(size=(3, q, 3))
    Xp = rng.uniform(size=(p, 3))
    disc = rng.uniform(size=(5, 3))
    mc = 64
    table = rng.standard_normal((mc // 2) * (q + p))
    best = float(ref.mean_additional(disc).min())
    kg, grad, st = gp.kg(cands, Xp, mc, best, gd, unit_bounds(3), disc, table=table, grad=True, stats=True)
    assert st["mc_samples"] == 3 * mc and st["posterior_evals"] >= 3 * mc
    for c in range(3):
        v, g = ref.kg(cands[c], Xp, mc, best, table, gd, unit_bounds(3), disc, grad=True)
        # same normals, same algorithm: the only difference is floating-point re-association
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


def test_kg_fidelity_dimension(capi):
    prob = make_problem(14, 3, seed=21, noise=0.1)
    gp, ref = _pair(capi, 1, prob)
    rng = np.random.default_rng(8)
    cands = rng.uniform(size=(2, 2, 3))
    disc = rng.uniform(size=(6, 2))
    table = rng.standard_normal(8 * 2)
    kg, grad = gp.kg(cands, None, 16, 0.1, EXAMPLE_INNER_GD, unit_bounds(2), disc, num_fidelity=1, table=table, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], None, 16, 0.1, table, EXAMPLE_INNER_GD, unit_bounds(2), disc, num_fidelity=1, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


def test_kg_philox_stream_and_3sigma(capi):
    """Native Philox == host restatement fed to the checker (tight); another seed agrees within 3 sigma (north star)."""
    prob = make_problem(60, 6, seed=5, noise=1e-2)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(11)
    q, mc = 4, 256
    cands = rng.uniform(size=(4, q, 6))
    disc = rng.uniform(size=(10, 6))
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(6), disc, seed=0xC0FFEE, grad=True)
    table = orc.philox_normals(0xC0FFEE, 0, mc // 2, q)
    for c in range(2):
        v, g = ref.kg(cands[c], None, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(6), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(grad[c], g, rtol=1e-4, atol=1e-7)
    kg2 = gp.kg(cands, None, 4096, best, EXAMPLE_INNER_GD, unit_bounds(6), disc, seed=1)
    kg3 = gp.kg(cands, None, 4096, best, EXAMPLE_INNER_GD, unit_bounds(6), disc, seed=2)
    assert np.all(kg2 > 0)
    assert np.all(np.abs(kg2 - kg3) < 3.0 * np.sqrt(2.0) * (np.abs(kg2) + 0.5) / np.sqrt(4096))


def test_kg_north_star_shape_properties(capi):
    """Full-size shape (N=500, d=8, q=8): properties that do not need the CPU path at full size, plus a spot check of
    two candidates against the checker at reduced num_mc."""
    prob = make_problem(500, 8, seed=20260924 % 1000, noise=1e-2)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(7)
    cands = rng.uniform(size=(16, 8, 8))
    disc = rng.uniform(size=(10, 8))
    best = float(ref.mean_additional(disc).min())
    mc = 1024
    kg, grad, st = gp.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xC0FFEE, grad=True, stats=True)
    assert np.all(np.isfinite(kg)) and np.all(np.isfinite(grad)) and np.all(kg > -1e-9)
    # permutation equivariance over candidates and determinism (same seed -> bit-identical)
    perm = rng.permutation(16)
    kg_p, grad_p = gp.kg(cands[perm], None, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xC0FFEE, grad=True)
    np.testing.assert_array_equal(kg_p, kg[perm])
    np.testing.assert_array_equal(grad_p, grad[perm])
    table = orc.philox_normals(0xC0FFEE, 0, 32, 8)
    kg64, g64 = gp.kg(cands[:2], None, 64, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xC0FFEE, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], None, 64, best, table, EXAMPLE_INNER_GD, unit_bounds(8), disc, grad=True)
        np.testing.assert_allclose(kg64[c], v, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(g64[c], g, rtol=1e-4, atol=1e-7)


@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("gd", [DISCRETE_ONLY_GD, EXAMPLE_INNER_GD])
@pytest.mark.parametrize("q,p,g_idx", [(1, 0, (0,)), (2, 1, (0, 1)), (2, 0, (0, 1, 2))])
def test_dkg_derivative_observations_table_fed(capi, kernel, gd, q, p, g_idx):
    """d-KG: the GP holds derivative observations, candidates carry derivative rows (config 4's structure)."""
    prob = make_problem(12, 3, g_idx=g_idx, seed=9, noise=0.1)
    gp, ref = _pair(capi, kernel, prob)
    rng = np.random.default_rng(27)
    cands = rng.uniform(size=(3, q, 3))
    Xp = rng.uniform(size=(p, 3))
    disc = rng.uniform(size=(5, 3))
    mc = 32
    Q = (q + p) * (1 + len(g_idx))
    table = rng.standard_normal((mc // 2) * Q)
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, Xp, mc, best, gd, unit_bounds(3), disc, table=table, grad=True)
    for c in range(3):
        v, g = ref.kg(cands[c], Xp, mc, best, table, gd, unit_bounds(3), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("dim,g_idx,q", [(8, tuple(range(8)), 2), (4, (1, 3), 3), (6, (0, 2, 3, 4, 5), 1)])
def test_dkg_weight_column_paths(capi, kernel, dim, g_idx, q):
    """The per-sample weight columns of the d-KG kernel on shapes the other tests do not reach: 8 derivative observations
    (9 rows per point: one point per ring stage), even / odd row counts, and 1024 samples per candidate so that lanes
    take several samples each — cohorts of lanes (own-lane column fill) as well as stragglers (warp-cooperative fill)."""
    prob = make_problem(10, dim, g_idx=g_idx, seed=21 + dim, noise=0.1)
    gp, ref = _pair(capi, kernel, prob)
    rng = np.random.default_rng(5 + dim)
    cands = rng.uniform(size=(2, q, dim))
    disc = rng.uniform(size=(6, dim))
    mc = 1024
    Q = q * (1 + len(g_idx))
    table = rng.standard_normal((mc // 2) * Q)
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, table=table, grad=True)
    v, g = ref.kg(cands[1], None, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(dim), disc, grad=True)
    np.testing.assert_allclose(kg[1], v, rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(grad[1], g, rtol=1e-5, atol=1e-8)


def test_dkg_config4_shape_spot_check(capi):
    """BASELINE.json configs[3] structure: d = 4, all 4 partial derivatives observed, q = 4 (system n = N*5); reduced N
    and num_mc so that the CPU checker finishes in seconds, Philox stream on the device."""
    prob = make_problem(40, 4, g_idx=(0, 1, 2, 3), seed=4, noise=1e-2)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(3)
    q, mc = 4, 64
    cands = rng.uniform(size=(4, q, 4))
    disc = rng.uniform(size=(10, 4))
    best = float(ref.mean_additional(disc).min())
    kg, grad, st = gp.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(4), disc, seed=0xC0FFEE, grad=True, stats=True)
    assert st["posterior_evals"] >= 4 * mc
    table = orc.philox_normals(0xC0FFEE, 0, mc // 2, q * 5)
    for c in range(2):
        v, g = ref.kg(cands[c], None, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(4), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(grad[c], g, rtol=1e-4, atol=1e-7)


def test_dkg_config4_full_size(capi):
    """BASELINE.json configs[3] at FULL training size: d = 4, N = 300 with all 4 partial derivatives observed (system
    n = 1500), q = 4 (20 union rows -> the 24-row instantiation); two candidates, 64 samples, same normals as the
    reference (table replay)."""
    prob = make_problem(300, 4, g_idx=(0, 1, 2, 3), seed=44, noise=1e-2)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(5)
    q, mc = 4, 64
    cands = rng.uniform(size=(2, q, 4))
    disc = rng.uniform(size=(10, 4))
    best = float(ref.mean_additional(disc).min())
    table = orc.philox_normals(0xC0FFEE, 0, mc // 2, q * 5)
    kg, grad = gp.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(4), disc, seed=0xC0FFEE, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], None, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(4), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(grad[c], g, rtol=1e-4, atol=1e-7)


@pytest.mark.parametrize("case", ["second_batch", "out_of_range_factors", "exhausted_search", "tiny_length_scale"])
def test_kg_line_batch_edge_paths(capi, case):
    """The SquareExponential fast path evaluates all backtracking trials of a step in one pass (8 step sizes per batch).
    Edge paths: more than 8 halvings (second batch), exponent factors that would leave the double range (falls back to
    one evaluation per trial), and 30 halvings without acceptance (the reference stops the run)."""
    if case == "second_batch":
        prob = make_problem(16, 3, seed=9, noise=0.1)
        gd = [1, 5, 2, 3, 0.0, 32.0, 0.5, 1e-10]          # a_0 = 32: 8-9 halvings before the Armijo test holds
    elif case == "out_of_range_factors":
        prob = make_problem(16, 3, seed=9, noise=0.1)
        gd = [1, 5, 2, 3, 0.0, 4096.0, 0.5, 1e-10]        # a_0 |p_j| >> 650: exp(a_0 p_j) is not representable
    elif case == "tiny_length_scale":
        # scaled coordinates up to ~8e3 length scales: outside the shared-memory fast path's range contract
        # (kFastPathRadius), so the host must route the step through the fully guarded kernel
        prob = make_problem(16, 3, seed=9, noise=0.1, length=2e-4)
        gd = [1, 4, 2, 3, 0.0, 1e-6, 0.5, 1e-10]
    else:
        prob = make_problem(16, 3, seed=9, noise=0.1)
        gd = [1, 3, 2, 3, 0.0, 1e12, 0.5, 1e-10]          # a_0 2^-29 is still far too large: search hits 30
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(41)
    q, mc = 2, 32
    cands = rng.uniform(size=(2, q, 3))
    disc = rng.uniform(size=(5, 3))
    table = rng.standard_normal((mc // 2) * q)
    best = float(ref.mean_additional(disc).min())
    kg, grad, st = gp.kg(cands, None, mc, best, gd, unit_bounds(3), disc, table=table, grad=True, stats=True)
    print(case, st)
    if case == "second_batch":
        assert st["line_batches"] >= 1.5 * st["line_search_steps"]  # two batches for most steps ...
        assert st["point_evals"] < st["posterior_evals"] / 3  # ... and few one-at-a-time trials
    if case == "out_of_range_factors":
        assert st["point_evals"] > 5 * st["line_search_steps"]  # the trials were evaluated one at a time
    for c in range(2):
        v, g, bp = ref.kg(cands[c], None, mc, best, table, gd, unit_bounds(3), disc, grad=True, want_best_points=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)

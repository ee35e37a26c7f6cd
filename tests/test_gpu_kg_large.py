"""GPU tests of cmoe_kg_eval_large (q-KG past 32 union rows, DESIGN.md K17), every case through the C ABI: agreement
with cmoe_kg_eval where both apply, the CPU checker past 32 rows on identical table-fed normals, Philox against table
mode, batch and chunk invariance, the edges of the size contract, the multistart driver past 32 rows and the GPP
module's routing."""
import os
import sys

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


def _gp(capi, kernel, prob):
    return capi.GaussianProcess(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                                prob["derivs"])


def _ref(kernel, prob):
    ref, lm = checker().gp(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    return ref


# (id, kernel, dim, g_idx, q, p, N): Q = (q + p)(1 + g) <= 32, both calls apply
SMALL_CASES = [
    ("se-g0", 0, 3, (), 3, 2, 16),
    ("matern-g0", 1, 3, (), 2, 3, 16),
    ("se-g2", 0, 3, (0, 2), 2, 1, 12),
    ("matern-g2", 1, 3, (1, 2), 1, 2, 12),
    ("se-g10-wide", 0, 10, tuple(range(10)), 2, 0, 9),
]


@pytest.mark.parametrize("gd", ["discrete", "inner"])
@pytest.mark.parametrize("case", SMALL_CASES, ids=[c[0] for c in SMALL_CASES])
def test_agrees_with_kg_eval_up_to_32_rows(capi, case, gd):
    _, kernel, dim, g_idx, q, p, N = case
    prob = make_problem(N, dim, g_idx=g_idx, seed=13, noise=0.1)
    gp = _gp(capi, kernel, prob)
    rng = np.random.default_rng(5)
    cands = rng.uniform(size=(3, q, dim))
    Xp = rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(6, dim))
    inner = DISCRETE_ONLY_GD if gd == "discrete" else EXAMPLE_INNER_GD
    args = (cands, Xp, 64, 0.2, inner, unit_bounds(dim), disc)
    v0, g0, s0 = gp.kg(*args, seed=77, grad=True, stats=True)
    v1, g1, s1 = gp.kg_large(*args, seed=77, grad=True, stats=True)
    assert s1["mc_samples"] == s0["mc_samples"] == 3 * 64
    if gd == "discrete":
        np.testing.assert_allclose(v1, v0, rtol=1e-11, atol=1e-14)
        for c in range(3):
            assert np.max(np.abs(g1[c] - g0[c])) <= 1e-9 * np.max(np.abs(g0[c])) + 1e-14, (g1[c], g0[c])
        assert s1["posterior_evals"] == s0["posterior_evals"]
        assert s1["line_search_steps"] == s0["line_search_steps"] == 0
    else:
        np.testing.assert_allclose(v1, v0, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(g1, g0, rtol=1e-5, atol=1e-8)
        assert abs(int(s1["posterior_evals"]) - int(s0["posterior_evals"])) <= 0.01 * s0["posterior_evals"]
        assert abs(int(s1["line_search_steps"]) - int(s0["line_search_steps"])) <= 0.01 * s0["line_search_steps"] + 1


# (id, kernel, dim, g_idx, q, p, N, num_fidelity): Q > 32, cmoe_kg_eval refuses every one of them
LARGE_CASES = [
    ("se-q8p25", 0, 3, (), 8, 25, 20, 0),
    ("matern-q8p25", 1, 3, (), 8, 25, 20, 0),
    ("se-q40", 0, 3, (), 40, 0, 20, 0),
    ("matern-q40", 1, 3, (), 40, 0, 20, 0),
    ("se-q4p60", 0, 3, (), 4, 60, 20, 0),
    ("matern-q4p60", 1, 3, (), 4, 60, 20, 0),
    ("dkg-g2-u12", 0, 3, (0, 1), 3, 9, 12, 0),
    ("dkg-d8-g8-u4", 0, 8, tuple(range(8)), 2, 2, 10, 0),
    ("wide-d10-g10-q3", 0, 10, tuple(range(10)), 3, 0, 9, 0),
    ("se-q34-nf1", 0, 3, (), 30, 4, 16, 1),
]


@pytest.mark.parametrize("gd", ["discrete", "inner"])
@pytest.mark.parametrize("case", LARGE_CASES, ids=[c[0] for c in LARGE_CASES])
def test_matches_checker_past_32_rows(capi, case, gd):
    _, kernel, dim, g_idx, q, p, N, nf = case
    prob = make_problem(N, dim, g_idx=g_idx, seed=29, noise=0.1)
    gp, ref = _gp(capi, kernel, prob), _ref(kernel, prob)
    Q = (q + p) * (1 + len(g_idx))
    assert Q > 32
    with pytest.raises(capi.BoundsError):
        gp.kg(np.full((1, q, dim), 0.5), np.full((p, dim), 0.25), 16, 0.0, DISCRETE_ONLY_GD, unit_bounds(dim - nf),
              np.full((2, dim - nf), 0.5), num_fidelity=nf)
    rng = np.random.default_rng(17)
    cands = rng.uniform(size=(2, q, dim))
    Xp = rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(5, dim - nf))
    mc = 16 if gd == "discrete" else 32
    inner = DISCRETE_ONLY_GD if gd == "discrete" else EXAMPLE_INNER_GD
    table = rng.standard_normal((mc // 2) * Q)
    best = 0.1
    kg, grad = gp.kg_large(cands, Xp, mc, best, inner, unit_bounds(dim - nf), disc, num_fidelity=nf, table=table,
                           grad=True)
    rv, rg = (1e-8, 1e-6) if gd == "discrete" else (1e-7, 1e-5)
    for c in range(2):
        v, g = ref.kg(cands[c], Xp, mc, best, table, inner, unit_bounds(dim - nf), disc, num_fidelity=nf, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=rv, atol=1e-11)
        np.testing.assert_allclose(grad[c], g, rtol=rg, atol=1e-8)


def test_philox_equals_table_mode(capi):
    prob = make_problem(20, 3, seed=3, noise=0.1)
    gp = _gp(capi, 0, prob)
    rng = np.random.default_rng(2)
    q, p, mc = 10, 30, 64
    cands = rng.uniform(size=(2, q, 3))
    Xp = rng.uniform(size=(p, 3))
    disc = rng.uniform(size=(4, 3))
    args = (cands, Xp, mc, 0.1, EXAMPLE_INNER_GD, unit_bounds(3), disc)
    v0, g0 = gp.kg_large(*args, seed=0xBEEF, grad=True)
    table = capi.philox_normals(0xBEEF, 0, mc // 2, q + p)
    v1, g1 = gp.kg_large(*args, table=table, grad=True)
    np.testing.assert_array_equal(v1, v0)
    np.testing.assert_array_equal(g1, g0)


def test_batch_and_chunk_invariance(capi):
    """65536 samples per candidate make one candidate's workspace about 170 MB, so 14 candidates run in two 2 GiB
    chunks; candidates 0 and 13 are bit-identical alone and inside that batch."""
    prob = make_problem(50, 3, seed=4, noise=0.05)
    gp = _gp(capi, 0, prob)
    rng = np.random.default_rng(9)
    q, p, mc = 20, 20, 65536
    cands = rng.uniform(size=(14, q, 3))
    Xp = rng.uniform(size=(p, 3))
    disc = rng.uniform(size=(10, 3))
    args = (mc, 0.1, EXAMPLE_INNER_GD, unit_bounds(3), disc)
    v, g = gp.kg_large(cands, Xp, *args, seed=5, grad=True)
    assert np.all(np.isfinite(v)) and np.all(np.isfinite(g))
    for c in (0, 13):
        v1, g1 = gp.kg_large(cands[c:c + 1], Xp, *args, seed=5, grad=True)
        np.testing.assert_array_equal(v1[0], v[c])
        np.testing.assert_array_equal(g1[0], g[c])


def test_size_edges(capi):
    prob = make_problem(8, 2, seed=1, noise=0.1)
    gp = _gp(capi, 0, prob)
    rng = np.random.default_rng(0)
    cands = rng.uniform(size=(1, 24, 2))
    Xp = rng.uniform(size=(1000, 2))
    disc = rng.uniform(size=(3, 2))
    v = gp.kg_large(cands, Xp, 8, 0.1, DISCRETE_ONLY_GD, unit_bounds(2), disc, seed=1)
    assert np.all(np.isfinite(v))
    with pytest.raises(capi.BoundsError):
        gp.kg_large(cands, np.vstack([Xp, Xp[:1]]), 8, 0.1, DISCRETE_ONLY_GD, unit_bounds(2), disc, seed=1)
    # exactly 1025 rows as U (1 + g): 205 points with four derivative observations each
    dprob = make_problem(8, 4, g_idx=(0, 1, 2, 3), seed=1, noise=0.1)
    dgp = _gp(capi, 0, dprob)
    with pytest.raises(capi.BoundsError):
        dgp.kg_large(rng.uniform(size=(1, 5, 4)), rng.uniform(size=(200, 4)), 8, 0.1, DISCRETE_ONLY_GD,
                     unit_bounds(4), rng.uniform(size=(3, 4)), seed=1)
    # cmoe_kg_eval and cmoe_kg_eval_large refuse the same bad inner arguments with the same message
    small, long_gd, empty = rng.uniform(size=(1, 2, 2)), list(DISCRETE_ONLY_GD), unit_bounds(2).copy()
    long_gd[1] = 4097
    empty[0] = 2.0
    for gd, ib in [(long_gd, unit_bounds(2)), (DISCRETE_ONLY_GD, empty)]:
        msgs = []
        for call in (gp.kg, gp.kg_large):
            with pytest.raises(capi.BoundsError) as e:
                call(small, None, 8, 0.1, gd, ib, disc, seed=1)
            msgs.append(str(e.value))
        assert msgs[0] == msgs[1], msgs


def test_singular_union_reports_the_leading_minor(capi):
    prob = make_problem(12, 2, seed=8, noise=0.0)
    gp = _gp(capi, 0, prob)
    rng = np.random.default_rng(4)
    cands = rng.uniform(size=(2, 2, 2))
    cands[1, 1] = prob["X"][3]  # duplicates a training point with zero noise
    disc = rng.uniform(size=(3, 2))
    args = (cands, rng.uniform(size=(1, 2)), 8, 0.1, DISCRETE_ONLY_GD, unit_bounds(2), disc)
    with pytest.raises(capi.SingularMatrixError) as small:
        gp.kg(*args, seed=1)
    with pytest.raises(capi.SingularMatrixError) as large:
        gp.kg_large(*args, seed=1)
    assert large.value.info > 0
    assert large.value.info == small.value.info


def _ms_problem(capi):
    prob = make_problem(20, 3, seed=41, noise=0.05)
    gp = _gp(capi, 0, prob)
    rng = np.random.default_rng(42)
    q, p = 2, 32  # Q = 34
    starts = rng.uniform(0.1, 0.9, size=(8, q, 3))
    Xp = rng.uniform(size=(p, 3))
    disc = rng.uniform(size=(5, 3))
    return prob, gp, starts, Xp, disc


def test_multistart_kg_past_32_rows_matches_reference_driver(capi):
    """cmoe_multistart_kg at q + p = 34 against the reference's unmodified driver on identical normals, one descent step
    per start so that the comparison is exact: the screening values (the reference state keeps the first start's points
    in its discretisation set), the found flag and the best point."""
    if not orc.have_reference():
        pytest.skip("needs the compiled reference driver (oracle/_ref)")
    prob, gp, starts, Xp, disc = _ms_problem(capi)
    ref = _ref(0, prob)
    q, p = starts.shape[1], Xp.shape[0]
    mc, seed = 32, 4243
    best = float(ref.mean_additional(disc).min())
    b3 = unit_bounds(3)
    outer = [8, 1, 1, 0, 0.7, 0.4, 0.2, 1e-7]
    table = orc.normal_draws(seed, (mc // 2) * (q + p))
    bp, bv, found, sv = capi.multistart_kg(gp, starts, Xp, mc, best, outer, EXAMPLE_INNER_GD, b3, b3, disc, seed=1,
                                           table=table)
    for i in (0, 3, 7):
        v = ref.kg_reused_state(starts[0], starts[i], Xp, mc, best, table, EXAMPLE_INNER_GD, b3, disc)
        np.testing.assert_allclose(sv[i], v, rtol=1e-7, atol=1e-10)
    rbp, rfound = orc.ref_multistart_kg(ref, starts, Xp, mc, best, outer, EXAMPLE_INNER_GD, b3, b3, disc, seed)
    assert found == rfound
    np.testing.assert_allclose(bp, rbp, rtol=0, atol=1e-9)


def test_multistart_kg_past_32_rows_multi_device_is_bit_identical(capi):
    if capi.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    _, gp, starts, Xp, disc = _ms_problem(capi)
    b3 = unit_bounds(3)
    outer = [8, 3, 1, 0, 0.7, 0.4, 0.2, 1e-7]
    one = capi.multistart_kg(gp, starts, Xp, 64, 0.0, outer, EXAMPLE_INNER_GD, b3, b3, disc, seed=5)
    devs = list(range(min(4, capi.device_count())))
    many = capi.multistart_kg(gp, starts, Xp, 64, 0.0, outer, EXAMPLE_INNER_GD, b3, b3, disc, seed=5, devices=devs)
    np.testing.assert_array_equal(one[3], many[3])
    np.testing.assert_array_equal(one[0], many[0])
    assert one[1] == many[1] and one[2] == many[2]


def test_gpp_routes_past_32_rows_only(capi):
    """GPP.compute_knowledge_gradient / compute_grad_knowledge_gradient: at q + p = 40 the large call on the same seed,
    at q + p <= 32 still the 32-row call, bit for bit."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cornell-moe_b200"))
    import GPP as C_GP
    prob = make_problem(20, 3, seed=43, noise=0.05)
    gp = _gp(capi, 1, prob)  # the Python boundary's kernel is Matern-5/2
    gpp = C_GP.GaussianProcess([prob["alpha"], list(prob["lengths"])], list(prob["X"].ravel()), list(prob["y"]),
                               list(prob["noise"]), [], 0, 3, prob["N"])

    class Params:
        domain_type = C_GP.DomainTypes.tensor_product
        optimizer_type = C_GP.OptimizerTypes.gradient_descent
        num_random_samples = 8
        optimizer_parameters = C_GP.GradientDescentParameters(*EXAMPLE_INNER_GD)

    rng = np.random.default_rng(44)
    disc = rng.uniform(size=(5, 3))
    mc, best, b3 = 64, 0.1, unit_bounds(3)
    for q, p, large in ((4, 36, True), (4, 28, False)):
        Xq, Xp = rng.uniform(size=(q, 3)), rng.uniform(size=(p, 3))
        rnd = C_GP.RandomnessSourceContainer(1)
        rnd.SetExplicitNormalRNGSeed(123)
        args = (gpp, 0, Params, list(b3), list(disc.ravel()), list(Xq.ravel()), list(Xp.ravel()), 5, q, p, mc, best, rnd)
        kg = C_GP.compute_knowledge_gradient(*args)
        gkg = np.array(C_GP.compute_grad_knowledge_gradient(*args)).reshape(q, 3)
        call = gp.kg_large if large else gp.kg
        v, g = call(Xq[None], Xp, mc, best, EXAMPLE_INNER_GD, b3, disc, seed=123, grad=True)
        assert kg == v[0]
        np.testing.assert_array_equal(gkg, g[0])
        if not large:
            with pytest.raises(capi.BoundsError):
                gp.kg(Xq[None], np.vstack([Xp, Xp[:5]]), mc, best, EXAMPLE_INNER_GD, b3, disc, seed=123)

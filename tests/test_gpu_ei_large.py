"""Posterior covariance and q-EI past the 96-row bound of the per-set kernels (DESIGN.md K16): cmoe_gp_posterior_large
and cmoe_ei_eval_large against the CPU checker (which has no size limit), against cmoe_ei_eval below the bound, against
finite differences, and through the multistart driver and the GPP front end."""
import os
import sys

import numpy as np
import pytest

import oracle as orc
from gpu_util import checker
from synth import make_problem, unit_bounds

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


# (Q, GP derivative rows, set derivative rows)
POSTERIOR_CASES = [(97, (), ()), (130, (0,), (1,)), (257, (1,), ()), (1000, (), (0, 1, 2))]


@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("case", range(len(POSTERIOR_CASES)))
def test_posterior_large_matches_checker(capi, kernel, case):
    Q, g_idx, ds = POSTERIOR_CASES[case]
    num = Q // (1 + len(ds))
    assert num * (1 + len(ds)) == Q
    prob = make_problem(40, 3, g_idx=g_idx, seed=5 + case, noise=1e-2, length=0.15)
    gp, ref = _pair(capi, kernel, prob)
    sets = np.random.default_rng(case).uniform(size=(2, num, 3))
    out = gp.posterior_large(sets, ds, ("mean", "var", "chol_var"))
    for s in range(2):
        r = ref.posterior(sets[s], ds, ("mean", "var", "chol_var"))
        assert r["rc"] == 0
        np.testing.assert_allclose(out["mean"][s], r["mean"], rtol=1e-9, atol=1e-10)
        V = out["var"][s].reshape(Q, Q).T
        np.testing.assert_allclose(np.tril(V), np.tril(r["var"].reshape(Q, Q).T), rtol=1e-8, atol=1e-10)
        np.testing.assert_array_equal(V, V.T)
        L = out["chol_var"][s].reshape(Q, Q).T
        assert np.all(np.triu(L, 1) == 0.0) and np.all(np.diag(L) > 0.0)
        Vr = r["var"].reshape(Q, Q).T
        # backward error of the factor, whatever the conditioning; elementwise against the checker where Var is
        # well conditioned (the sets with three derivative rows per point are not: factors differ by rounding there)
        assert np.abs(L @ L.T - Vr).max() <= 1e-10 * np.abs(Vr).max()
        if np.linalg.cond(Vr) < 1e6:
            np.testing.assert_allclose(np.tril(L), np.tril(r["chol_var"].reshape(Q, Q).T), rtol=1e-7, atol=1e-9)


def test_posterior_large_singular(capi):
    prob = make_problem(20, 2, seed=2)
    gp, _ = _pair(capi, 0, prob)
    pts = np.random.default_rng(4).uniform(size=(120, 2))
    pts[60] = pts[10]
    with pytest.raises(capi.SingularMatrixError) as e:
        gp.posterior_large(pts[None], (), ("chol_var",))
    assert e.value.info == 61


# (kernel, GP derivative rows, q, p)
EI_CASES = [(0, (), 97, 0), (1, (), 100, 28), (0, (1,), 60, 140), (1, (), 8, 512)]


@pytest.mark.parametrize("case", range(len(EI_CASES)))
def test_ei_large_table_matches_checker(capi, case):
    kernel, g_idx, q, p = EI_CASES[case]
    prob = make_problem(30, 3, g_idx=g_idx, seed=11 + case, noise=1e-2, length=0.3)
    gp, ref = _pair(capi, kernel, prob)
    rng = np.random.default_rng(100 + case)
    cands = rng.uniform(size=(2, q, 3))
    Xp = rng.uniform(size=(p, 3))
    mc = 64
    table = rng.standard_normal(mc * (q + p))
    best = float(prob["y"][:: 1 + len(g_idx)].min()) + 0.3
    ei, grad = gp.ei_large(cands, Xp, mc, best, table=table, grad=True)
    for c in range(2):
        v, g = ref.ei(cands[c], Xp, mc, best, table, grad=True)
        assert abs(ei[c] - v) <= 1e-10 * max(1.0, abs(v)), (ei[c], v)
        np.testing.assert_allclose(grad[c], g, rtol=1e-7, atol=1e-9 * max(1.0, np.abs(g).max()))


@pytest.mark.parametrize("q,p", [(1, 0), (2, 0), (30, 7), (90, 6)])
def test_ei_large_agrees_with_ei_eval(capi, q, p):
    prob = make_problem(30, 3, seed=3, length=0.3)
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"])
    rng = np.random.default_rng(q + p)
    cands = rng.uniform(size=(3, q, 3))
    Xp = rng.uniform(size=(p, 3))
    best = float(prob["y"].min()) + 0.3
    v0, g0 = gp.ei(cands, Xp, 500, best, seed=77, grad=True)
    v1, g1 = gp.ei_large(cands, Xp, 500, best, seed=77, grad=True)
    np.testing.assert_allclose(v1, v0, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(g1, g0, rtol=1e-9, atol=1e-12 * np.abs(g0).max())


def test_ei_large_gradient_finite_differences(capi):
    prob = make_problem(30, 3, seed=21, length=0.3)
    gp = capi.GaussianProcess(1, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"])
    rng = np.random.default_rng(5)
    q, p, mc = 110, 10, 128
    cand = rng.uniform(size=(1, q, 3))
    Xp = rng.uniform(size=(p, 3))
    table = rng.standard_normal(mc * (q + p))
    best = float(prob["y"].min()) + 0.3
    _, g = gp.ei_large(cand, Xp, mc, best, table=table, grad=True)
    h = 1e-6
    for (i, d) in [(0, 0), (17, 1), (63, 2), (109, 0)]:
        plus, minus = cand.copy(), cand.copy()
        plus[0, i, d] += h
        minus[0, i, d] -= h
        fd = (gp.ei_large(plus, Xp, mc, best, table=table)[0] - gp.ei_large(minus, Xp, mc, best, table=table)[0]) / (2 * h)
        assert abs(fd - g[0, i, d]) <= 1e-5 * max(1e-3, abs(g[0, i, d])), (i, d, fd, g[0, i, d])


def test_ei_large_monte_carlo_error(capi):
    prob = make_problem(30, 3, seed=8, length=0.3)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(6)
    q, mc, big = 100, 4000, 40000
    cand = rng.uniform(size=(1, q, 3))
    best = float(prob["y"].min()) + 0.3
    v = gp.ei_large(cand, None, mc, best, seed=12345)[0]
    table = rng.standard_normal((big, q))
    vr = ref.ei(cand[0], None, big, best, table)
    # the spread of one sample's improvement, from the same draws in numpy (Var + 1e-6 I, as the estimator factors it)
    post = gp.posterior_large(cand, (), ("mean", "var"))
    C = np.linalg.cholesky(post["var"][0].reshape(q, q).T + 1e-6 * np.eye(q))
    imp = np.maximum(0.0, (best - (post["mean"][0][None, :] + table @ C.T)).max(axis=1))
    assert abs(imp.mean() - vr) <= 1e-9 * max(1.0, vr)
    sd = imp.std()
    assert abs(v - vr) <= 3.0 * sd * np.sqrt(1.0 / mc + 1.0 / big), (v, vr, sd)


def test_ei_large_batch_invariance_across_chunks(capi):
    prob = make_problem(30, 3, seed=9, length=0.3)
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"])
    rng = np.random.default_rng(7)
    q, p, mc = 100, 2900, 64  # about 216 MB of device scratch per candidate with the gradient: 9 per 2 GiB chunk
    cands = rng.uniform(size=(10, q, 3))
    Xp = rng.uniform(size=(p, 3))
    best = float(prob["y"].min()) + 0.3
    vb, gb = gp.ei_large(cands, Xp, mc, best, seed=3, grad=True)
    for c in (0, 9):
        v1, g1 = gp.ei_large(cands[c:c + 1], Xp, mc, best, seed=3, grad=True)
        assert v1[0] == vb[c]
        np.testing.assert_array_equal(g1[0], gb[c])


def test_ei_large_size_edges(capi):
    prob = make_problem(20, 2, seed=1, length=0.3)
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"])
    rng = np.random.default_rng(8)
    v = gp.ei_large(rng.uniform(size=(1, 8192, 2)), None, 32, 0.5, seed=1)
    assert np.isfinite(v[0]) and v[0] >= 0.0
    with pytest.raises(capi.BoundsError):
        gp.ei_large(rng.uniform(size=(1, 8000, 2)), rng.uniform(size=(193, 2)), 32, 0.5, seed=1)
    with pytest.raises(capi.BoundsError):
        gp.posterior_large(rng.uniform(size=(1, 4097, 2)), (0,), ("var",))


def test_multistart_ei_q100_matches_reference_driver(capi):
    if not orc.have_reference():
        pytest.skip("needs the compiled reference (oracle/_ref)")
    prob = make_problem(15, 2, seed=8, noise=0.05, length=0.4)
    gp, ref = _pair(capi, 0, prob)
    q, mc, seed = 100, 32, 99
    starts = np.random.default_rng(9).uniform(0.05, 0.95, size=(3, q, 2))
    best = float(prob["y"].min()) + 0.2
    outer = [3, 2, 1, 0, 0.7, 0.5, 0.2, 1e-7]
    table = orc.normal_draws(seed, mc * q)
    bp, bv, found, sv = capi.multistart_ei(gp, starts, None, mc, best, outer, unit_bounds(2), seed=1, table=table)
    for i in range(3):
        assert abs(sv[i] - ref.ei(starts[i], None, mc, best, table)) <= 1e-10
    ref_bp = orc.ref_multistart_ei(ref, starts, None, mc, best, outer, unit_bounds(2), seed)
    assert found
    np.testing.assert_allclose(bp, ref_bp, rtol=0, atol=1e-8)


def test_gpp_routes_past_96_rows(capi):
    sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
    import GPP as C_GP
    prob = make_problem(20, 3, g_idx=(0, 1), seed=4, length=0.3)
    gpp = C_GP.GaussianProcess([1.0, list(prob["lengths"])], list(prob["X"].ravel()), list(prob["y"]),
                               list(prob["noise"]), [0, 1], 2, 3, 20)
    ref, _ = checker().gp(1, 1.0, prob["lengths"], prob["X"], prob["y"], prob["noise"], (0, 1))  # Matern-5/2
    pts = np.random.default_rng(3).uniform(size=(40, 3))
    L = np.array(gpp.compute_cholesky_variance_of_points(list(pts.ravel()), 40)).reshape(120, 120)
    r = ref.posterior(pts, (0, 1), ("chol_var",))
    np.testing.assert_allclose(np.tril(L), np.tril(r["chol_var"].reshape(120, 120).T), rtol=1e-7, atol=1e-9)
    with pytest.raises(Exception) as e:
        gpp.compute_grad_variance_of_points(list(pts.ravel()), 40, 1)
    assert "96" in str(e.value)
    gp = capi.GaussianProcess(1, 1.0, prob["lengths"], prob["X"], prob["y"], prob["noise"], (0, 1))
    rnd = C_GP.RandomnessSourceContainer(4)
    rnd.SetExplicitNormalRNGSeed(123)
    Xq = np.random.default_rng(5).uniform(size=(100, 3))
    best = float(prob["y"][::3].min()) + 0.2
    ei = C_GP.compute_expected_improvement(gpp, list(Xq.ravel()), [], 100, 0, 64, best, False, rnd)
    assert ei == gp.ei_large(Xq, None, 64, best, seed=123)[0]

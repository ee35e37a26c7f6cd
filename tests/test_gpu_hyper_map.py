"""GPU tests of the hyper-parameter MAP fit (cmoe_hyperparameter_map, DESIGN.md K19) and of the exact hyper-parameter
gradient (cmoe_grad_log_marginal_likelihood_list_exact): the gradient against central differences of the checker's
likelihood, the objective against the NumPy restatement (tests/hyper_map_ref.py), end points against the reference's
own optimize() call (scipy BFGS with finite differences), batch invariance, the status paths, the size edges and the
GPP entry."""
import os
import sys

import numpy as np
import pytest
from scipy import optimize

import hyper_map_ref as M
import hyper_mcmc_ref as R
from gpu_util import checker
from synth import make_problem

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))  # the GPP module

HUGE_GTOL = 1e300  # stops every start at its first evaluation: the objective and gradient at the start


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def checker_lml(kernel, prob):
    dim = prob["dim"]
    return lambda h: checker().log_marginal_likelihood(kernel, h[0], h[1:1 + dim], prob["X"], prob["y"], h[1 + dim:],
                                                       prob["derivs"])


# ---- 1. the exact gradient ------------------------------------------------------------------------------------------
EXACT = [(k, g) for k in (0, 1) for g in ((), (1,), (0, 1, 2))]


@pytest.mark.parametrize("kernel,g_idx", EXACT, ids=[f"k{k}-g{len(g)}" for k, g in EXACT])
def test_exact_gradient_matches_central_differences(capi, kernel, g_idx):
    prob = make_problem(12, 3, g_idx=g_idx, seed=31 + len(g_idx))
    dim, g = 3, len(g_idx)
    rng = np.random.default_rng(5)
    H = np.concatenate([[1.2], rng.uniform(0.4, 0.9, dim), rng.uniform(0.01, 0.05, 1 + g)])
    # two sets: the second shares the first's points, so coincident pairs are on every diagonal
    v, gr = capi.grad_log_marginal_likelihood_list_exact(kernel, np.stack([H, 1.1 * H]), prob["X"], prob["y"],
                                                         prob["derivs"])
    lml = checker_lml(kernel, prob)
    for s, h in enumerate([H, 1.1 * H]):
        fd = np.empty(len(h))
        for k in range(len(h)):  # fourth-order central differences with a relative step
            e = np.zeros(len(h))
            e[k] = 1e-3 * h[k]
            fd[k] = (-lml(h + 2 * e) + 8 * lml(h + e) - 8 * lml(h - e) + lml(h - 2 * e)) / (12 * e[k])
        assert np.max(np.abs(gr[s] - fd)) <= 1e-6 * np.max(np.abs(fd)), (s, gr[s], fd)
        assert v[s] == pytest.approx(lml(h), rel=1e-10)
    vq, gq = capi.grad_log_marginal_likelihood_list(kernel, np.stack([H, 1.1 * H]), prob["X"], prob["y"],
                                                    prob["derivs"])
    assert np.array_equal(v, vq)
    if g == 0 or kernel == 0:  # no quirk to differ from: the same bits
        assert np.array_equal(gr, gq)


# ---- 2. the objective at given theta --------------------------------------------------------------------------------
def restated(capi, kernel, prob, theta, noisy, prior):
    dim, g = prob["dim"], len(prob["derivs"])
    lml = lambda h: capi.log_marginal_likelihood_list(kernel, h[None], prob["X"], prob["y"], prob["derivs"])[0]  # noqa
    lml_g = lambda h: capi.grad_log_marginal_likelihood_list_exact(kernel, h[None], prob["X"], prob["y"],  # noqa
                                                                   prob["derivs"])[1][0]
    f = M.nll(theta, lml, dim, g, noisy, prior)
    return f, (M.nll_grad(theta, lml_g, dim, g, noisy, prior) if np.isfinite(f) else None)


OBJ = [(1, (), True, True), (1, (), False, True), (0, (), True, False), (1, (0, 2), False, False),
       (1, (0, 2), True, True), (0, (1,), False, True)]


@pytest.mark.parametrize("kernel,g_idx,noisy,prior", OBJ,
                         ids=[f"k{k}-g{len(g)}-{'noisy' if z else 'pinned'}-{'prior' if p else 'none'}"
                              for k, g, z, p in OBJ])
def test_objective_and_gradient_match_restatement(capi, kernel, g_idx, noisy, prior):
    prob = make_problem(20, 3, g_idx=g_idx, seed=7)
    dim, g = 3, len(g_idx)
    rng = np.random.default_rng(11)
    T = R.initial_walkers(rng, 6, dim, g)
    T[1, 0] = 20.5  # the box
    T[2, 2] = 3.5  # the tophat wall (only with the prior)
    r = capi.hyperparameter_map(kernel, T, prob["X"], prob["y"], prob["derivs"], noisy=noisy, default_prior=prior,
                                gtol=HUGE_GTOL)
    assert np.array_equal(r["positions"], T)  # the pinning acts on a copy
    assert np.all(r["evaluations"] == 1) and np.all(r["iterations"] == 0)
    for s in range(len(T)):
        f, gr = restated(capi, kernel, prob, T[s], noisy, prior)
        if not np.isfinite(f):
            assert r["values"][s] == np.inf and r["status"][s] == 2
            continue
        assert r["status"][s] == 0
        # the pinned noise of 1e-8 leaves K with a condition number near 1e8 once there are derivative rows, and the
        # one-ulp differences between numpy's and the device's exp(theta) grow by about that much
        rel = 1e-12 if noisy or g == 0 else 1e-8
        assert r["values"][s] == pytest.approx(f, rel=rel, abs=1e-300)
        np.testing.assert_allclose(r["gradients"][s], gr, rtol=rel, atol=rel * np.max(np.abs(gr)))
        if not noisy:
            assert np.all(r["gradients"][s, 1 + dim:] == 0.0)


# ---- 3. end points against the reference's optimize() ---------------------------------------------------------------
END = [("pinned-prior", 1, (), False, True), ("noisy-none", 1, (), True, False), ("matern-g2", 1, (0, 1), False, True)]


def fd_hessian(f, x, h=1e-4):
    n = len(x)
    Hs = np.empty((n, n))
    for i in range(n):
        for j in range(n):
            ei, ej = np.eye(n)[i] * h, np.eye(n)[j] * h
            Hs[i, j] = (f(x + ei + ej) - f(x + ei - ej) - f(x - ei + ej) + f(x - ei - ej)) / (4 * h * h)
    return 0.5 * (Hs + Hs.T)


@pytest.mark.parametrize("name,kernel,g_idx,noisy,prior", END, ids=[e[0] for e in END])
def test_end_points_match_scipy_bfgs(capi, name, kernel, g_idx, noisy, prior):
    prob = make_problem(15, 2, g_idx=g_idx, seed=3)
    dim, g = 2, len(g_idx)
    p0 = np.concatenate([[0.2], np.full(dim, -0.5), np.full(1 + g, -4.0)])
    lml = checker_lml(kernel, prob)
    nll = lambda t: M.nll(t, lml, dim, g, noisy, prior)  # noqa: E731
    ref = optimize.minimize(nll, p0)  # log_likelihood_mcmc.py:271: minimize(self.nll, p0)
    r = capi.hyperparameter_map(kernel, p0[None], prob["X"], prob["y"], prob["derivs"], noisy=noisy,
                                default_prior=prior)
    assert r["status"][0] == 0, r
    assert np.max(np.abs(r["gradients"][0])) <= 1e-5
    f_s = float(ref.fun)
    assert r["values"][0] <= f_s + 1e-7 * (1 + abs(f_s)), (r["values"][0], f_s)
    free = slice(None) if noisy else slice(0, 1 + dim)
    Hs = fd_hessian(nll, ref.x)[free, free]
    w = np.linalg.eigvalsh(Hs)
    if w.min() >= 1.0 and w.max() / w.min() < 1e6:
        np.testing.assert_allclose(r["positions"][0][free], ref.x[free], atol=1e-4)


# ---- 4. batch invariance ---------------------------------------------------------------------------------------------
def test_start_alone_equals_start_in_permuted_batch(capi):
    prob = make_problem(18, 2, g_idx=(1,), seed=9)
    P = R.initial_walkers(np.random.default_rng(2), 64, 2, 1)
    alone = capi.hyperparameter_map(1, P[17:18], prob["X"], prob["y"], prob["derivs"], noisy=True)
    perm = np.random.default_rng(4).permutation(64)
    batch = capi.hyperparameter_map(1, P[perm], prob["X"], prob["y"], prob["derivs"], noisy=True)
    j = int(np.argwhere(perm == 17)[0, 0])
    for key in alone:
        assert np.array_equal(alone[key][0], batch[key][j], equal_nan=True), key
    assert batch["evaluations"].max() > batch["evaluations"].min()  # the starts really ran different rounds


# ---- 5. status paths --------------------------------------------------------------------------------------------------
def test_status_paths(capi):
    prob = make_problem(15, 2, seed=12)
    P = np.array([[0.5, 1.5, 1.5, -6.0], [0.5, 1.5, 1.5, -6.0], [20.5, 0.0, 0.0, -3.0], [0.3, -0.2, -0.1, -5.0]])
    one = capi.hyperparameter_map(1, P[:1], prob["X"], prob["y"], noisy=True, max_iterations=1)
    assert one["status"][0] == 1 and one["iterations"][0] == 1
    r = capi.hyperparameter_map(1, P, prob["X"], prob["y"], noisy=True, default_prior=False)
    assert r["status"][2] == 2 and r["values"][2] == np.inf and np.array_equal(r["positions"][2], P[2])
    assert r["status"][0] == 0 and r["status"][3] == 0
    for s in (0, 3):  # the failed start leaves the others as they are alone
        alone = capi.hyperparameter_map(1, P[s:s + 1], prob["X"], prob["y"], noisy=True, default_prior=False)
        assert np.array_equal(alone["positions"][0], r["positions"][s]) and alone["values"][0] == r["values"][s]


# ---- 6. size edges ----------------------------------------------------------------------------------------------------
def test_nh_66_at_the_row_bound(capi):
    N = 8192 // 33
    prob = make_problem(N, 32, g_idx=tuple(range(32)), seed=1)
    p0 = np.concatenate([[0.0], np.log(prob["lengths"]), np.full(33, np.log(1e-2))])
    r = capi.hyperparameter_map(1, p0[None], prob["X"], prob["y"], prob["derivs"], noisy=True, default_prior=False,
                                max_iterations=1)
    assert r["positions"].shape == (1, 66) and np.isfinite(r["values"][0])
    assert r["status"][0] in (0, 1) and r["values"][0] <= restated(capi, 1, prob, p0, True, False)[0]


def test_one_start_at_8192_rows(capi):
    prob = make_problem(8192, 1, seed=2)
    p0 = np.array([0.0, np.log(0.3), np.log(1e-2)])
    r = capi.hyperparameter_map(0, p0[None], prob["X"], prob["y"], noisy=True, default_prior=False, max_iterations=1)
    assert np.isfinite(r["values"][0]) and r["status"][0] in (0, 1)


def test_start_count_at_the_chunk_limit(capi):
    prob = make_problem(6, 1, seed=3)
    P = R.initial_walkers(np.random.default_rng(8), 4096, 1, 0)
    r = capi.hyperparameter_map(1, P, prob["X"], prob["y"], max_iterations=3)
    assert r["positions"].shape == (4096, 3) and np.all(np.isin(r["status"], (0, 1, 2, 3)))
    alone = capi.hyperparameter_map(1, P[4095:], prob["X"], prob["y"], max_iterations=3)
    assert np.array_equal(alone["positions"][0], r["positions"][4095])
    with pytest.raises(capi.BoundsError, match="chunk"):
        capi.hyperparameter_map(1, np.vstack([P, P[:1]]), prob["X"], prob["y"])


# ---- 7. the GPP entry -------------------------------------------------------------------------------------------------
def test_gpp_entry_matches_capi_and_optimize(capi):
    import GPP as C_GP
    prob = make_problem(15, 2, seed=21)
    p0 = np.array([0.1, -0.4, -0.6, -4.0])
    pos, vals, status = C_GP.hyperparameter_map_optimization(list(prob["X"].ravel()), list(prob["y"]), 2, 15, [], 0,
                                                             list(p0), 1, False, True)
    r = capi.hyperparameter_map(1, p0[None], prob["X"], prob["y"], noisy=False, default_prior=True)
    assert np.array_equal(np.array(pos), r["positions"][0]) and vals[0] == r["values"][0]
    assert list(status) == [0]
    nll = lambda t: M.nll(t, checker_lml(1, prob), 2, 0, False, True)  # noqa: E731
    ref = optimize.minimize(nll, p0)
    assert vals[0] <= ref.fun + 1e-7 * (1 + abs(ref.fun))

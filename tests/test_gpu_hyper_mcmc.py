"""GPU tests of the hyper-parameter MCMC (cmoe_hyperparameter_mcmc, DESIGN.md K12): table-fed parity with the NumPy
restatement of emcee 2.2.1 and GaussianProcessLogLikelihoodMCMC.compute_log_likelihood (tests/hyper_mcmc_ref.py),
Philox determinism and chain splitting, the stationary distribution against quadrature, the size edges and the GPP
entry."""
import os
import sys

import numpy as np
import pytest

import hyper_mcmc_ref as R
from synth import make_problem

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def list_lml(capi, kernel, prob):
    return lambda H: capi.log_marginal_likelihood_list(kernel, H, prob["X"], prob["y"], prob["derivs"])


# (kernel, observed partials, N, dim, noisy, default prior, walkers): SE and Matern-5/2, g = 0 and 2, noisy and not,
# both priors, N (1 + g) on both sides of the 64-row block edge, 16 and 64 walkers
PARITY = [
    (1, (), 15, 2, False, True, 16),
    (0, (), 63, 2, True, True, 16),
    (1, (), 65, 3, True, False, 64),
    (0, (0, 2), 21, 3, False, False, 16),
    (1, (0, 2), 22, 3, True, True, 64),
    (0, (), 8, 1, False, False, 64),
]
STEPS = 50


@pytest.mark.parametrize("kernel,g_idx,N,dim,noisy,prior,W", PARITY,
                         ids=[f"k{k}-g{len(g)}-N{N}-d{d}-{'noisy' if z else 'pinned'}-{'prior' if p else 'none'}-W{W}"
                              for k, g, N, d, z, p, W in PARITY])
def test_table_fed_chain_matches_restatement(capi, kernel, g_idx, N, dim, noisy, prior, W):
    prob = make_problem(N, dim, g_idx=g_idx, seed=200 + N + dim)
    g = len(g_idx)
    lml = list_lml(capi, kernel, prob)
    lnprob_fn = lambda P: R.log_prob(P, lml, dim, g, noisy, prior)  # noqa: E731
    # seeds for which every decision of the restatement has a margin above 1e-9 and walker 3's out-of-box start is
    # accepted at its first proposal; the search is deterministic
    for seed in range(100):
        p0 = R.initial_walkers(np.random.default_rng(seed), W, dim, g)
        p0[3, 0] = 20.25  # outside the [-20, 20] box: lnp = -inf
        tables = R.random_state_tables(np.random.RandomState(seed), STEPS, W)
        want_p, want_l, acc, margins = R.stretch_chain(p0, STEPS, lnprob_fn, tables)
        if margins.min() > 1e-9 and acc[0, 3]:
            break
    else:
        pytest.fail("no seed with margins above 1e-9")
    assert acc.mean() > 0.05  # the chain moves
    got_p, got_l = capi.hyperparameter_mcmc(kernel, p0, prob["X"], prob["y"], STEPS, derivs=prob["derivs"],
                                            noisy=noisy, default_prior=prior, table=tables)
    assert np.array_equal(got_p, want_p), np.argwhere(got_p != want_p)[:5]
    if not noisy:
        inside = np.all(np.abs(want_p) <= 20, axis=1)
        assert np.all(got_p[inside, 1 + dim:] == R.LOG_NOISE_FREE)
    assert np.array_equal(np.isfinite(got_l), np.isfinite(want_l))
    np.testing.assert_allclose(got_l, want_l, rtol=1e-8)


def test_philox_chain_is_deterministic_and_splits(capi):
    prob = make_problem(20, 2, seed=5)
    p0 = R.initial_walkers(np.random.default_rng(1), 16, 2, 0)
    args = (1, p0, prob["X"], prob["y"])
    a = capi.hyperparameter_mcmc(*args, 30, noisy=False, seed=1234)
    b = capi.hyperparameter_mcmc(*args, 30, noisy=False, seed=1234)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    mid = capi.hyperparameter_mcmc(*args, 12, noisy=False, seed=1234)
    end = capi.hyperparameter_mcmc(1, mid[0], prob["X"], prob["y"], 18, noisy=False, seed=1234, first_step=12)
    assert np.array_equal(end[0], a[0]) and np.array_equal(end[1], a[1])
    other = capi.hyperparameter_mcmc(*args, 30, noisy=False, seed=1235)
    assert not np.array_equal(other[0], a[0])
    assert not np.array_equal(a[0], p0)


def test_stationary_distribution_matches_quadrature(capi):
    """d = 1, N = 5, the default prior, noisy walkers (see hyper_mcmc_ref.stationary_problem for why not pinned): the
    pooled walkers of 64 chains, 1000 burn-in steps then 400 continuation calls of 10 steps, against the posterior
    moments by quadrature with the list call.  Tolerances and their reason: hyper_mcmc_ref.MEAN_TOL_SD, SD_TOL_REL."""
    X, y = R.stationary_problem()
    mean, sd = R.grid_moments(lambda H: capi.log_marginal_likelihood_list(1, H, X, y))
    p = R.initial_walkers(np.random.default_rng(3), 64, 1, 0)
    p, _ = capi.hyperparameter_mcmc(1, p, X, y, 1000, noisy=True, seed=77)
    pool = []
    for c in range(400):
        p, _ = capi.hyperparameter_mcmc(1, p, X, y, 10, noisy=True, seed=77, first_step=1000 + 10 * c)
        pool.append(p.copy())
    ok, m, s = R.stationary_check(np.concatenate(pool), mean, sd)
    assert ok, (mean, sd, m, s)


def test_largest_system_and_bounds(capi):
    X = np.linspace(0.0, 1.0, 8192)[:, None]
    y = np.sin(3.0 * X[:, 0])
    p0 = np.array([[0.0, np.log(0.3), np.log(0.05)]] * 6) + 0.01 * np.arange(18).reshape(6, 3)
    pos, lnp = capi.hyperparameter_mcmc(0, p0, X, y, 1, noisy=True, default_prior=False, seed=3)
    assert pos.shape == (6, 3) and np.all(np.isfinite(lnp))
    with pytest.raises(capi.BoundsError, match="chunk"):
        capi.hyperparameter_mcmc(0, np.vstack([p0, p0[:2]]), X, y, 1)
    with pytest.raises(capi.BoundsError, match="8192"):
        capi.hyperparameter_mcmc(0, p0, np.linspace(0.0, 1.0, 8193)[:, None], np.zeros(8193), 1)
    with pytest.raises(capi.BoundsError, match="even"):
        capi.hyperparameter_mcmc(0, p0[:5], X[:10], y[:10], 1)
    with pytest.raises(capi.BoundsError, match="twice"):
        capi.hyperparameter_mcmc(0, p0[:4], X[:10], y[:10], 1)
    with pytest.raises(capi.BoundsError, match="num_steps"):
        capi.hyperparameter_mcmc(0, p0, X[:10], y[:10], 0)


def test_gpp_entry_matches_capi(capi):
    sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
    import GPP as C_GP
    prob = make_problem(12, 2, g_idx=(1,), seed=8)
    p0 = R.initial_walkers(np.random.default_rng(2), 16, 2, 1)
    pos, lnp = C_GP.sample_hyperparameters_mcmc(list(prob["X"].ravel()), list(prob["y"]), 2, 12, [1], 1,
                                                list(p0.ravel()), 16, 20, False, True, 99, 5)
    want_p, want_l = capi.hyperparameter_mcmc(1, p0, prob["X"], prob["y"], 20, derivs=[1], noisy=False,
                                              default_prior=True, seed=99, first_step=5)
    assert np.array_equal(np.reshape(pos, (16, 5)), want_p) and np.array_equal(lnp, want_l)
    inside = np.all(np.abs(want_p) <= 20, axis=1)
    assert inside.any() and np.all(want_p[inside, 3:] == R.LOG_NOISE_FREE)

"""GPU tests of the log marginal likelihood at a list of hyper-parameter sets (cmoe_log_marginal_likelihood_list,
GPP.evaluate_log_likelihood_at_hyperparameter_list): every set against the CPU checker's single-set value, the GPP
entry point against the answers of the reference's EvaluateLogLikelihoodAtPointList (tests/golden/reference_lml_list.npz,
written by tests/golden/make_lml_list_golden.py), bit-identical values however a set is batched (alone, in a batch,
permuted, across the 4096-set chunk bound), the size edges (n = 8192 across the 2 GiB chunk bound, n = 8193,
num_sets = 0, invalid sets) and a singular set among regular ones."""
import os
import sys

import numpy as np
import pytest

from gpu_util import checker
from synth import make_problem

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_lml_list.npz")


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def gpp():
    sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
    import GPP as C_GP
    return C_GP


def log_sets(rng, num_sets, dim, g, noise_lo=1e-3, noise_hi=1e-1):
    """Sets (alpha, lengths[dim], noise[1 + g]) drawn log-uniformly, the way emcee walkers spread over a log prior."""
    scale = np.sqrt(dim / 8.0) if dim >= 8 else 1.0
    alpha = np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=(num_sets, 1)))
    lengths = scale * np.exp(rng.uniform(np.log(0.25), np.log(1.5), size=(num_sets, dim)))
    noise = np.exp(rng.uniform(np.log(noise_lo), np.log(noise_hi), size=(num_sets, 1 + g)))
    return np.concatenate([alpha, lengths, noise], axis=1)


def per_set_checker(kernel, H, prob):
    dim = prob["dim"]
    return np.array([checker().log_marginal_likelihood(kernel, h[0], h[1:1 + dim], prob["X"], prob["y"], h[1 + dim:],
                                                       prob["derivs"]) for h in H])


FULL3, FULL32 = (0, 1, 2), tuple(range(32))
# (kernel, observed partials, N, dim, num_sets): SE and Matern-5/2; g = 0, 2 and dim; N across the 64-row block edges
PARITY = [
    (0, (), 1, 1, 7),
    (1, (), 2, 3, 7),
    (0, (), 20, 3, 33),
    (1, (), 20, 32, 33),
    (1, (), 64, 1, 33),
    (0, (), 65, 32, 7),
    (0, (), 300, 3, 7),
    (1, (), 300, 32, 1),
    (0, (0, 2), 20, 3, 7),
    (1, (0, 2), 65, 3, 7),
    (1, (0, 2), 2, 32, 1),
    (0, (0,), 20, 1, 33),
    (1, FULL3, 20, 3, 7),
    (0, FULL3, 64, 3, 7),
    (0, FULL32, 2, 32, 7),
    (1, FULL32, 20, 32, 1),
]


@pytest.mark.parametrize("kernel,g_idx,N,dim,num_sets", PARITY,
                         ids=[f"k{k}-g{len(g)}-N{N}-d{d}-s{s}" for k, g, N, d, s in PARITY])
def test_each_set_matches_checker(capi, kernel, g_idx, N, dim, num_sets):
    prob = make_problem(N, dim, g_idx=g_idx, seed=100 + N + dim)
    H = log_sets(np.random.default_rng(N * 7 + dim), num_sets, dim, len(g_idx))
    got = capi.log_marginal_likelihood_list(kernel, H, prob["X"], prob["y"], prob["derivs"])
    want = per_set_checker(kernel, H, prob)
    assert got.shape == (num_sets,) and np.all(np.isfinite(got))
    # the tolerance (and its reason) of test_log_marginal_likelihood_matches_checker: -1/2 y^T K^-1 y and
    # -sum log L_ii nearly cancel at larger N, so factorisation rounding shows up two digits higher in the sum
    np.testing.assert_allclose(got, want, rtol=1e-8)


# ---- the reference's entry point -------------------------------------------------------------------------------------
REF_CASES = {"g0": ((), 20, 3, 7), "g2": ((0, 2), 15, 3, 5)}


def _ref_case(name):
    g_idx, N, dim, num_sets = REF_CASES[name]
    prob = make_problem(N, dim, g_idx=g_idx, seed=61 + N)
    H = log_sets(np.random.default_rng(62 + N), num_sets, dim, len(g_idx))
    return prob, H


@pytest.mark.parametrize("name", sorted(REF_CASES))
def test_gpp_entry_matches_reference(capi, name):
    ref = dict(np.load(GOLDEN))  # the reference's own EvaluateLogLikelihoodAtPointList: make_lml_list_golden.py
    prob, H = _ref_case(name)
    C_GP = gpp()
    dim, g = prob["dim"], len(prob["derivs"])
    status = {}
    vals = C_GP.evaluate_log_likelihood_at_hyperparameter_list(
        list(H.ravel()), list(prob["X"].ravel()), list(prob["y"]), dim, prob["N"],
        C_GP.LogLikelihoodTypes.log_marginal_likelihood, [prob["alpha"], list(prob["lengths"])], list(prob["noise"]),
        [int(a) for a in prob["derivs"]], g, H.shape[0], 8, status)
    np.testing.assert_allclose(vals, ref[f"{name}_values"], rtol=1e-8)
    assert status == {"evaluate_log_marginal_likelihood_at_hyperparameter_list": bool(ref[f"{name}_found"])}


# ---- batch invariance ------------------------------------------------------------------------------------------------
def test_value_does_not_depend_on_the_batch(capi):
    """4097 sets at N = 10 run as chunks of 4096 + 1: a set's value is bit-identical alone, in a batch, under
    permutation and on either side of the chunk split."""
    prob = make_problem(10, 2, seed=3)
    rng = np.random.default_rng(4)
    H = log_sets(rng, 4097, 2, 0)
    args = (prob["X"], prob["y"])
    allv = capi.log_marginal_likelihood_list(1, H, *args)
    assert np.all(np.isfinite(allv))
    for i in (0, 1, 2048, 4095, 4096):
        assert np.array_equal(capi.log_marginal_likelihood_list(1, H[i:i + 1], *args), allv[i:i + 1]), i
    assert np.array_equal(capi.log_marginal_likelihood_list(1, H[4090:], *args), allv[4090:])
    perm = rng.permutation(4097)
    assert np.array_equal(capi.log_marginal_likelihood_list(1, H[perm], *args), allv[perm])
    # derivative observations, several 64-row blocks
    prob = make_problem(30, 3, g_idx=(0, 2), seed=5)
    H = log_sets(rng, 33, 3, 2)
    args = (prob["X"], prob["y"], prob["derivs"])
    allv = capi.log_marginal_likelihood_list(0, H, *args)
    perm = rng.permutation(33)
    assert np.array_equal(capi.log_marginal_likelihood_list(0, H[perm], *args), allv[perm])
    assert np.array_equal(capi.log_marginal_likelihood_list(0, H[17:18], *args), allv[17:18])


# ---- size edges ------------------------------------------------------------------------------------------------------
def test_largest_system_across_the_workspace_bound(capi):
    """n = 8192: one set's matrix and staging take 516 MiB, so 4 sets run as chunks of 3 + 1."""
    prob = make_problem(8192, 4, seed=9, noise=0.05)
    rng = np.random.default_rng(10)
    H = log_sets(rng, 4, 4, 0, noise_lo=0.02, noise_hi=0.1)
    got = capi.log_marginal_likelihood_list(0, H, prob["X"], prob["y"])
    assert np.all(np.isfinite(got))
    single = np.array([capi.log_marginal_likelihood(0, h[0], h[1:5], prob["X"], prob["y"], h[5:]) for h in H])
    np.testing.assert_allclose(got, single, rtol=1e-8)
    assert np.array_equal(capi.log_marginal_likelihood_list(0, H[3:], prob["X"], prob["y"]), got[3:])


def test_size_and_set_checks(capi):
    X = np.linspace(0.0, 1.0, 8193)[:, None]
    with pytest.raises(capi.BoundsError, match="8192"):
        capi.log_marginal_likelihood_list(0, [[1.0, 0.5, 0.01]], X, np.zeros(8193))
    with pytest.raises(capi.BoundsError, match="8192"):  # n = N (1 + g) = 2731 * 3
        capi.log_marginal_likelihood_list(0, [[1.0, 0.5, 0.5, 0.01, 0.01, 0.01]], np.zeros((2731, 2)),
                                          np.zeros(2731 * 3), [0, 1])
    prob = make_problem(5, 2, seed=1)
    with pytest.raises(capi.BoundsError):
        capi.log_marginal_likelihood_list(0, np.zeros((0, 4)), prob["X"], prob["y"])
    good = [1.0, 0.5, 0.5, 0.01]
    with pytest.raises(capi.BoundsError, match="set 3: Invalid hyperparameter \\(alpha\\)"):
        capi.log_marginal_likelihood_list(0, [good] * 3 + [[0.0, 0.5, 0.5, 0.01]], prob["X"], prob["y"])
    with pytest.raises(capi.BoundsError, match="set 1: Invalid hyperparameter \\(length\\)"):
        capi.log_marginal_likelihood_list(1, [good, [1.0, 0.5, -0.5, 0.01]], prob["X"], prob["y"])


# ---- singular sets ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", [0, 1])
def test_singular_set_is_minus_infinity_and_leaves_the_others(capi, kernel):
    """A duplicate point with noise -1e-6 (so noise + 1e-6 is exactly 0) and alpha = 1: the second copy's pivot is
    exactly 0 for the single call and here."""
    prob = make_problem(12, 3, g_idx=(1,), seed=31)
    X = prob["X"].copy()
    X[1] = X[0]
    y, derivs = prob["y"], prob["derivs"]
    H = log_sets(np.random.default_rng(32), 5, 3, 1)
    H[2] = [1.0, 0.4, 0.6, 0.8, -1e-6, -1e-6]
    single = capi.log_marginal_likelihood(kernel, 1.0, H[2, 1:4], X, y, H[2, 4:], derivs)
    assert single == -np.inf
    got = capi.log_marginal_likelihood_list(kernel, H, X, y, derivs)
    assert got[2] == -np.inf
    for i in (0, 1, 3, 4):
        assert np.isfinite(got[i])
        assert np.array_equal(capi.log_marginal_likelihood_list(kernel, H[i:i + 1], X, y, derivs), got[i:i + 1])
        np.testing.assert_allclose(got[i], capi.log_marginal_likelihood(kernel, H[i, 0], H[i, 1:4], X, y, H[i, 4:],
                                                                        derivs), rtol=1e-8)
    if kernel != 1:
        return
    C_GP = gpp()

    def call(Hs):
        status = {}
        vals = C_GP.evaluate_log_likelihood_at_hyperparameter_list(
            list(Hs.ravel()), list(X.ravel()), list(y), 3, 12, C_GP.LogLikelihoodTypes.log_marginal_likelihood,
            [1.0, [0.5, 0.5, 0.5]], [0.01, 0.01], [1], 1, Hs.shape[0], 1, status)
        return np.array(vals), status["evaluate_log_marginal_likelihood_at_hyperparameter_list"]

    vals, found = call(H)
    assert np.array_equal(vals, got) and found is True
    vals, found = call(H[[2, 2, 2]])
    assert np.all(vals == -np.inf) and found is False

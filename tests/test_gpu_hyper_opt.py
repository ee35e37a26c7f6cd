"""GPU tests of the hyper-parameter gradient at a list of sets (cmoe_grad_log_marginal_likelihood_list), the multistart
hyper-parameter descent on top of it (cmoe_hyperparameter_gradient_descent) and the GPP entries
multistart_hyperparameter_optimization / restarted_hyperparameter_optimization: every set's gradient against the CPU
checker, bit-identical results however a set is batched, the size edges, singular sets, the descent against a numpy
restatement of the reference's optimiser, and the GPP entries against the answers of the reference's own drivers
(tests/golden/reference_hyper_opt.npz, written by tests/golden/make_hyper_opt_golden.py)."""
import os
import sys

import numpy as np
import pytest

from gpu_util import checker
from synth import make_problem
from test_gpu_lml_list import PARITY, log_sets

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_hyper_opt.npz")


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def gpp():
    sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
    import GPP as C_GP
    return C_GP


def checker_grads(kernel, H, prob):
    dim = prob["dim"]
    return np.array([checker().grad_log_marginal_likelihood(kernel, h[0], h[1:1 + dim], prob["X"], prob["y"],
                                                            h[1 + dim:], prob["derivs"]) for h in H])


# ---- gradient list against the checker -------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel,g_idx,N,dim,num_sets", PARITY,
                         ids=[f"k{k}-g{len(g)}-N{N}-d{d}-s{s}" for k, g, N, d, s in PARITY])
def test_each_gradient_matches_checker(capi, kernel, g_idx, N, dim, num_sets):
    prob = make_problem(N, dim, g_idx=g_idx, seed=100 + N + dim)
    H = log_sets(np.random.default_rng(N * 7 + dim), num_sets, dim, len(g_idx))
    vals, grads = capi.grad_log_marginal_likelihood_list(kernel, H, prob["X"], prob["y"], prob["derivs"])
    assert np.array_equal(vals, capi.log_marginal_likelihood_list(kernel, H, prob["X"], prob["y"], prob["derivs"]))
    want = checker_grads(kernel, H, prob)
    assert grads.shape == want.shape
    for got_s, want_s in zip(grads, want):  # the tolerance of test_grad_log_marginal_likelihood_matches_reference
        np.testing.assert_allclose(got_s, want_s, rtol=1e-7, atol=1e-9 * np.max(np.abs(want_s)))


# ---- batch invariance ------------------------------------------------------------------------------------------------
def test_gradient_does_not_depend_on_the_batch(capi):
    """4097 sets at N = 10 run as chunks of 4096 + 1; several 64-row blocks with derivative rows."""
    prob = make_problem(10, 2, seed=3)
    rng = np.random.default_rng(4)
    H = log_sets(rng, 4097, 2, 0)
    args = (prob["X"], prob["y"])
    allv, allg = capi.grad_log_marginal_likelihood_list(1, H, *args)
    assert np.all(np.isfinite(allg))
    for i in (0, 1, 2048, 4095, 4096):
        v, g = capi.grad_log_marginal_likelihood_list(1, H[i:i + 1], *args)
        assert np.array_equal(v, allv[i:i + 1]) and np.array_equal(g, allg[i:i + 1]), i
    v, g = capi.grad_log_marginal_likelihood_list(1, H[4090:], *args)
    assert np.array_equal(g, allg[4090:])
    perm = rng.permutation(4097)
    v, g = capi.grad_log_marginal_likelihood_list(1, H[perm], *args)
    assert np.array_equal(v, allv[perm]) and np.array_equal(g, allg[perm])
    prob = make_problem(150, 3, g_idx=(0, 2), seed=5)
    H = log_sets(rng, 9, 3, 2)
    args = (prob["X"], prob["y"], prob["derivs"])
    for kernel in (0, 1):
        allv, allg = capi.grad_log_marginal_likelihood_list(kernel, H, *args)
        perm = rng.permutation(9)
        v, g = capi.grad_log_marginal_likelihood_list(kernel, H[perm], *args)
        assert np.array_equal(g, allg[perm])
        v, g = capi.grad_log_marginal_likelihood_list(kernel, H[4:5], *args)
        assert np.array_equal(g, allg[4:5])


# ---- size edges ------------------------------------------------------------------------------------------------------
def test_largest_system_across_the_workspace_bound(capi):
    """n = 8192: a set's factor, inverse and staging take over 1 GiB, so 2 sets run as two chunks of one."""
    prob = make_problem(8192, 4, seed=9, noise=0.05)
    H = log_sets(np.random.default_rng(10), 2, 4, 0, noise_lo=0.02, noise_hi=0.1)
    vals, grads = capi.grad_log_marginal_likelihood_list(0, H, prob["X"], prob["y"])
    assert np.all(np.isfinite(grads))
    assert np.array_equal(vals, capi.log_marginal_likelihood_list(0, H, prob["X"], prob["y"]))
    single = capi.grad_log_marginal_likelihood(0, H[1, 0], H[1, 1:5], prob["X"], prob["y"], H[1, 5:])
    np.testing.assert_allclose(grads[1], single, rtol=1e-6, atol=1e-8 * np.max(np.abs(single)))
    v, g = capi.grad_log_marginal_likelihood_list(0, H[1:], prob["X"], prob["y"])
    assert np.array_equal(g, grads[1:])


def test_size_and_set_checks(capi):
    X = np.linspace(0.0, 1.0, 8193)[:, None]
    with pytest.raises(capi.BoundsError, match="8192"):
        capi.grad_log_marginal_likelihood_list(0, [[1.0, 0.5, 0.01]], X, np.zeros(8193))
    prob = make_problem(5, 2, seed=1)
    with pytest.raises(capi.BoundsError):
        capi.grad_log_marginal_likelihood_list(0, np.zeros((0, 4)), prob["X"], prob["y"])
    good = [1.0, 0.5, 0.5, 0.01]
    with pytest.raises(capi.BoundsError, match="set 3: Invalid hyperparameter \\(alpha\\)"):
        capi.grad_log_marginal_likelihood_list(0, [good] * 3 + [[0.0, 0.5, 0.5, 0.01]], prob["X"], prob["y"])
    with pytest.raises(capi.BoundsError, match="set 1: Invalid hyperparameter \\(length\\)"):
        capi.grad_log_marginal_likelihood_list(1, [good, [1.0, 0.5, -0.5, 0.01]], prob["X"], prob["y"])


# ---- singular sets ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", [0, 1])
def test_singular_set_gets_zeros_and_leaves_the_others(capi, kernel):
    prob = make_problem(12, 3, g_idx=(1,), seed=31)
    X = prob["X"].copy()
    X[1] = X[0]
    y, derivs = prob["y"], prob["derivs"]
    H = log_sets(np.random.default_rng(32), 5, 3, 1)
    H[2] = [1.0, 0.4, 0.6, 0.8, -1e-6, -1e-6]
    vals, grads = capi.grad_log_marginal_likelihood_list(kernel, H, X, y, derivs)
    assert vals[2] == -np.inf and np.all(grads[2] == 0.0)
    for i in (0, 1, 3, 4):
        v, g = capi.grad_log_marginal_likelihood_list(kernel, H[i:i + 1], X, y, derivs)
        assert np.isfinite(v[0]) and np.array_equal(g[0], grads[i])


# ---- the descent driver against a restatement of the reference's optimiser -------------------------------------------
def _limit_step(step, x, lo, hi, mrc):
    """TensorProductDomain::LimitUpdate for one coordinate (gpp_domain.cpp:64-104)."""
    dist = min(x - lo, hi - x)
    if abs(step) > mrc * dist:
        step = np.copysign(mrc * dist, step)
    nxt = x + step
    if nxt < lo:
        step = (lo - x) * 0.5 if x + step * 0.5 < lo else step * 0.5
    elif nxt > hi:
        step = (hi - x) * 0.5 if x + step * 0.5 > hi else step * 0.5
    return step


def _restated_descent(grad, x0, gd, bounds):
    """GradientDescentOptimizer::Optimize / GradientDescentOptimization (gpp_optimization.hpp:620-705, 1144-1185)."""
    _, max_steps, max_restarts, _, gamma, pre_mult, mrc, tol = gd
    x = np.array(x0, dtype=np.float64)
    for _ in range(int(max_restarts)):
        start = x.copy()
        for i in range(int(max_steps)):
            g = grad(x)
            a = pre_mult * (i + 1.0) ** (-gamma)
            step = np.array([_limit_step(a * g[k], x[k], bounds[k, 0], bounds[k, 1], mrc) for k in range(x.size)])
            x = x + step
            if np.linalg.norm(step) < tol / max_steps:
                break
        if np.linalg.norm(start - x) <= tol:
            break
    return x


GD = (8, 15, 2, 0, 0.5, 0.02, 0.2, 1e-7)


def _descent_problem():
    prob = make_problem(25, 2, g_idx=(1,), seed=71, noise=0.02)
    bounds = np.array([[0.3, 3.0], [0.1, 2.0], [0.1, 2.0], [1e-4, 0.1], [1e-4, 0.1]])
    rng = np.random.default_rng(72)
    starts = bounds[:, 0] + (bounds[:, 1] - bounds[:, 0]) * rng.uniform(0.2, 0.8, size=(256, 5))
    return prob, bounds, starts


def test_descent_matches_restated_reference(capi):
    prob, bounds, starts = _descent_problem()
    best, best_v, found, ends, end_v = capi.hyperparameter_gradient_descent(1, GD, bounds, starts[:8], prob["X"],
                                                                            prob["y"], prob["derivs"])
    d = prob["dim"]

    def grad(h):
        return checker().grad_log_marginal_likelihood(1, h[0], h[1:1 + d], prob["X"], prob["y"], h[1 + d:],
                                                      prob["derivs"])

    for s in range(8):
        want = _restated_descent(grad, starts[s], GD, bounds)
        np.testing.assert_allclose(ends[s], want, rtol=1e-6)
    np.testing.assert_array_equal(end_v, capi.log_marginal_likelihood_list(1, ends, prob["X"], prob["y"],
                                                                           prob["derivs"]))
    start_v = capi.log_marginal_likelihood_list(1, starts[:8], prob["X"], prob["y"], prob["derivs"])
    assert found == (np.max(start_v) < np.max(end_v))
    if found:
        assert np.array_equal(best, ends[int(np.argmax(end_v))]) and best_v == np.max(end_v)


def test_descent_end_points_do_not_depend_on_the_batch(capi):
    prob, bounds, starts = _descent_problem()
    args = (prob["X"], prob["y"], prob["derivs"])
    _, _, _, ends, end_v = capi.hyperparameter_gradient_descent(1, GD, bounds, starts, *args)
    for s in (0, 17, 255):
        _, _, _, e1, v1 = capi.hyperparameter_gradient_descent(1, GD, bounds, starts[s:s + 1], *args)
        assert np.array_equal(e1[0], ends[s]) and v1[0] == end_v[s], s


# ---- the GPP entries against the reference's drivers -----------------------------------------------------------------
# name: (observed partials, N, dim, optimizer (0: LHC search, 1: gradient descent), GradientDescentParameters, seed)
REF_CASES = {
    "gd_g0": ((), 40, 2, 1, (24, 30, 1, 0, 0.5, 0.02, 0.2, 1e-7), 7),
    "gd_g2": ((0, 2), 20, 3, 1, (16, 20, 2, 0, 0.5, 0.01, 0.2, 1e-7), 11),
    "lhc_g0": ((), 30, 3, 0, (40, 1, 1, 0, 0.5, 0.02, 0.2, 1e-7), 13),
    "lhc_g2": ((0, 2), 20, 3, 0, (30, 1, 1, 0, 0.5, 0.02, 0.2, 1e-7), 17),
}
NUM_CALLS = 2  # two consecutive calls on one generator pin the advance of the uniform stream


def ref_case(name):
    g_idx, N, dim, optimizer, gd, seed = REF_CASES[name]
    prob = make_problem(N, dim, g_idx=g_idx, seed=seed, noise=0.02)
    nh = 2 + dim + len(g_idx)
    log_domain = np.array([[-0.5, 0.5]] + [[-1.0, 0.3]] * dim + [[-4.0, -1.0]] * (1 + len(g_idx)))
    assert log_domain.shape == (nh, 2)
    return prob, log_domain, optimizer, gd, seed


class _OptimizerParameters:
    """What cpp_wrappers/optimization.py passes as optimizer_parameters (gpp_python_model_selection.cpp:236-244)."""

    def __init__(self, C_GP, optimizer, gd, objective=None):
        self.domain_type = C_GP.DomainTypes.tensor_product
        self.objective_type = objective if objective is not None else C_GP.LogLikelihoodTypes.log_marginal_likelihood
        self.optimizer_type = (C_GP.OptimizerTypes.null, C_GP.OptimizerTypes.gradient_descent,
                               C_GP.OptimizerTypes.newton)[optimizer]
        self.num_random_samples = gd[0]
        self.optimizer_parameters = C_GP.GradientDescentParameters(*gd)


def _args(prob, log_domain):
    d, g = prob["dim"], len(prob["derivs"])
    return (list(log_domain.ravel()), list(prob["X"].ravel()), list(prob["y"]), d, prob["N"],
            [prob["alpha"], list(prob["lengths"])], list(prob["noise"]), [int(a) for a in prob["derivs"]], g)


@pytest.mark.parametrize("name", sorted(REF_CASES))
def test_multistart_entry_matches_reference(capi, name):
    ref = dict(np.load(GOLDEN))
    prob, log_domain, optimizer, gd, seed = ref_case(name)
    C_GP = gpp()
    params = _OptimizerParameters(C_GP, optimizer, gd)
    rnd = C_GP.RandomnessSourceContainer(1)
    rnd.SetExplicitUniformGeneratorSeed(seed)
    key = ("log_marginal_likelihood_lhc_found_update", "log_marginal_likelihood_gradient_descent_found_update")[optimizer]
    for c in range(NUM_CALLS):
        status = {}
        best = np.array(C_GP.multistart_hyperparameter_optimization(params, *_args(prob, log_domain), 4, rnd, status))
        assert status == {key: bool(ref[f"{name}_found"][c])}
        if optimizer == 0:  # a start drawn by the same engine
            np.testing.assert_allclose(best, ref[f"{name}_best"][c], rtol=1e-13)
        else:
            np.testing.assert_allclose(best, ref[f"{name}_best"][c], rtol=1e-6)


@pytest.mark.parametrize("name", ["gd_g0", "gd_g2"])
def test_restarted_entry_matches_reference(capi, name):
    ref = dict(np.load(GOLDEN))
    prob, log_domain, _, gd, _ = ref_case(name)
    C_GP = gpp()
    params = _OptimizerParameters(C_GP, 1, gd)
    starts = ref[f"{name}_starts"][0]
    for s in range(4):
        p = dict(prob)
        d = prob["dim"]
        p["alpha"], p["lengths"], p["noise"] = starts[s, 0], starts[s, 1:1 + d], starts[s, 1 + d:]
        got = C_GP.restarted_hyperparameter_optimization(params, *_args(p, log_domain), {})
        np.testing.assert_allclose(got, ref[f"{name}_restarted"][s], rtol=1e-6)


def test_restarted_without_restarts_returns_zeros(capi):
    prob, log_domain, _, gd, _ = ref_case("gd_g2")
    C_GP = gpp()
    params = _OptimizerParameters(C_GP, 1, gd[:2] + (0,) + gd[3:])
    assert C_GP.restarted_hyperparameter_optimization(params, *_args(prob, log_domain), {}) == [0.0] * 7


def test_multistart_without_restarts_returns_the_best_start(capi):
    prob, log_domain, _, gd, seed = ref_case("gd_g0")
    C_GP = gpp()
    params = _OptimizerParameters(C_GP, 1, gd[:2] + (0,) + gd[3:])
    rnd = C_GP.RandomnessSourceContainer(1)
    rnd.SetExplicitUniformGeneratorSeed(seed)
    status = {}
    best = C_GP.multistart_hyperparameter_optimization(params, *_args(prob, log_domain), 1, rnd, status)
    assert status == {"log_marginal_likelihood_gradient_descent_found_update": False}
    starts = np.load(GOLDEN)["gd_g0_starts"][0]
    vals = capi.log_marginal_likelihood_list(1, starts, prob["X"], prob["y"])
    # the reference's starts: the same draws, the box arithmetic of the two Latin hypercubes differs by rounding
    np.testing.assert_allclose(best, starts[int(np.argmax(vals))], rtol=1e-13)


def test_newton_and_leave_one_out_raise_the_reference_messages(capi):
    prob, log_domain, _, gd, _ = ref_case("gd_g0")
    C_GP = gpp()
    rnd = C_GP.RandomnessSourceContainer(1)
    with pytest.raises(C_GP.OptimalLearningException, match="ERROR: invalid optimizer choice. Setting all "
                                                            "hyperparameters to 1.0."):
        C_GP.multistart_hyperparameter_optimization(_OptimizerParameters(C_GP, 2, gd), *_args(prob, log_domain), 1,
                                                    rnd, {})
    loo = C_GP.LogLikelihoodTypes.leave_one_out_log_likelihood
    with pytest.raises(C_GP.OptimalLearningException, match="ERROR: invalid objective type choice. Setting all "
                                                            "hyperparameters to 1.0."):
        C_GP.multistart_hyperparameter_optimization(_OptimizerParameters(C_GP, 1, gd, loo), *_args(prob, log_domain),
                                                    1, rnd, {})

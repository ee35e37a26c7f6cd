"""GPU tests of heuristic batch EI (cmoe_heuristic_ei, GPP.heuristic_expected_improvement_optimization, DESIGN.md K20).

The oracle is the q-round loop of calls already checked against the reference: a fresh GP handle with the same data,
cmoe_multistart_ei with q = 1 on the round's start block, cmoe_gp_posterior at the chosen point and
cmoe_gp_add_sampled_points with the policy's value.  Where the policy's noise differs from the GP's, the NumPy refit of
tests/heuristic_ei_ref.py is the oracle instead."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

import heuristic_ei_ref as R  # noqa: E402
from synth import make_problem, unit_bounds  # noqa: E402

pytestmark = pytest.mark.gpu

# examples/main.py's cpp_sgd_params_kg with 40 starts per round
GD = [40, 50, 2, 4, 0.7, 1.0, 0.5, 1.0e-10]
POLICIES = [("CL", capi.CONSTANT_LIAR, None), ("KB0", capi.KRIGING_BELIEVER, 0.0), ("KB1", capi.KRIGING_BELIEVER, 1.0)]
SHAPES = [(20, 2), (200, 5), (1000, 5)]


def _gp(pr, kernel):
    return capi.GaussianProcess(kernel, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"])


def _estimate(kind, value, mu, var):
    return value if kind == capi.CONSTANT_LIAR else mu + value * np.sqrt(max(var, 0.0))


def _margin_ok(vals, ends):
    """The winner's final EI beats every kept start that ended elsewhere (farther than 1e-6 of the unit box) by more than
    1e-8 relative: starts that reach the same optimum tie by construction and choose the same point."""
    w = int(np.argmax(vals))
    far = np.abs(ends - ends[w]).max(axis=1) > 1e-6
    return not far.any() or (vals[w] - vals[far].max()) > 1e-8 * abs(vals[w])


def _loop(pr, kernel, starts, best, kind, value, gd):
    """The q rounds from existing calls; returns (points, fantasy values, EI values, found, margins held)."""
    gp = _gp(pr, kernel)
    q, ns, dim = starts.shape
    bounds = unit_bounds(dim)
    pts, fv, ev, found, ok = [], [], [], [], True
    for r in range(q):
        S = starts[r]
        if gd is None:
            vals = capi.ei_analytic(gp, S, best)
            bv, bi = -1.0, -1
            for i, v in enumerate(vals):
                if bv < v:
                    bv, bi = v, i
            point, f = (S[bi] if bi >= 0 else S[0]), bi >= 0
        else:
            point, bv, f, screen = capi.multistart_ei(gp, S[:, None, :], None, 1, best, gd, bounds)
            point = point[0]
            top = np.argsort(-screen, kind="stable")[:20]
            fin, ends = capi.ei_gradient_descent(gp, S[top][:, None, :], None, 1, best, gd, bounds)
            ok = ok and _margin_ok(fin, ends[:, 0, :])
        post = gp.posterior(point.reshape(1, 1, dim))
        y = _estimate(kind, value, post["mean"][0, 0], post["var"][0, 0])
        pts.append(point.copy())
        fv.append(y)
        ev.append(bv)
        found.append(bool(f))
        gp.add_sampled_points(point[None], [y])
    return np.array(pts), np.array(fv), np.array(ev), np.array(found), ok


def _assert_matches(got, want):
    pts, fv, ev, found = got
    wp, wf, we, wfound = want
    np.testing.assert_allclose(pts, wp, rtol=0, atol=1e-7)  # the unit box: 1e-7 of its width
    np.testing.assert_allclose(fv, wf, rtol=1e-9, atol=1e-14)
    np.testing.assert_allclose(ev, we, rtol=1e-9, atol=1e-14)
    np.testing.assert_array_equal(found, wfound)


@pytest.mark.parametrize("N,dim", SHAPES, ids=[f"N{n}d{d}" for n, d in SHAPES])
@pytest.mark.parametrize("q", [1, 3, 8])
@pytest.mark.parametrize("pname,kind,coef", POLICIES, ids=[p[0] for p in POLICIES])
@pytest.mark.parametrize("kernel", [capi.SQUARE_EXPONENTIAL, capi.MATERN_NU_2P5], ids=["SE", "M52"])
def test_matches_the_loop_of_existing_calls(kernel, pname, kind, coef, q, N, dim):
    pr = make_problem(N, dim, seed=N + dim + kernel)
    best = float(pr["y"].min())
    value = best if kind == capi.CONSTANT_LIAR else coef
    gp = _gp(pr, kernel)
    for seed in (q, q + 100, q + 200):  # the first seed whose every round has a clear winner
        starts = np.random.default_rng(seed).uniform(size=(q, GD[0], dim))
        want = _loop(pr, kernel, starts, best, kind, value, GD)
        if want[4]:
            break
    else:
        pytest.fail("no seed gives every round a winner 1e-8 ahead of the runner-up")
    got = capi.heuristic_ei(gp, starts, best, kind, value, pr["noise"][0], GD, unit_bounds(dim))
    _assert_matches(got, want[:4])


def test_one_point_equals_the_multistart_gpp_entry():
    pr = make_problem(60, 3, seed=7)
    gpp = C_GP.GaussianProcess([1.0, list(pr["lengths"])], list(pr["X"].ravel()), list(pr["y"]), list(pr["noise"]), [],
                               0, 3, 60)
    params = type("P", (), dict(domain_type=C_GP.DomainTypes.tensor_product,
                                optimizer_type=C_GP.OptimizerTypes.gradient_descent, num_random_samples=16,
                                optimizer_parameters=C_GP.GradientDescentParameters(*GD)))
    best = float(pr["y"].min())
    out = []
    for entry in ("multistart", "heuristic"):
        rnd = C_GP.RandomnessSourceContainer(1)
        rnd.SetExplicitUniformGeneratorSeed(2024)
        status = {}
        if entry == "multistart":
            out.append(C_GP.multistart_expected_improvement_optimization(params, gpp, list(unit_bounds(3)), [], 1, 0,
                                                                         best, 1000, 1, False, 0, rnd, status))
        else:
            out.append(C_GP.heuristic_expected_improvement_optimization(
                params, gpp, list(unit_bounds(3)), C_GP.ConstantLiarEstimationPolicy(best, 0.01), 1, best, 1, rnd,
                status))
        assert status["gradient_descent_tensor_product_domain_found_update"] is True
    np.testing.assert_allclose(out[1], out[0], rtol=0, atol=1e-7)


@pytest.mark.parametrize("pname,kind,coef", POLICIES, ids=[p[0] for p in POLICIES])
def test_random_search_matches_the_loop(pname, kind, coef):
    pr = make_problem(200, 5, seed=3)
    best = float(pr["y"].min())
    value = best if kind == capi.CONSTANT_LIAR else coef
    starts = np.random.default_rng(11).uniform(size=(4, 500, 5))
    want = _loop(pr, capi.MATERN_NU_2P5, starts, best, kind, value, None)
    got = capi.heuristic_ei(_gp(pr, capi.MATERN_NU_2P5), starts, best, kind, value, pr["noise"][0], None,
                            unit_bounds(5))
    np.testing.assert_array_equal(got[0], want[0])  # the chosen starts themselves
    np.testing.assert_array_equal(got[2], want[2])  # the screen's values, bit for bit
    np.testing.assert_array_equal(got[3], want[3])
    np.testing.assert_allclose(got[1], want[1], rtol=1e-9, atol=1e-14)


@pytest.mark.parametrize("kernel", [capi.SQUARE_EXPONENTIAL, capi.MATERN_NU_2P5], ids=["SE", "M52"])
@pytest.mark.parametrize("pname,kind,coef", POLICIES, ids=[p[0] for p in POLICIES])
@pytest.mark.parametrize("N,dim", [(20, 2), (200, 5)], ids=["N20d2", "N200d5"])
def test_policy_noise_against_the_numpy_refit(kernel, pname, kind, coef, N, dim):
    pr = make_problem(N, dim, seed=5 + N)
    best = float(pr["y"].min())
    value = best + 0.3 if kind == capi.CONSTANT_LIAR else coef
    noise = 0.07  # the GP's noise is 0.01
    starts = np.random.default_rng(9).uniform(size=(4, 30, dim))
    pts, fv, ev, found = capi.heuristic_ei(_gp(pr, kernel), starts, best, kind, value, noise, GD, unit_bounds(dim))
    assert found.all()
    ref = R.rounds(kernel, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"][0], pts, fv, noise, best)
    for r, (mu, var, ei) in enumerate(ref):
        np.testing.assert_allclose(ev[r], ei, rtol=1e-10, atol=1e-15)
        np.testing.assert_allclose(fv[r], _estimate(kind, value, mu, var), rtol=1e-10, atol=1e-15)


def _snapshot(gp, probe, best):
    K, kinvy, mean = gp.state()
    return K, kinvy, mean, capi.lib().cmoe_gp_num_sampled(gp.h), capi.ei_analytic(gp, probe, best)


def _assert_same(a, b):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_handle_unchanged_and_singular_fantasy():
    """A degenerate box at a point away from the data, zero noise, Constant Liar with noise 0: round 1 appends the
    point of round 0 again, whose leading minor fails.  The caller's handle is bit-identical after the successful call
    and after the failed one, and so is a later evaluation on it."""
    pr = make_problem(20, 2, seed=1, noise=0.0)
    gp = _gp(pr, capi.MATERN_NU_2P5)
    probe = np.random.default_rng(4).uniform(size=(16, 2))
    best = float(pr["y"].min())
    before = _snapshot(gp, probe, best)
    starts = np.random.default_rng(2).uniform(size=(3, 25, 2))
    capi.heuristic_ei(gp, starts, best, capi.KRIGING_BELIEVER, 1.0, 0.01, GD, unit_bounds(2))
    _assert_same(before, _snapshot(gp, probe, best))
    box = np.tile([1.5, 1.5], 2)
    degenerate = np.full((2, 8, 2), 1.5)
    with pytest.raises(capi.SingularMatrixError) as e:
        capi.heuristic_ei(gp, degenerate, best, capi.CONSTANT_LIAR, best, 0.0, GD, box)
    assert e.value.info == 20 + 2  # the second appended row of the 22-row factor
    _assert_same(before, _snapshot(gp, probe, best))
    # argument errors that need the handle: an empty box, and a GP with derivative observations
    with pytest.raises(capi.BoundsError):
        capi.heuristic_ei(gp, starts, best, capi.CONSTANT_LIAR, best, 0.0, GD, np.tile([1.0, 0.0], 2))
    dpr = make_problem(10, 2, g_idx=(0,), seed=2)
    dgp = capi.GaussianProcess(capi.MATERN_NU_2P5, 1.0, dpr["lengths"], dpr["X"], dpr["y"], dpr["noise"], dpr["derivs"])
    with pytest.raises(capi.BoundsError, match="derivative"):
        capi.heuristic_ei(dgp, starts, best, capi.CONSTANT_LIAR, best, 0.0, GD, unit_bounds(2))
    _assert_same(before, _snapshot(gp, probe, best))


def test_reproducible_and_the_gpp_entry_equals_its_loop():
    pr = make_problem(80, 3, seed=13)
    best = float(pr["y"].min())
    gp = _gp(pr, capi.MATERN_NU_2P5)
    starts = np.random.default_rng(21).uniform(size=(5, 40, 3))
    a = capi.heuristic_ei(gp, starts, best, capi.KRIGING_BELIEVER, 1.0, 0.01, GD, unit_bounds(3))
    b = capi.heuristic_ei(gp, starts, best, capi.KRIGING_BELIEVER, 1.0, 0.01, GD, unit_bounds(3))
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)

    def gpp_gp():
        return C_GP.GaussianProcess([1.0, list(pr["lengths"])], list(pr["X"].ravel()), list(pr["y"]),
                                    list(pr["noise"]), [], 0, 3, 80)

    params = type("P", (), dict(domain_type=C_GP.DomainTypes.tensor_product,
                                optimizer_type=C_GP.OptimizerTypes.gradient_descent, num_random_samples=16,
                                optimizer_parameters=C_GP.GradientDescentParameters(*GD)))
    lie = best + 0.1
    rnd = C_GP.RandomnessSourceContainer(1)
    rnd.SetExplicitUniformGeneratorSeed(77)
    status = {}
    whole = C_GP.heuristic_expected_improvement_optimization(params, gpp_gp(), list(unit_bounds(3)),
                                                             C_GP.ConstantLiarEstimationPolicy(lie, 0.01), 3, best, 1,
                                                             rnd, status)
    assert status["gradient_descent_tensor_product_domain_found_update"] is True
    rnd2 = C_GP.RandomnessSourceContainer(1)
    rnd2.SetExplicitUniformGeneratorSeed(77)
    loop_gp = gpp_gp()
    rounds = []
    for _ in range(3):
        pt = C_GP.heuristic_expected_improvement_optimization(params, loop_gp, list(unit_bounds(3)),
                                                              C_GP.ConstantLiarEstimationPolicy(lie, 0.01), 1, best, 1,
                                                              rnd2, {})
        rounds.extend(pt)
        loop_gp.add_sampled_points(list(pt), [lie], 1)
    np.testing.assert_allclose(whole, rounds, rtol=0, atol=1e-7)
    # random search only: the status key of the kNull branch
    params.optimizer_type = C_GP.OptimizerTypes.null
    status = {}
    pts = C_GP.heuristic_expected_improvement_optimization(params, gpp_gp(), list(unit_bounds(3)),
                                                           C_GP.KrigingBelieverEstimationPolicy(0.5, 0.01), 2, best, 1,
                                                           rnd, status)
    assert len(pts) == 6 and status["lhc_tensor_product_domain_found_update"] is True
    params.domain_type = C_GP.DomainTypes.simplex
    with pytest.raises(C_GP.OptimalLearningException, match="tensor_product"):
        C_GP.heuristic_expected_improvement_optimization(params, gpp_gp(), list(unit_bounds(3)),
                                                         C_GP.KrigingBelieverEstimationPolicy(0.5, 0.01), 2, best, 1,
                                                         rnd, {})

"""GPU tests of the LCB batch selection (cmoe_lcb_select, DESIGN.md K13): selections, mean and sd against the unmodified
reference routine (tests/golden/reference_lcb.npz), including its singular cases; the screen against the CPU checker at
the warp edges and across a chunk boundary; the enlarged matrix's pivot failure against the NumPy restatement
(tests/lcb_ref.py); the untouched GP handle, the three front ends and the size limits."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

from cornell_moe_b200 import capi  # noqa: E402

import lcb_ref as R  # noqa: E402
from gpu_util import checker  # noqa: E402
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds  # noqa: E402

pytestmark = pytest.mark.gpu


def _gp(pr, kernel):
    return capi.GaussianProcess(kernel, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"])


def _ref(pr, kernel, cand, q):
    return R.reference_loop(checker(), kernel, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"],
                            cand, q)


@pytest.mark.parametrize("name,c", R.golden_cases(), ids=[n for n, _ in R.golden_cases()])
def test_selection_matches_the_golden_reference_run(name, c):
    """tests/golden/reference_lcb.npz: the unmodified reference routine on the compiled reference.  Same points (ties to
    the lowest candidate index), mu and sigma within 1e-10, or the same singular failure; every decision of the
    reference has a margin above 1e-8, so identical choices are not an accident of rounding."""
    pr = {k: c[k] for k in ("alpha", "lengths", "X", "y", "noise", "derivs")}
    gp = _gp(pr, int(c["kernel"]))
    cand, q = c["cand"], int(c["q"])
    if int(c["info"]) != 0:
        with pytest.raises(capi.SingularMatrixError) as e:
            gp.lower_confidence_bound(cand, q)
        assert e.value.info == int(c["info"]) and f"candidate {int(c['fail_cand'])}" in str(e.value)
        return
    assert np.all(c["margins"] > 1e-8), c["margins"]
    idx, mean, sd = gp.lower_confidence_bound(cand, q)
    np.testing.assert_array_equal(idx, c["index"])
    np.testing.assert_array_equal(cand[idx], c["points"])
    np.testing.assert_allclose(mean, c["mean"], rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(sd, c["sd"], rtol=1e-10)
    assert capi.lib().cmoe_gp_num_sampled(gp.h) == c["X"].shape[0]  # the reference left N + q - 1 points behind


def test_pivot_failure_of_the_enlarged_matrix_reports_its_leading_minor():
    pr, cand = R.pivot_failure_problem()
    with pytest.raises(R.LcbSingular) as r:
        R.bordered(checker(), 0, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"], cand, 2)
    gp = _gp(pr, 0)
    idx, _, _ = gp.lower_confidence_bound(cand, 1)  # the screen passes: only the value row is checked
    assert idx[0] == 0
    with pytest.raises(capi.SingularMatrixError) as e:
        gp.lower_confidence_bound(cand, 2)
    assert e.value.info == r.value.info == pr["X"].shape[0] * 3 + 2


@pytest.mark.parametrize("C", [1, 63, 64, 65])
def test_screen_matches_the_checker(C):
    pr = make_problem(70, 4, (1,), seed=10)
    cand = np.random.default_rng(11).uniform(size=(C, 4))
    ref = _ref(pr, 1, cand, 1)
    idx, mean, sd = _gp(pr, 1).lower_confidence_bound(cand, 1)
    assert idx[0] == ref["selected"][0]
    np.testing.assert_allclose(mean, ref["mean"], rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(sd, ref["sd"], rtol=1e-10)


def test_screen_does_not_depend_on_the_chunk():
    pr = make_problem(2000, 10, (), seed=12)
    gp = _gp(pr, 1)
    chunk = (1 << 31) // (8 * 2000)
    cand = np.random.default_rng(13).uniform(size=(chunk + 1, 10))
    _, mean, sd = gp.lower_confidence_bound(cand, 1)
    _, m1, s1 = gp.lower_confidence_bound(cand[:chunk], 1)
    _, m2, s2 = gp.lower_confidence_bound(cand[chunk:], 1)
    np.testing.assert_array_equal(mean, np.concatenate([m1, m2]))
    np.testing.assert_array_equal(sd, np.concatenate([s1, s2]))


def test_gp_handle_is_unchanged_and_a_plan_still_runs():
    pr = make_problem(40, 3, (), seed=14)
    gp = _gp(pr, 1)
    plan = capi.KGPlan(gp, 32, 0.0, EXAMPLE_INNER_GD, unit_bounds(3), pr["X"][:4], 2, 1)
    cands = np.random.default_rng(15).uniform(size=(2, 1, 3))
    plan.upload(cands)
    plan.run()
    plan.sync()
    kg0 = plan.download()[0].copy()
    before = gp.state()
    gp.lower_confidence_bound(np.random.default_rng(16).uniform(size=(300, 3)), 6)
    after = gp.state()
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a, b)
    assert capi.lib().cmoe_gp_num_sampled(gp.h) == 40
    plan.upload(cands)
    plan.run()
    plan.sync()
    np.testing.assert_array_equal(plan.download()[0], kg0)


def test_gpp_wrapper_and_capi_agree():
    import GPP as C_GP
    pr = make_problem(30, 2, (), seed=17)
    cand = np.random.default_rng(18).uniform(size=(200, 2))
    gpp = C_GP.GaussianProcess([pr["alpha"], list(pr["lengths"])], list(pr["X"].ravel()), list(pr["y"]),
                               list(pr["noise"]), [], 0, 2, 30)

    class Wrapper:
        _gaussian_process = gpp

    flat = list(cand.ravel())
    a = np.array(C_GP.lower_confidence_bound_optimization(gpp, flat, 200, 4)).reshape(4, 2)
    b = np.array(C_GP.lower_confidence_bound_optimization(Wrapper(), flat, 200, 4)).reshape(4, 2)
    idx = _gp(pr, 1).lower_confidence_bound(cand, 4)[0]
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(a, cand[idx])
    assert gpp.num_sampled == 30
    with pytest.raises(C_GP.BoundsException):
        C_GP.lower_confidence_bound_optimization(gpp, flat, 200, 0)


def test_bounds_just_past_each_limit():
    pr = make_problem(10, 2, (), seed=19)
    gp = _gp(pr, 0)
    cand = np.random.default_rng(20).uniform(size=(5, 2))
    with pytest.raises(capi.BoundsError, match="1024"):
        gp.lower_confidence_bound(cand, 1026)  # (q - 1)(1 + g) = 1025
    pr3 = make_problem(10, 2, (0, 1), seed=19)
    with pytest.raises(capi.BoundsError, match="1024"):
        _gp(pr3, 0).lower_confidence_bound(cand, 343)  # 342 * 3 = 1026
    same = np.tile(np.array([[0.3, 0.6]]), ((1 << 18) + 1, 1))  # every copy is satisfied: C' = 2^18 + 1
    with pytest.raises(capi.BoundsError, match="2\\^28"):
        gp.lower_confidence_bound(same, 1025)

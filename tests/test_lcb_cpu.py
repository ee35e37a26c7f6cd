"""CPU checks of the LCB batch selection (cmoe_lcb_select, GaussianProcess.lower_confidence_bound and
GPP.lower_confidence_bound_optimization): the argument checks that run before any device work, and the NumPy
restatement of the bordered update (tests/lcb_ref.py) against the refit loop of the reference routine on the CPU
checker.  No GPU needed."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

import lcb_ref as R  # noqa: E402
import oracle as orc  # noqa: E402
from synth import make_problem  # noqa: E402


def _select(gp, cand, C, q):
    sel = np.zeros(max(q, 1), dtype=np.int32)
    info = ctypes.c_int(0)
    rc = capi.lib().cmoe_lcb_select(gp, None if cand is None else cand.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                    int(C), int(q), sel.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), None, None, None,
                                    ctypes.byref(info))
    return rc


def test_sizes_and_null_arguments_are_rejected_before_device_work():
    cand = np.zeros((3, 2))
    assert _select(None, cand, 0, 1) == capi.ERR_BOUNDS
    assert _select(None, cand, 3, 0) == capi.ERR_BOUNDS
    assert _select(None, cand, 3, 2) == capi.ERR_INVALID_VALUE
    assert _select(None, None, 3, 2) == capi.ERR_INVALID_VALUE
    assert "NULL" in capi.lib().cmoe_last_error().decode()


def test_gpp_entry_is_exported():
    assert callable(C_GP.lower_confidence_bound_optimization)
    with pytest.raises(RuntimeError, match="GaussianProcess"):  # neither a GaussianProcess nor a wrapper of one
        C_GP.lower_confidence_bound_optimization(object(), [0.0], 1, 1)


def _backend():
    return orc.load_reference() if orc.have_reference() else orc.load_oracle()


CASES = [  # kernel, N, d, derivs, C, q, seed
    (0, 20, 2, (), 40, 4, 0),
    (1, 20, 2, (), 40, 5, 1),
    (1, 12, 3, (0, 2), 25, 3, 2),
    (0, 15, 2, (), 6, 6, 3),  # small satisfied set: points repeat
]


@pytest.mark.parametrize("kernel,N,d,derivs,C,q,seed", CASES)
def test_bordered_update_reproduces_the_refit_loop(kernel, N, d, derivs, C, q, seed):
    pr = make_problem(N, d, derivs, seed=seed, noise=1e-2)
    rng = np.random.default_rng(100 + seed)
    cand = rng.uniform(0.0, 1.0, size=(C, d))
    be = _backend()
    args = (be, kernel, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"], cand, q)
    ref = R.reference_loop(*args)
    brd = R.bordered(*args)
    np.testing.assert_array_equal(brd["selected"], ref["selected"])
    np.testing.assert_array_equal(brd["sat"], ref["sat"])
    np.testing.assert_allclose(brd["mean"], ref["mean"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(brd["sd"], ref["sd"], rtol=1e-10)
    for a, b in zip(brd["rounds"], ref["rounds"]):
        np.testing.assert_allclose(a, b, rtol=1e-10)


def test_zero_noise_fails_at_a_training_point_and_in_the_rounds():
    pr = make_problem(10, 2, (), seed=4, noise=0.0, alpha=1e-3)
    be = _backend()
    base = (be, 0, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"])
    cand = np.vstack([np.random.default_rng(5).uniform(size=(6, 2)), pr["X"][3:4]])
    for fn in (R.reference_loop, R.bordered):
        with pytest.raises(R.LcbSingular) as e:
            fn(*base, cand, 1)
        assert (e.value.info, e.value.cand) == (1, 6)
    cand = np.random.default_rng(6).uniform(size=(8, 2))
    for fn in (R.reference_loop, R.bordered):
        with pytest.raises(R.LcbSingular) as e:
            fn(*base, cand, 3)
        assert e.value.info == 1


@pytest.mark.parametrize("name,c", R.golden_cases(), ids=[n for n, _ in R.golden_cases()])
def test_bordered_update_reproduces_the_golden_reference_run(name, c):
    """Fed the checker's kernel blocks, the bordered update makes the reference's selections, with its screen and every
    round's sigma within 1e-10; the reference leaves its q - 1 fantasy points in the caller's GP."""
    args = (_backend(), int(c["kernel"]), float(c["alpha"]), c["lengths"], c["X"], c["y"], c["noise"], c["derivs"],
            c["cand"], int(c["q"]))
    if int(c["info"]) != 0:
        with pytest.raises(R.LcbSingular) as e:
            R.bordered(*args)
        assert (e.value.info, e.value.cand) == (int(c["info"]), int(c["fail_cand"]))
        return
    brd = R.bordered(*args)
    np.testing.assert_array_equal(c["cand"][brd["selected"]], c["points"])
    np.testing.assert_array_equal(brd["sat"], c["sat"])
    np.testing.assert_allclose(brd["mean"], c["mean"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(brd["sd"], c["sd"], rtol=1e-10)
    for a, b in zip(brd["rounds"], c["rounds"]):
        np.testing.assert_allclose(a, b, rtol=1e-10)
    assert int(c["num_sampled_after"]) == c["X"].shape[0] + int(c["q"]) - 1


def test_bordered_update_pivot_failure_counts_the_leading_minor():
    pr, cand = R.pivot_failure_problem()
    with pytest.raises(R.LcbSingular) as e:
        R.bordered(_backend(), 0, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"], cand, 2)
    assert (e.value.info, e.value.cand) == (8 * 3 + 2, None)

"""CPU checks of the hyper-parameter MAP fit (cmoe_hyperparameter_map, capi.hyperparameter_map,
GPP.hyperparameter_map_optimization) and of cmoe_grad_log_marginal_likelihood_list_exact: the argument and bound checks
that run before any device work, and the NumPy restatement of the objective and its analytic gradient against central
differences.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

import hyper_map_ref as M  # noqa: E402
import hyper_mcmc_ref as R  # noqa: E402

X = np.array([[0.1, 0.2], [0.7, 0.4]])  # two points in two dimensions: nh = 4
Y = np.array([0.3, 0.9])


def starts(num, nh=4):
    return np.zeros((num, nh))


def raw_map(kernel=1, prior=1, noisy=1, S=None, num=1, opts=None, X_=X, Y_=Y, out_none=False):
    lib = capi.lib()
    S = np.ascontiguousarray(starts(num) if S is None else S)
    pos, grads, vals = np.empty(S.shape), np.empty(S.shape), np.empty(len(S))
    it, ev, st = (np.empty(len(S), dtype=np.int32) for _ in range(3))
    info = capi.ctypes.c_int()
    Xc, Yc = np.ascontiguousarray(X_), np.ascontiguousarray(Y_)
    rc = lib.cmoe_hyperparameter_map(kernel, prior, noisy, capi._d(S), len(S), opts, capi._d(Xc), capi._d(Yc), None,
                                     0, Xc.shape[1], Xc.shape[0], 0, None if out_none else capi._d(pos),
                                     capi._d(vals), capi._d(grads), capi._i(it), capi._i(ev), capi._i(st),
                                     capi.ctypes.byref(info))
    return rc, lib.cmoe_last_error().decode()


def test_no_device_no_compute():
    if capi.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    with pytest.raises(capi.NoDeviceError):
        capi.hyperparameter_map(1, starts(2), X, Y)
    with pytest.raises(capi.NoDeviceError):
        capi.grad_log_marginal_likelihood_list_exact(1, np.ones((2, 4)), X, Y)
    with pytest.raises(C_GP.OptimalLearningException):
        C_GP.hyperparameter_map_optimization(list(X.ravel()), list(Y), 2, 2, [], 0, [0.0] * 4, 1, True, True)


def test_invalid_values():
    assert raw_map(prior=2) == (capi.ERR_INVALID_VALUE, raw_map(prior=2)[1])
    assert "prior" in raw_map(prior=2)[1]
    rc, msg = raw_map(noisy=2)
    assert rc == capi.ERR_INVALID_VALUE and "noisy" in msg
    rc, msg = raw_map(kernel=7)
    assert rc == capi.ERR_INVALID_VALUE and "kernel" in msg
    rc, msg = raw_map(out_none=True)
    assert rc == capi.ERR_INVALID_VALUE and "NULL" in msg
    rc, msg = raw_map(opts=capi.ctypes.byref(capi.MapOpts(-1.0, 0)))
    assert rc == capi.ERR_INVALID_VALUE and "gtol" in msg
    rc, msg = raw_map(opts=capi.ctypes.byref(capi.MapOpts(1e-5, -3)))
    assert rc == capi.ERR_INVALID_VALUE and "max_iterations" in msg


def test_bounds_before_device_work():
    with pytest.raises(capi.BoundsError, match="num_starts"):
        capi.hyperparameter_map(1, np.zeros((0, 4)), X, Y)
    with pytest.raises(capi.BoundsError, match="chunk"):  # a chunk holds 4096 sets of this size
        capi.hyperparameter_map(1, starts(4097), X, Y)
    with pytest.raises(capi.BoundsError, match="8192"):
        capi.hyperparameter_map(0, starts(1, 3), np.linspace(0.0, 1.0, 8193)[:, None], np.zeros(8193))
    with pytest.raises(capi.BoundsError, match="chunk"):  # n = 8192 with the gradient's buffers: one set per chunk
        capi.hyperparameter_map(0, starts(2, 3), np.linspace(0.0, 1.0, 8192)[:, None], np.zeros(8192))
    with pytest.raises(capi.BoundsError, match="dim"):  # nh <= 2 + 2 CMOE_MAX_DIM
        capi.hyperparameter_map(1, starts(1, 35), np.zeros((2, 33)), Y)
    with pytest.raises(capi.BoundsError, match="num_derivatives"):
        capi.hyperparameter_map(1, starts(1, 7), X, np.zeros(8), derivs=[0, 1, 0])
    with pytest.raises(capi.BoundsError, match="8192"):
        capi.grad_log_marginal_likelihood_list_exact(0, np.ones((1, 3)), np.linspace(0, 1, 8193)[:, None],
                                                     np.zeros(8193))
    with pytest.raises(C_GP.BoundsException, match="chunk"):
        C_GP.hyperparameter_map_optimization(list(X.ravel()), list(Y), 2, 2, [], 0, [0.0] * 4 * 4097, 4097, True,
                                             True)


# ---- the restatement -------------------------------------------------------------------------------------------------
DIM, G = 2, 1
NH = 2 + DIM + G
A_LIN = np.array([0.7, -0.3, 0.5, 0.2, -0.4])
B_LIN = np.array([1.3, 0.8, 0.6, 2.0, 1.1])


def toy_lml(h):
    """A smooth likelihood of a linear-scale set with a known gradient."""
    return float(A_LIN @ np.log(h) - 0.5 * np.sum((h - B_LIN) ** 2))


def toy_lml_grad(h):
    return A_LIN / h - (h - B_LIN)


@pytest.mark.parametrize("noisy,prior", [(True, True), (False, True), (True, False), (False, False)])
def test_restated_gradient_matches_central_differences(noisy, prior):
    theta = np.array([0.4, -0.5, 1.2, -1.7, -3.1])
    f = lambda t: M.nll(t, toy_lml, DIM, G, noisy, prior)  # noqa: E731
    want = M.central_diff(f, theta)
    got = M.nll_grad(theta, toy_lml_grad, DIM, G, noisy, prior)
    np.testing.assert_allclose(got, want, rtol=1e-7, atol=1e-8)
    if not noisy:
        assert np.all(got[1 + DIM:] == 0.0)


def test_prior_terms_against_central_differences():
    h = np.array([-0.8, 0.3, 2.5, -2.2, 0.05])
    lp = lambda t: R.default_prior_lnprob(t, 1 + G)  # noqa: E731
    np.testing.assert_allclose(M.default_prior_grad(h, DIM, G, True), M.central_diff(lp, h, 1e-7), rtol=1e-6)
    # the pdf term (not the log pdf) and the horseshoe term taken on theta itself
    assert M.default_prior_grad(h, DIM, G, True)[0] == pytest.approx(0.8 * np.exp(-0.32) / np.sqrt(2 * np.pi))


def test_box_tophat_and_pinning():
    assert M.nll(np.array([20.5, 0, 0, 0, 0]), toy_lml, DIM, G, True, False) == np.inf
    assert M.nll(np.array([0, 3.2, 0, -1, -1]), toy_lml, DIM, G, True, True) == np.inf  # the tophat wall
    assert np.isfinite(M.nll(np.array([0, 3.2, 0, -1, -1]), toy_lml, DIM, G, True, False))
    t = np.array([0.1, 0.2, 0.3, 5.0, 7.0])
    a = M.nll(t, toy_lml, DIM, G, False, True)
    t2 = t.copy()
    t2[1 + DIM:] = [-4.0, 2.0]
    assert a == M.nll(t2, toy_lml, DIM, G, False, True) and t[3] == 5.0  # pinned on a copy

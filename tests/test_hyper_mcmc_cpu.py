"""CPU checks of the hyper-parameter MCMC (cmoe_hyperparameter_mcmc, capi.hyperparameter_mcmc and
GPP.sample_hyperparameters_mcmc): the size and argument checks that run before any device work, device-less calls
failing with the library's own exceptions, and the NumPy restatement's own sanity.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

import hyper_mcmc_ref as R  # noqa: E402

X = np.array([[0.1, 0.2], [0.7, 0.4]])  # two points in two dimensions: nh = 4
Y = np.array([0.3, 0.9])


def p0(num_walkers, nh=4):
    return np.zeros((num_walkers, nh))


def test_no_device_no_compute():
    if capi.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    with pytest.raises(capi.NoDeviceError):
        capi.hyperparameter_mcmc(1, p0(8), X, Y, 1)
    with pytest.raises(C_GP.OptimalLearningException):
        C_GP.sample_hyperparameters_mcmc(list(X.ravel()), list(Y), 2, 2, [], 0, [0.0] * 32, 8, 1, False, True, 0)


def test_walker_count_and_steps_are_bounds_errors():
    with pytest.raises(capi.BoundsError, match="even"):
        capi.hyperparameter_mcmc(1, p0(9), X, Y, 1)
    with pytest.raises(capi.BoundsError, match="twice"):
        capi.hyperparameter_mcmc(1, p0(6), X, Y, 1)
    with pytest.raises(capi.BoundsError, match="num_steps"):
        capi.hyperparameter_mcmc(1, p0(8), X, Y, 0)
    with pytest.raises(C_GP.BoundsException, match="twice"):
        C_GP.sample_hyperparameters_mcmc(list(X.ravel()), list(Y), 2, 2, [], 0, [0.0] * 24, 6, 1, False, True, 0)


def test_size_contract_is_checked_before_device_work():
    Xbig = np.linspace(0.0, 1.0, 8193)[:, None]
    with pytest.raises(capi.BoundsError, match="8192"):  # n = 8193 rows
        capi.hyperparameter_mcmc(0, p0(6, 3), Xbig, np.zeros(8193), 1)
    X8k = np.linspace(0.0, 1.0, 8192)[:, None]
    with pytest.raises(capi.BoundsError, match="chunk"):  # 4 sets of n = 8192 per half: one chunk holds 3
        capi.hyperparameter_mcmc(0, p0(8, 3), X8k, np.zeros(8192), 1)
    with pytest.raises(capi.BoundsError, match="chunk"):  # more than 4096 sets per half
        capi.hyperparameter_mcmc(0, p0(8194), X, Y, 1)


def test_argument_checks():
    with pytest.raises(capi.InvalidValueError, match="not finite"):
        bad = p0(8)
        bad[3, 1] = np.nan
        capi.hyperparameter_mcmc(1, bad, X, Y, 1)
    with pytest.raises(capi.InvalidValueError, match="kernel"):
        capi.hyperparameter_mcmc(7, p0(8), X, Y, 1)
    tz, tp, tu = np.zeros((2, 8)), np.zeros((2, 8), np.int32), np.zeros((2, 8))
    tp[1, 5] = 4  # partners index the other half: [0, 4)
    with pytest.raises(capi.BoundsError, match="partner"):
        capi.hyperparameter_mcmc(1, p0(8), X, Y, 2, table=(tz, tp, tu))
    with pytest.raises(capi.BoundsError, match="num_steps \\* num_walkers"):
        capi.hyperparameter_mcmc(1, p0(8), X, Y, 3, table=(tz, tp, tu))


def test_prior_id_is_checked():
    lib = capi.lib()
    out, lnp, info = np.empty((8, 4)), np.empty(8), capi.ctypes.c_int()
    P, Xc, Yc = np.ascontiguousarray(p0(8)), np.ascontiguousarray(X), np.ascontiguousarray(Y)
    rc = lib.cmoe_hyperparameter_mcmc(1, 2, 1, capi._d(P), 8, 1, capi.ctypes.c_uint64(0), capi.ctypes.c_uint64(0),
                                      None, capi._d(Xc), capi._d(Yc), None, 0, 2, 2, 0, capi._d(out), capi._d(lnp),
                                      capi.ctypes.byref(info))
    assert rc == capi.ERR_INVALID_VALUE
    assert "prior" in lib.cmoe_last_error().decode()


# ---- the restatement -------------------------------------------------------------------------------------------------
def test_restatement_pins_noise_in_the_walkers_and_skips_the_box():
    calls = []

    def lml(H):
        calls.append(H.copy())
        return np.zeros(len(H))

    P = np.array([[0.0, 0.5, 0.5, -3.0], [25.0, 0.5, 0.5, -3.0], [0.0, 0.5, 5.0, -3.0]])
    out = R.log_prob(P, lml, dim=2, g=0, noisy=False, default_prior=True)
    assert P[0, 3] == R.LOG_NOISE_FREE and P[2, 3] == R.LOG_NOISE_FREE
    assert P[1, 3] == -3.0  # outside the box: returned before the pinning
    assert out[1] == -np.inf and out[2] == -np.inf  # the tophat over the lengths is [-2, 3]
    assert len(calls) == 1 and calls[0].shape == (1, 4)
    np.testing.assert_allclose(calls[0][0], np.exp([0.0, 0.5, 0.5, R.LOG_NOISE_FREE]))
    want = 1 / np.sqrt(2 * np.pi) + np.log(np.log(1 + 3.0 * (0.1 / R.LOG_NOISE_FREE) ** 2))
    assert out[0] == pytest.approx(want, rel=1e-15)


def test_restatement_rejects_what_emcee_rejects():
    with pytest.raises(ValueError):
        R.stretch_chain(np.zeros((7, 3)), 1, lambda P: np.zeros(len(P)), None)
    with pytest.raises(ValueError):
        R.stretch_chain(np.zeros((4, 3)), 1, lambda P: np.zeros(len(P)), None)

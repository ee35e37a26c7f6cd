"""CPU checks of the log marginal likelihood at a list of hyper-parameter sets (cmoe_log_marginal_likelihood_list and
GPP.evaluate_log_likelihood_at_hyperparameter_list): argument checks that run before any device work, and device-less
calls failing with the library's own exceptions.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

X = [0.1, 0.2, 0.7, 0.4]  # two points in two dimensions
Y = [0.3, 0.9]
LML = C_GP.LogLikelihoodTypes.log_marginal_likelihood


def _gpp_call(hyper_list, num_sets, mode=LML, status=None):
    return C_GP.evaluate_log_likelihood_at_hyperparameter_list(hyper_list, X, Y, 2, 2, mode, [1.0, [1.0, 1.0]],
                                                               [0.01], [], 0, num_sets, 4,
                                                               {} if status is None else status)


def test_no_device_no_compute():
    if capi.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    with pytest.raises(C_GP.OptimalLearningException):
        _gpp_call([1.0, 0.5, 0.5, 0.01, 2.0, 0.3, 0.3, 0.1], 2)
    with pytest.raises(capi.NoDeviceError):
        capi.log_marginal_likelihood_list(0, [[1.0, 0.5, 0.5, 0.01]], np.reshape(X, (2, 2)), Y)


def test_short_hyperparameter_list_is_a_bounds_error():
    # each set is 2 + dim + g = 4 numbers: 7 numbers do not make two sets
    with pytest.raises(C_GP.BoundsException):
        _gpp_call([1.0, 0.5, 0.5, 0.01, 2.0, 0.3, 0.3], 2)


def test_leave_one_out_mode_raises_the_reference_message():
    status = {}
    with pytest.raises(C_GP.OptimalLearningException,
                       match="ERROR: invalid objective mode choice. Setting all results to -DBL_MAX."):
        _gpp_call([1.0, 0.5, 0.5, 0.01], 1, mode=C_GP.LogLikelihoodTypes.leave_one_out_log_likelihood, status=status)
    assert status == {"evaluate_invalid_log_likelihood_at_hyperparameter_list": False}


def test_covariance_hyperparameters_and_multistart_count_are_checked():
    with pytest.raises(C_GP.BoundsException, match="alpha"):
        C_GP.evaluate_log_likelihood_at_hyperparameter_list([1.0, 0.5, 0.5, 0.01], X, Y, 2, 2, LML, [0.0, [1.0, 1.0]],
                                                           [0.01], [], 0, 1, 1, {})
    with pytest.raises(C_GP.BoundsException, match="length"):
        C_GP.evaluate_log_likelihood_at_hyperparameter_list([1.0, 0.5, 0.5, 0.01], X, Y, 2, 2, LML, [1.0, [1.0, -1.0]],
                                                           [0.01], [], 0, 1, 1, {})
    with pytest.raises(C_GP.BoundsException):
        _gpp_call([], 0)


def test_c_abi_size_and_set_checks_precede_device_work():
    Xa = np.reshape(X, (2, 2))
    with pytest.raises(capi.BoundsError):  # num_sets = 0
        capi.log_marginal_likelihood_list(0, np.zeros((0, 4)), Xa, Y)
    with pytest.raises(capi.BoundsError, match="hyperparameter set 1: Invalid hyperparameter \\(alpha\\)"):
        capi.log_marginal_likelihood_list(0, [[1.0, 0.5, 0.5, 0.01], [-1.0, 0.5, 0.5, 0.01]], Xa, Y)
    with pytest.raises(capi.BoundsError, match="hyperparameter set 2: Invalid hyperparameter \\(length\\)"):
        capi.log_marginal_likelihood_list(1, [[1.0, 0.5, 0.5, 0.01]] * 2 + [[1.0, 0.5, 0.0, 0.01]], Xa, Y)
    Xbig = np.linspace(0.0, 1.0, 8193)[:, None]
    with pytest.raises(capi.BoundsError, match="8192"):  # n = 8193 rows
        capi.log_marginal_likelihood_list(0, [[1.0, 0.5, 0.01]], Xbig, np.zeros(8193))

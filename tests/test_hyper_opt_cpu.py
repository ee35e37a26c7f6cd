"""CPU checks of the hyper-parameter gradient list and optimisers (cmoe_grad_log_marginal_likelihood_list,
cmoe_hyperparameter_gradient_descent, GPP.multistart_hyperparameter_optimization and
GPP.restarted_hyperparameter_optimization): argument checks that run before any device work, and device-less calls
failing with the library's own exceptions.  No GPU needed."""
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
XA = np.reshape(X, (2, 2))
DOMAIN = [-1.0, 1.0, -1.0, 0.5, -1.0, 0.5, -4.0, -1.0]  # log10 box of (alpha, l1, l2, noise)
GD = (4, 10, 1, 0, 0.5, 0.01, 0.2, 1e-7)


class Params:
    def __init__(self, optimizer=C_GP.OptimizerTypes.gradient_descent,
                 objective=C_GP.LogLikelihoodTypes.log_marginal_likelihood, gd=GD):
        self.domain_type = C_GP.DomainTypes.tensor_product
        self.optimizer_type = optimizer
        self.objective_type = objective
        self.num_random_samples = gd[0]
        self.optimizer_parameters = C_GP.GradientDescentParameters(*gd)


def _multistart(params, hypers=(1.0, [1.0, 1.0]), domain=DOMAIN, rnd=None, status=None):
    return C_GP.multistart_hyperparameter_optimization(params, domain, X, Y, 2, 2, [hypers[0], list(hypers[1])],
                                                       [0.01], [], 0, 4, rnd or C_GP.RandomnessSourceContainer(1),
                                                       {} if status is None else status)


def _restarted(params, hypers=(1.0, [1.0, 1.0]), domain=DOMAIN):
    return C_GP.restarted_hyperparameter_optimization(params, domain, X, Y, 2, 2, [hypers[0], list(hypers[1])],
                                                      [0.01], [], 0, {})


def test_no_device_no_compute():
    if capi.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    with pytest.raises(C_GP.OptimalLearningException):
        _multistart(Params())
    with pytest.raises(C_GP.OptimalLearningException):
        _multistart(Params(optimizer=C_GP.OptimizerTypes.null))
    with pytest.raises(C_GP.OptimalLearningException):
        _restarted(Params())
    with pytest.raises(capi.NoDeviceError):
        capi.grad_log_marginal_likelihood_list(0, [[1.0, 0.5, 0.5, 0.01]], XA, Y)
    with pytest.raises(capi.NoDeviceError):
        capi.hyperparameter_gradient_descent(0, GD, [[0.1, 10.0], [0.1, 3.0], [0.1, 3.0], [1e-4, 0.1]],
                                             [[1.0, 0.5, 0.5, 0.01]], XA, Y)


def test_restarted_without_restarts_returns_zeros_without_device_work():
    assert _restarted(Params(gd=GD[:2] + (0,) + GD[3:])) == [0.0] * 4


def test_calls_matching_no_signature_raise_the_library_exception():
    for name in ("multistart_hyperparameter_optimization", "restarted_hyperparameter_optimization"):
        with pytest.raises(C_GP.OptimalLearningException, match="match no signature"):
            getattr(C_GP, name)(Params(), DOMAIN)


def test_covariance_checks_short_lists_and_optimizer_choice_precede_device_work():
    with pytest.raises(C_GP.BoundsException, match="alpha"):
        _multistart(Params(), hypers=(0.0, [1.0, 1.0]))
    with pytest.raises(C_GP.BoundsException, match="length"):
        _restarted(Params(), hypers=(1.0, [1.0, -1.0]))
    with pytest.raises(C_GP.BoundsException):  # the domain needs 2 * (2 + dim + g) numbers
        _multistart(Params(), domain=DOMAIN[:-1])
    with pytest.raises(C_GP.BoundsException, match="num_multistarts"):
        _multistart(Params(gd=(0,) + GD[1:]))
    with pytest.raises(C_GP.OptimalLearningException,
                       match="ERROR: invalid optimizer choice. Setting all hyperparameters to 1.0."):
        _multistart(Params(optimizer=C_GP.OptimizerTypes.newton))
    with pytest.raises(C_GP.OptimalLearningException,
                       match="ERROR: invalid objective type choice. Setting all hyperparameters to 1.0."):
        _multistart(Params(objective=C_GP.LogLikelihoodTypes.leave_one_out_log_likelihood))


def test_c_abi_checks_precede_device_work():
    with pytest.raises(capi.BoundsError):  # num_sets = 0
        capi.grad_log_marginal_likelihood_list(0, np.zeros((0, 4)), XA, Y)
    with pytest.raises(capi.BoundsError, match="hyperparameter set 1: Invalid hyperparameter \\(alpha\\)"):
        capi.grad_log_marginal_likelihood_list(0, [[1.0, 0.5, 0.5, 0.01], [-1.0, 0.5, 0.5, 0.01]], XA, Y)
    Xbig = np.linspace(0.0, 1.0, 8193)[:, None]
    with pytest.raises(capi.BoundsError, match="8192"):
        capi.grad_log_marginal_likelihood_list(0, [[1.0, 0.5, 0.01]], Xbig, np.zeros(8193))
    bounds = [[0.1, 10.0], [0.1, 3.0], [0.1, 3.0], [1e-4, 0.1]]
    with pytest.raises(capi.BoundsError):  # no starts
        capi.hyperparameter_gradient_descent(0, GD, bounds, np.zeros((0, 4)), XA, Y)
    with pytest.raises(capi.BoundsError, match="EMPTY"):
        capi.hyperparameter_gradient_descent(0, GD, [[10.0, 0.1]] + bounds[1:], [[1.0, 0.5, 0.5, 0.01]], XA, Y)

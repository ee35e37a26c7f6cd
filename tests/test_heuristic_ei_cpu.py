"""CPU checks of heuristic batch EI (cmoe_heuristic_ei, GPP.heuristic_expected_improvement_optimization, DESIGN.md K20):
the argument checks that run before any device work, the estimation-policy classes with the reference's positional
constructors, and the catch-all overload.  No GPU needed."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402


def _call(policy, q=2, num_starts=4, gp=None, gd=None, bounds=True, starts=True, points=True):
    dim = 2
    db = np.tile([0.0, 1.0], dim)
    st = np.zeros((max(q, 1), max(num_starts, 1), dim))
    pts = np.zeros((max(q, 1), dim))
    info = ctypes.c_int(0)
    return capi.lib().cmoe_heuristic_ei(gp, None if policy is None else ctypes.byref(policy),
                                        None if gd is None else ctypes.byref(gd),
                                        capi._d(db) if bounds else None, capi._d(st) if starts else None,
                                        int(num_starts), int(q), ctypes.c_double(0.0),
                                        capi._d(pts) if points else None, None, None, None, ctypes.byref(info))


def _policy(kind=capi.CONSTANT_LIAR, value=0.0, noise=0.0):
    return capi.EstimationPolicy(kind, value, noise)


def test_sizes_are_rejected_before_device_work():
    assert _call(_policy(), q=0) == capi.ERR_BOUNDS
    assert _call(_policy(), num_starts=0) == capi.ERR_BOUNDS
    gd = capi.GDParams.from_seq([4, (1 << 20) + 1, 1, 0, 0.7, 1.0, 1.0, 1e-6])
    assert _call(_policy(), gd=gd) == capi.ERR_BOUNDS


@pytest.mark.parametrize("policy", [
    None,
    capi.EstimationPolicy(2, 0.0, 0.0),
    capi.EstimationPolicy(-1, 0.0, 0.0),
    capi.EstimationPolicy(capi.CONSTANT_LIAR, math.inf, 0.0),
    capi.EstimationPolicy(capi.KRIGING_BELIEVER, math.nan, 0.0),
    capi.EstimationPolicy(capi.CONSTANT_LIAR, 0.0, -1e-12),
    capi.EstimationPolicy(capi.KRIGING_BELIEVER, 1.0, math.nan),
], ids=["null", "unknown-2", "unknown-neg", "inf-lie", "nan-coef", "negative-noise", "nan-noise"])
def test_bad_policies_are_invalid_values(policy):
    assert _call(policy) == capi.ERR_INVALID_VALUE


def test_null_arguments_are_invalid_values():
    assert _call(_policy()) == capi.ERR_INVALID_VALUE  # gp NULL
    assert "NULL" in capi.lib().cmoe_last_error().decode()
    assert _call(_policy(), bounds=False) == capi.ERR_INVALID_VALUE
    assert _call(_policy(), starts=False) == capi.ERR_INVALID_VALUE
    assert _call(_policy(), points=False) == capi.ERR_INVALID_VALUE


def test_policy_classes_take_the_reference_positional_arguments():
    cl = C_GP.ConstantLiarEstimationPolicy(-0.5, 0.01)
    kb = C_GP.KrigingBelieverEstimationPolicy(1.0, 0.0)
    assert isinstance(cl, C_GP.ObjectiveEstimationPolicyInterface)
    assert isinstance(kb, C_GP.ObjectiveEstimationPolicyInterface)
    C_GP.ConstantLiarEstimationPolicy(lie_value=0.0, lie_noise_variance=0.0)
    C_GP.KrigingBelieverEstimationPolicy(std_deviation_coef=0.0, kriging_noise_variance=0.0)
    with pytest.raises(TypeError):
        C_GP.ConstantLiarEstimationPolicy(0.0)


def test_the_catch_all_overload_raises_the_library_exception():
    with pytest.raises(C_GP.OptimalLearningException, match="no signature"):
        C_GP.heuristic_expected_improvement_optimization(1, 2, x=3)
    with pytest.raises(C_GP.OptimalLearningException, match="no signature"):
        C_GP.heuristic_expected_improvement_optimization()

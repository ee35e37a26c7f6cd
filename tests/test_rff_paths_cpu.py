"""CPU checks of the kernel-matched random features and the sample-function evaluator (cmoe_rff_opts,
cmoe_gp_sample_rff_optima_ex, cmoe_gp_sample_rff_functions, cmoe_rff_evaluate, cmoe_rff_chi2_draws): the restated chi^2_5
mixture reproduces the Matern-5/2 correlation and rejects SquareExponential frequencies, and the new entries refuse bad
arguments before any device work.  No GPU needed."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

import rff_paths_ref as RP  # noqa: E402

LENGTHS = [np.array([0.3, 0.3, 0.3]), np.array([0.2, 0.7, 1.5]), np.array([0.05, 2.0])]


def _matern_W(lengths, n, seed=3):
    rng = np.random.default_rng(seed)
    F = 2000
    om = rng.normal(size=(n // F, F, len(lengths)))
    g = np.stack([RP.chi2_draws(seed, k, F) for k in range(n // F)])
    return RP.matern_frequencies(om, lengths, g).reshape(-1, len(lengths))


def test_restated_chi2_stream_is_chi2_with_5_degrees_of_freedom():
    g = np.concatenate([RP.chi2_draws(7, k, 5000) for k in range(40)])
    n = g.size
    assert np.all(g > 0.0)
    assert abs(g.mean() - 5.0) < 5.0 * np.sqrt(10.0 / n)  # var chi^2_5 = 10
    assert abs(g.var() - 10.0) < 5.0 * np.sqrt(440.0 / n)  # var of s^2: (mu_4 - sigma^4) / n, mu_4 = 12 k (k + 4)
    # different draws and features give different numbers; word 3 = 3 is not the uniforms' stream (word 3 = 2)
    assert len(np.unique(g)) == n


@pytest.mark.parametrize("li", range(len(LENGTHS)), ids=["iso3", "aniso3", "aniso2"])
def test_mixture_reproduces_the_matern52_correlation(li):
    lengths = LENGTHS[li]
    W = _matern_W(lengths, 400000)
    deltas = RP.offsets(lengths)
    assert len(deltas) >= 6
    z = RP.correlation_z(W, deltas, lambda dl: RP.matern52_corr(dl, lengths))
    assert np.all(np.abs(z) < 5.0), z


@pytest.mark.parametrize("li", range(len(LENGTHS)), ids=["iso3", "aniso3", "aniso2"])
def test_the_same_check_rejects_squared_exponential_frequencies(li):
    lengths = LENGTHS[li]
    W = np.random.default_rng(4).normal(size=(400000, len(lengths))) / lengths
    deltas = RP.offsets(lengths)
    z_se = RP.correlation_z(W, deltas, lambda dl: RP.se_corr(dl, lengths))
    assert np.all(np.abs(z_se) < 5.0), z_se  # they are SE frequencies ...
    z = RP.correlation_z(W, deltas, lambda dl: RP.matern52_corr(dl, lengths))
    assert np.max(np.abs(z)) > 20.0, z  # ... and the Matern check tells them apart


def _dp(a):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _functions(gp, F, P, opts=None, outs=True):
    buf = np.zeros(max(F * P * 4, 1))
    info = ctypes.c_int(0)
    return capi.lib().cmoe_gp_sample_rff_functions(gp, int(F), int(P), ctypes.c_uint64(0), ctypes.c_uint64(0), None,
                                                  opts, _dp(buf) if outs else None, _dp(buf), _dp(buf),
                                                  ctypes.byref(info))


def _optima_ex(gp, F, P, G, opts=None):
    b = np.array([0.0, 1.0, 0.0, 1.0])
    g = np.zeros((max(G, 1), 2))
    out = np.zeros(max(P, 1) * 2)
    info = ctypes.c_int(0)
    return capi.lib().cmoe_gp_sample_rff_optima_ex(gp, int(F), int(P), _dp(b), _dp(g), int(G), ctypes.c_uint64(0),
                                                  ctypes.c_uint64(0), None, opts, _dp(out), _dp(out), None, None, None,
                                                  ctypes.byref(info))


def test_sample_entries_reject_sizes_and_a_null_gp_before_the_handle_is_read():
    opts = ctypes.byref(capi.RffOpts(capi.RFF_SPECTRAL_KERNEL, None))
    assert _functions(None, 0, 2) == capi.ERR_BOUNDS
    assert _functions(None, 10, 0) == capi.ERR_BOUNDS
    assert _functions(None, 10, 2, opts) == capi.ERR_INVALID_VALUE
    assert "gp is NULL" in capi.lib().cmoe_last_error().decode()
    assert _optima_ex(None, 0, 2, 3, opts) == capi.ERR_BOUNDS
    assert _optima_ex(None, 10, 2, 0, opts) == capi.ERR_BOUNDS
    assert _optima_ex(None, 10, 2, 3, opts) == capi.ERR_INVALID_VALUE


def _evaluate(d=2, F=3, P=2, X=4, per_function=0, values=True, grads=True, bad=None, c=0.5, device=0):
    om, b, th = np.full((P, F, max(d, 1)), 0.3), np.full((P, F), 0.1), np.full((P, F), 1.0)
    pts = np.full(((P if per_function else 1), X, max(d, 1)), 0.2)
    if bad is not None:
        {"omega": om, "b": b, "theta": th, "points": pts}[bad].flat[-1] = np.nan
    v = np.zeros(max(P * X, 1))
    g = np.zeros(max(P * X * max(d, 1), 1))
    info = ctypes.c_int(0)
    return capi.lib().cmoe_rff_evaluate(int(d), int(F), int(P), _dp(om), _dp(b), _dp(th), ctypes.c_double(c), _dp(pts),
                                        int(X), int(per_function), _dp(v) if values else None,
                                        _dp(g) if grads else None, int(device), ctypes.byref(info))


@pytest.mark.parametrize("kw,code", [
    (dict(d=0), capi.ERR_BOUNDS), (dict(d=33), capi.ERR_BOUNDS), (dict(F=0), capi.ERR_BOUNDS),
    (dict(P=0), capi.ERR_BOUNDS), (dict(X=0), capi.ERR_BOUNDS),
    (dict(values=False, grads=False), capi.ERR_INVALID_VALUE),
    (dict(bad="omega"), capi.ERR_INVALID_VALUE), (dict(bad="b"), capi.ERR_INVALID_VALUE),
    (dict(bad="theta"), capi.ERR_INVALID_VALUE), (dict(bad="points"), capi.ERR_INVALID_VALUE),
    (dict(bad="points", per_function=1), capi.ERR_INVALID_VALUE), (dict(c=np.inf), capi.ERR_INVALID_VALUE),
])
def test_evaluator_rejects_bad_arguments_before_any_device_work(kw, code):
    """These refusals come before the device is touched, so they are the same with or without one."""
    assert _evaluate(**kw) == code


def test_evaluator_size_limit_is_checked_before_the_inputs_are_read():
    # one function's features F (d + 2) plus one point's d + 1 + d doubles (shared points, both outputs) within 2^28
    d = 1
    F = ((1 << 28) - 3) // (d + 2) + 1
    tiny = np.zeros(4)
    info = ctypes.c_int(0)
    rc = capi.lib().cmoe_rff_evaluate(d, F, 1, _dp(tiny), _dp(tiny), _dp(tiny), ctypes.c_double(1.0), _dp(tiny), 1, 0,
                                      _dp(tiny), _dp(tiny), 0, ctypes.byref(info))
    assert rc == capi.ERR_BOUNDS


def test_chi2_draws_reject_sizes():
    out = np.zeros(4)
    lib = capi.lib()
    assert lib.cmoe_rff_chi2_draws(ctypes.c_uint64(0), ctypes.c_uint64(0), 0, 2, _dp(out), 0) == capi.ERR_BOUNDS
    assert lib.cmoe_rff_chi2_draws(ctypes.c_uint64(0), ctypes.c_uint64(0), 2, 0, _dp(out), 0) == capi.ERR_BOUNDS
    assert lib.cmoe_rff_chi2_draws(ctypes.c_uint64(0), ctypes.c_uint64(0), 65536, 1, _dp(out), 0) == capi.ERR_BOUNDS
    assert lib.cmoe_rff_chi2_draws(ctypes.c_uint64(0), ctypes.c_uint64(0), 1, 1, None, 0) == capi.ERR_INVALID_VALUE


class _Handle:  # what GaussianProcess.sample_rff_* read before they call the library
    dim, n, h, device, alpha = 2, 10, None, 0, 1.0


def test_capi_checks_the_chi2_table_size_before_the_call():
    P, F = 2, 30
    tab = {"omega": np.zeros((P, F, 2)), "b": np.zeros((P, F)), "z": np.zeros((P, F)), "eps": np.zeros((P, 10)),
           "chi2": np.ones((P, F - 1))}
    with pytest.raises(capi.BoundsError, match="chi2"):
        capi.GaussianProcess.sample_rff_optima(_Handle(), F, P, [0.0, 1.0, 0.0, 1.0], np.zeros((1, 2)), table=tab,
                                               spectral=capi.RFF_SPECTRAL_KERNEL)
    with pytest.raises(capi.BoundsError, match="chi2"):
        capi.GaussianProcess.sample_rff_functions(_Handle(), F, P, table=tab, spectral=capi.RFF_SPECTRAL_KERNEL)


def test_capi_opts_struct_matches_the_header():
    assert [f for f, _ in capi.RffOpts._fields_] == ["spectral", "chi2"]
    assert ctypes.sizeof(capi.RffOpts) == 2 * ctypes.sizeof(ctypes.c_void_p)
    assert (capi.RFF_SPECTRAL_REFERENCE, capi.RFF_SPECTRAL_KERNEL) == (0, 1)


def test_gpp_names_are_exported():
    assert callable(C_GP.sample_gp_with_random_features)
    assert callable(C_GP.sample_from_global_optima_kernel_matched)
    with pytest.raises(RuntimeError, match="GaussianProcess"):
        C_GP.sample_gp_with_random_features(object(), 10)
    with pytest.raises(RuntimeError, match="GaussianProcess"):
        C_GP.sample_from_global_optima_kernel_matched(object(), 10, [0.0, 1.0], [0.5], 1, 1)

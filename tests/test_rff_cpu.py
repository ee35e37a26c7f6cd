"""CPU checks of the random-feature sampler (cmoe_gp_sample_rff_optima, GaussianProcess.sample_rff_optima and
GPP.sample_from_global_optima): the NumPy restatement (tests/rff_ref.py) against the reference's golden run, the
pathwise branch's covariance as an identity, and the argument checks that run before any device work.  No GPU needed."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

import GPP as C_GP  # noqa: E402
from cornell_moe_b200 import capi  # noqa: E402

import rff_ref as R  # noqa: E402

CASES = R.golden_cases()
IDS = [n for n, _ in CASES]


def _phi(c, omega=None, b=None):
    return R.design(c["X"], c["Y"], c["noise"], c["derivs"], float(c["alpha"]), c["lengths"],
                    c["omega"] if omega is None else omega, c["b"] if b is None else b)


def test_golden_covers_both_branches_and_the_edges():
    sizes = {n: (c["X"].shape[0] * (1 + len(c["derivs"])), int(c["F"])) for n, c in CASES}
    assert {m - f for m, f in sizes.values()} >= {-1, 0, 1}
    assert any(m < f for m, f in sizes.values()) and any(m >= f for m, f in sizes.values())
    assert {c["X"].shape[1] for _, c in CASES} == {2, 6}
    assert any(len(c["derivs"]) > 0 and len(set(c["noise"])) > 1 for _, c in CASES)
    assert any(np.all(c["noise"] == 1e-8) for _, c in CASES)


@pytest.mark.parametrize("name,c", CASES, ids=IDS)
def test_restatement_reproduces_the_golden_mean(name, c):
    Phi, yp, W, _ = _phi(c)
    F, M = Phi.shape
    m = R.theta(Phi, yp, np.zeros(F), np.zeros(M))
    np.testing.assert_array_equal(W, c["W"])
    # noise 1e-8 puts entries of size 1e4 into Phi: B (or A) has a condition number near 1e8 and m loses that much
    tol = 1e-5 if c["noise"][0] < 1e-6 else 1e-10
    np.testing.assert_allclose(m, c["m"], rtol=tol, atol=tol * np.abs(c["m"]).max())


@pytest.mark.parametrize("name,c", [x for x in CASES if x[1]["X"].shape[0] * (1 + len(x[1]["derivs"])) >= int(x[1]["F"])],
                         ids=[n for n, c in CASES if c["X"].shape[0] * (1 + len(c["derivs"])) >= int(c["F"])])
def test_restatement_replays_the_golden_draw_on_the_cholesky_branch(name, c):
    Phi, yp, _, _ = _phi(c)
    th = R.theta(Phi, yp, c["z"])
    tol = 1e-5 if c["noise"][0] < 1e-6 else 1e-10
    np.testing.assert_allclose(th, c["theta"], rtol=tol, atol=tol * np.abs(c["theta"]).max())


@pytest.mark.parametrize("F,M", [(40, 10), (21, 20), (300, 30)])
def test_pathwise_draw_has_the_posterior_covariance(F, M):
    rng = np.random.default_rng(F + M)
    Phi = rng.normal(size=(F, M)) * rng.uniform(0.1, 3.0, size=M)
    np.testing.assert_allclose(R.pathwise_cov(Phi), R.posterior_cov(Phi), rtol=0, atol=1e-12)


def _call(gp, F, P, bounds, grid, G, points=True, table=None):
    pts = np.zeros((max(P, 1), 2))
    vals = np.zeros(max(P, 1))
    info = ctypes.c_int(0)
    dp = lambda a: None if a is None else a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))  # noqa: E731
    return capi.lib().cmoe_gp_sample_rff_optima(gp, int(F), int(P), dp(bounds), dp(grid), int(G), ctypes.c_uint64(0),
                                               ctypes.c_uint64(0), table, dp(pts) if points else None, dp(vals), None,
                                               None, None, ctypes.byref(info))


def test_sizes_and_null_gp_are_rejected_before_the_handle_is_read():
    """Only these checks are reachable without a device: the others need M, d and the noise from a GP handle, which
    cannot be made without one; they run in tests/test_gpu_rff.py."""
    b = np.array([0.0, 1.0, 0.0, 1.0])
    g = np.zeros((3, 2))
    assert _call(None, 0, 2, b, g, 3) == capi.ERR_BOUNDS
    assert _call(None, 10, 0, b, g, 3) == capi.ERR_BOUNDS
    assert _call(None, 10, 2, b, g, 0) == capi.ERR_BOUNDS
    assert _call(None, 10, 2, b, g, 3) == capi.ERR_INVALID_VALUE
    assert "NULL" in capi.lib().cmoe_last_error().decode()


class _Handle:  # what GaussianProcess.sample_rff_optima reads before it calls the library
    dim, n, h = 2, 10, None


@pytest.mark.parametrize("F,key,bad", [(30, "omega", (1, 30, 2)), (30, "b", (2, 29)), (30, "z", (1,)),
                                        (30, "eps", (2, 9)), (30, "eps", None)])
def test_capi_checks_table_sizes_and_bounds_before_the_call(F, key, bad):
    P = 2
    tab = {"omega": np.zeros((P, F, 2)), "b": np.zeros((P, F)), "z": np.zeros((P, F)), "eps": np.zeros((P, 10))}
    tab[key] = None if bad is None else np.zeros(bad)
    with pytest.raises(capi.BoundsError, match=key):
        capi.GaussianProcess.sample_rff_optima(_Handle(), F, P, [0.0, 1.0, 0.0, 1.0], np.zeros((1, 2)), table=tab)
    with pytest.raises(capi.BoundsError, match="domain_bounds"):
        capi.GaussianProcess.sample_rff_optima(_Handle(), F, P, [0.0, 1.0], np.zeros((1, 2)))


def test_gpp_entry_is_exported():
    assert callable(C_GP.sample_from_global_optima)
    with pytest.raises(RuntimeError, match="GaussianProcess"):  # neither a GaussianProcess nor a wrapper of one
        C_GP.sample_from_global_optima(object(), 10, [0.0, 1.0], [0.5], 1, 1)


def test_capi_table_struct_matches_the_header():
    assert [f for f, _ in capi.RffTable._fields_] == ["omega", "b", "z", "eps"]
    assert ctypes.sizeof(capi.RffTable) == 4 * ctypes.sizeof(ctypes.c_void_p)


def test_no_device_is_refused():
    """Without a device no GP handle can be made, so the sampler is unreachable: the refusal comes from the handle."""
    if capi.device_count() > 0:
        pytest.skip("a device is visible")
    with pytest.raises(capi.NoDeviceError):
        capi.GaussianProcess(0, 1.0, [0.3, 0.3], np.zeros((2, 2)) + [[0.1, 0.2], [0.5, 0.6]], [0.0, 1.0], [1e-2])

"""GPU tests of the kernel-matched random features and the sample-function evaluator (cmoe_gp_sample_rff_optima_ex,
cmoe_gp_sample_rff_functions, cmoe_rff_evaluate, cmoe_rff_chi2_draws; DESIGN.md K14 addendum): the reference mode is
cmoe_gp_sample_rff_optima bit for bit; the matched mode is the reference mode on a SquareExponential handle and a per-row
sqrt(5 / g) rescaling of it on a Matern one; table replay against the NumPy restatement; the frequencies' correlation;
the evaluator against NumPy, finite differences and itself under changes of the batch and the chunking; the GPP
names."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

from cornell_moe_b200 import capi  # noqa: E402

import rff_paths_ref as RP  # noqa: E402
import rff_ref as R  # noqa: E402
from synth import make_problem  # noqa: E402

pytestmark = pytest.mark.gpu

REF, KER = capi.RFF_SPECTRAL_REFERENCE, capi.RFF_SPECTRAL_KERNEL
SE, MATERN = capi.SQUARE_EXPONENTIAL, capi.MATERN_NU_2P5


def _gp(kernel, n=30, d=3, derivs=(), seed=11):
    pr = make_problem(n, d, derivs, seed=seed, noise=1e-2, length=0.4)
    return pr, capi.GaussianProcess(kernel, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"])


def _dp(a):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _old_entry(gp, F, P, bounds, grid, seed, first, table=None):
    """cmoe_gp_sample_rff_optima itself (capi goes through the _ex entry)."""
    d = gp.dim
    keep = []
    tab = None
    if table is not None:
        tab = capi.RffTable()
        for k in ("omega", "b", "z", "eps"):
            a = None if table.get(k) is None else np.ascontiguousarray(table[k], dtype=np.float64).ravel()
            keep.append(a)
            setattr(tab, k, _dp(a))
    pts, vals = np.empty((P, d)), np.empty(P)
    om, b, th = np.empty((P, F, d)), np.empty((P, F)), np.empty((P, F))
    info = ctypes.c_int(0)
    rc = capi.lib().cmoe_gp_sample_rff_optima(gp.h, F, P, _dp(np.ascontiguousarray(bounds, dtype=np.float64).ravel()),
                                              _dp(np.ascontiguousarray(grid)), grid.shape[0], ctypes.c_uint64(seed),
                                              ctypes.c_uint64(first), None if tab is None else ctypes.byref(tab),
                                              _dp(pts), _dp(vals), _dp(om), _dp(b), _dp(th), ctypes.byref(info))
    capi._check(rc, info.value)
    return pts, vals, {"omega": om, "b": b, "theta": th}


def _ex_entry(gp, F, P, bounds, grid, seed, first, spectral):
    """cmoe_gp_sample_rff_optima_ex with a non-NULL opts."""
    d = gp.dim
    opts = capi.RffOpts(int(spectral), None)
    pts, vals = np.empty((P, d)), np.empty(P)
    om, b, th = np.empty((P, F, d)), np.empty((P, F)), np.empty((P, F))
    info = ctypes.c_int(0)
    rc = capi.lib().cmoe_gp_sample_rff_optima_ex(gp.h, F, P, _dp(np.ascontiguousarray(bounds, dtype=np.float64).ravel()),
                                                 _dp(np.ascontiguousarray(grid)), grid.shape[0], ctypes.c_uint64(seed),
                                                 ctypes.c_uint64(first), None, ctypes.byref(opts), _dp(pts), _dp(vals),
                                                 _dp(om), _dp(b), _dp(th), ctypes.byref(info))
    capi._check(rc, info.value)
    return pts, vals, {"omega": om, "b": b, "theta": th}


def _same(a, b):
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    for k in ("omega", "b", "theta"):
        np.testing.assert_array_equal(a[2][k], b[2][k])


def _table(gp, F, P, seed, first, out_b, chi2=None):
    M, d = gp.n, gp.dim
    nrm = capi.philox_normals(seed, first, P, F * d + F + M)
    t = {"omega": nrm[:, :F * d], "b": out_b, "z": nrm[:, F * d:F * d + F], "eps": nrm[:, F * d + F:]}
    if chi2 is not None:
        t["chi2"] = chi2
    return t


BRANCHES = [(30, 80), (30, 20)]  # (n, F): M < F (Woodbury), then M >= F (Cholesky)


@pytest.mark.parametrize("kernel", [SE, MATERN], ids=["se", "matern"])
@pytest.mark.parametrize("n,F", BRANCHES, ids=["woodbury", "cholesky"])
def test_reference_mode_and_null_opts_are_the_existing_entry(kernel, n, F):
    pr, gp = _gp(kernel, n=n)
    d, P, seed = 3, 5, 77
    grid = np.random.default_rng(4).uniform(size=(100, d))
    bounds = np.array([[0.0, 1.0]] * d)
    old = _old_entry(gp, F, P, bounds, grid, seed, 9)
    _same(gp.sample_rff_optima(F, P, bounds, grid, seed=seed, first_draw=9, return_functions=True), old)  # NULL opts
    _same(_ex_entry(gp, F, P, bounds, grid, seed, 9, REF), old)
    tab = _table(gp, F, P, seed, 9, old[2]["b"])
    old_t = _old_entry(gp, F, P, bounds, grid, 0, 0, tab)
    _same(old_t, old)  # table mode replays Philox mode
    _same(gp.sample_rff_optima(F, P, bounds, grid, table=tab, return_functions=True), old_t)
    tab_c = dict(tab, chi2=np.full((P, F), 3.0))  # chi2 is not read in the reference mode
    _same(gp.sample_rff_optima(F, P, bounds, grid, table=tab_c, return_functions=True, spectral=REF), old_t)


@pytest.mark.parametrize("n,F", BRANCHES, ids=["woodbury", "cholesky"])
def test_kernel_mode_on_a_squared_exponential_handle_is_the_reference_mode(n, F):
    pr, gp = _gp(SE, n=n)
    d, P = 3, 4
    grid = np.random.default_rng(5).uniform(size=(80, d))
    bounds = np.array([[0.0, 1.0]] * d)
    ref = gp.sample_rff_optima(F, P, bounds, grid, seed=3, first_draw=2, return_functions=True)
    _same(gp.sample_rff_optima(F, P, bounds, grid, seed=3, first_draw=2, return_functions=True, spectral=KER), ref)
    _same(_ex_entry(gp, F, P, bounds, grid, 3, 2, KER), ref)
    tab = _table(gp, F, P, 3, 2, ref[2]["b"])  # no chi2 needed: the SE draw reads none
    _same(gp.sample_rff_optima(F, P, bounds, grid, table=tab, return_functions=True, spectral=KER), ref)


@pytest.mark.parametrize("n,F", BRANCHES, ids=["woodbury", "cholesky"])
def test_matern_kernel_mode_rescales_the_reference_rows_and_replays_from_a_table(n, F):
    pr, gp = _gp(MATERN, n=n)
    d, P, seed, first = 3, 6, 41, 5
    grid = np.random.default_rng(6).uniform(size=(120, d))
    bounds = np.array([[0.0, 1.0]] * d)
    ref = gp.sample_rff_optima(F, P, bounds, grid, seed=seed, first_draw=first, return_functions=True)
    ker = gp.sample_rff_optima(F, P, bounds, grid, seed=seed, first_draw=first, return_functions=True, spectral=KER)
    g = capi.rff_chi2_draws(seed, first, P, F)
    host = np.stack([RP.chi2_draws(seed, first + s, F) for s in range(P)])
    np.testing.assert_allclose(g, host, rtol=1e-13, atol=0)
    np.testing.assert_array_equal(ker[2]["omega"], ref[2]["omega"] * np.sqrt(5.0 / g)[..., None])
    np.testing.assert_array_equal(ker[2]["b"], ref[2]["b"])
    assert not np.array_equal(ker[2]["theta"], ref[2]["theta"])
    tab = _table(gp, F, P, seed, first, ref[2]["b"], chi2=g)
    _same(gp.sample_rff_optima(F, P, bounds, grid, table=tab, return_functions=True, spectral=KER), ker)


def test_matern_table_replay_matches_the_restatement_on_the_cholesky_branch():
    pr, gp = _gp(MATERN, n=30, d=3)
    F, d = 25, 3
    M = gp.n
    assert M >= F
    rng = np.random.default_rng(8)
    om, bb, z, chi2 = rng.normal(size=(F, d)), rng.uniform(0, 2 * np.pi, size=F), rng.normal(size=F), \
        rng.chisquare(5, size=F)
    tab = {"omega": om[None], "b": bb[None], "z": z[None], "chi2": chi2[None]}
    grid = rng.uniform(size=(400, d))
    fun = gp.sample_rff_functions(F, 1, table=tab, spectral=KER)
    W = RP.matern_frequencies(om, pr["lengths"], chi2)
    np.testing.assert_array_equal(fun.omega[0], W)
    Phi, yp, _, c = R.design(pr["X"], pr["y"].reshape(-1, 1), pr["noise"], [], pr["alpha"], np.ones(d), W, bb)
    th = R.theta(Phi, yp, z)
    np.testing.assert_allclose(fun.theta[0], th, rtol=1e-10, atol=1e-10 * np.abs(th).max())
    gv = R.f_value(grid, W, bb, th, c)
    dv = fun(grid)[0]
    np.testing.assert_allclose(dv, gv, rtol=1e-10, atol=1e-10 * np.abs(gv).max())
    a = int(np.argmin(gv))
    assert np.sort(gv)[1] - np.sort(gv)[0] > 1e-6
    pts, vals = gp.sample_rff_optima(F, 1, np.repeat(grid[a], 2), grid, table=tab, spectral=KER)
    np.testing.assert_array_equal(pts[0], grid[a])


def test_matern_frequencies_have_the_matern_correlation():
    pr, gp = _gp(MATERN, n=8, d=3)
    F, P = 5000, 100
    fun = gp.sample_rff_functions(F, P, seed=19, spectral=KER)
    W = fun.omega.reshape(-1, 3)
    assert W.shape[0] >= 500000
    lengths = pr["lengths"]
    deltas = RP.offsets(lengths)
    z = RP.correlation_z(W, deltas, lambda dl: RP.matern52_corr(dl, lengths))
    assert np.all(np.abs(z) < 5.0), z
    z_se = RP.correlation_z(W, deltas, lambda dl: RP.se_corr(dl, lengths))
    assert np.max(np.abs(z_se)) > 20.0, z_se
    ref = gp.sample_rff_functions(F, 4, seed=19)  # and the reference mode's rows are SE rows
    z_ref = RP.correlation_z(ref.omega.reshape(-1, 3), deltas, lambda dl: RP.se_corr(dl, lengths))
    assert np.all(np.abs(z_ref) < 5.0), z_ref


@pytest.mark.parametrize("kernel,spectral", [(SE, REF), (MATERN, REF), (MATERN, KER)], ids=["se", "m-ref", "m-ker"])
@pytest.mark.parametrize("n,F", BRANCHES, ids=["woodbury", "cholesky"])
def test_functions_entry_is_the_optima_calls_functions(kernel, spectral, n, F):
    pr, gp = _gp(kernel, n=n)
    d, P = 3, 5
    grid = np.random.default_rng(9).uniform(size=(50, d))
    bounds = np.array([[0.0, 1.0]] * d)
    _, _, opt = gp.sample_rff_optima(F, P, bounds, grid, seed=12, first_draw=1, return_functions=True,
                                     spectral=spectral)
    fun = gp.sample_rff_functions(F, P, seed=12, first_draw=1, spectral=spectral)
    np.testing.assert_array_equal(fun.omega, opt["omega"])
    np.testing.assert_array_equal(fun.b, opt["b"])
    np.testing.assert_array_equal(fun.theta, opt["theta"])
    assert fun.c == np.sqrt(2.0 * pr["alpha"] / F)


def _functions(P=3, F=200, d=4, seed=1):
    rng = np.random.default_rng(seed)
    om = rng.normal(size=(P, F, d)) / 0.3
    b = rng.uniform(0, 2 * np.pi, size=(P, F))
    th = rng.normal(size=(P, F))
    return om, b, th, np.sqrt(2.0 * 1.3 / F)


def test_evaluator_against_numpy_and_central_differences():
    om, b, th, c = _functions()
    P, F, d = om.shape
    x = np.random.default_rng(2).uniform(-1, 2, size=(300, d))
    v, g = capi.rff_evaluate(om, b, th, c, x, grads=True)
    for p in range(P):
        scale = c * np.abs(th[p]).sum()
        np.testing.assert_allclose(v[p], RP.f_values(x, om[p], b[p], th[p], c), rtol=0, atol=1e-12 * scale)
        np.testing.assert_allclose(g[p], RP.f_grads(x, om[p], b[p], th[p], c), rtol=0,
                                   atol=1e-12 * scale * np.abs(om[p]).max())
    h = 1e-6
    for k in range(d):
        e = np.zeros(d)
        e[k] = h
        fd = (capi.rff_evaluate(om, b, th, c, x + e) - capi.rff_evaluate(om, b, th, c, x - e)) / (2 * h)
        np.testing.assert_allclose(g[..., k], fd, rtol=1e-6, atol=1e-6 * np.abs(g).max())


def test_evaluator_shared_and_per_function_points_and_batch_invariance():
    om, b, th, c = _functions(P=5, F=300, d=3, seed=3)
    x = np.random.default_rng(4).uniform(size=(257, 3))
    v, g = capi.rff_evaluate(om, b, th, c, x, grads=True)
    vp, gp_ = capi.rff_evaluate(om, b, th, c, np.tile(x, (5, 1, 1)), grads=True)
    np.testing.assert_array_equal(v, vp)
    np.testing.assert_array_equal(g, gp_)
    np.testing.assert_array_equal(capi.rff_evaluate(om, b, th, c, x), v)  # values alone: the same bits
    np.testing.assert_array_equal(capi.rff_evaluate(om, b, th, c, x, values=False, grads=True), g)
    for p in (0, 3):  # one function, a subset of points, points in another order
        one = capi.rff_evaluate(om[p:p + 1], b[p:p + 1], th[p:p + 1], c, x[::-7], grads=True)
        np.testing.assert_array_equal(one[0][0], v[p, ::-7])
        np.testing.assert_array_equal(one[1][0], g[p, ::-7])
    per = np.random.default_rng(5).uniform(size=(5, 40, 3))
    vv = capi.rff_evaluate(om, b, th, c, per)
    for p in range(5):
        np.testing.assert_array_equal(vv[p], capi.rff_evaluate(om[p:p + 1], b[p:p + 1], th[p:p + 1], c, per[p])[0])


def test_evaluator_chunks_over_functions():
    """70 000 functions: the chunk holds at most 65 535 (one grid row per function), so the call spans two."""
    P, F, d = 70000, 3, 2
    rng = np.random.default_rng(6)
    om, b, th = rng.normal(size=(P, F, d)), rng.uniform(0, 6, size=(P, F)), rng.normal(size=(P, F))
    x = rng.uniform(size=(5, d))
    v, g = capi.rff_evaluate(om, b, th, 0.7, x, grads=True)
    for lo in (0, 65533, P - 3):
        sv, sg = capi.rff_evaluate(om[lo:lo + 3], b[lo:lo + 3], th[lo:lo + 3], 0.7, x, grads=True)
        np.testing.assert_array_equal(sv, v[lo:lo + 3])
        np.testing.assert_array_equal(sg, g[lo:lo + 3])
    np.testing.assert_allclose(v[-1], RP.f_values(x, om[-1], b[-1], th[-1], 0.7), rtol=0, atol=1e-12 * 0.7 * 4)


def test_evaluator_chunks_over_points():
    """One function, values only, shared 1-d points: 2 doubles per point, so 2^27 + 2^20 points need two chunks of the
    2 GiB workspace (2^28 doubles)."""
    X = (1 << 27) + (1 << 20)
    om, b, th = np.array([[[3.7]]]), np.array([[0.4]]), np.array([[1.25]])
    x = np.linspace(-5.0, 5.0, X).reshape(X, 1)
    v = capi.rff_evaluate(om, b, th, 0.9, x)
    idx = np.array([0, 1, (1 << 27) - 3, (1 << 27) - 2, (1 << 27) - 1, 1 << 27, X - 2, X - 1])
    np.testing.assert_array_equal(capi.rff_evaluate(om, b, th, 0.9, x[idx])[0], v[0, idx])
    np.testing.assert_allclose(v[0, idx], RP.f_values(x[idx], om[0], b[0], th[0], 0.9), rtol=0, atol=1e-12 * 1.2)


def test_evaluator_at_the_returned_optima_gives_the_optima_values():
    pr, gp = _gp(MATERN, n=40, d=3)
    F, P = 300, 16
    grid = np.random.default_rng(10).uniform(size=(400, 3))
    bounds = np.array([[0.0, 1.0]] * 3)
    pts, vals, fun = gp.sample_rff_optima(F, P, bounds, grid, seed=5, return_functions=True, spectral=KER)
    c = np.sqrt(2.0 * pr["alpha"] / F)
    v = capi.rff_evaluate(fun["omega"], fun["b"], fun["theta"], c, pts[:, None, :])[:, 0]
    for s in range(P):
        on_grid = np.any(np.all(grid == pts[s], axis=1))
        if on_grid:  # the grid stage's arithmetic: the same bits
            assert v[s] == vals[s]
        else:
            assert abs(v[s] - vals[s]) <= 1e-12 * c * np.abs(fun["theta"][s]).sum()
    gvals = capi.rff_evaluate(fun["omega"], fun["b"], fun["theta"], c, grid)
    assert np.all(vals <= gvals.min(axis=1))


def test_evaluator_size_edges():
    om, b, th, c = _functions(P=1, F=1, d=1)
    v, g = capi.rff_evaluate(om, b, th, c, np.array([[0.3]]), grads=True)
    assert v.shape == (1, 1) and g.shape == (1, 1, 1)
    np.testing.assert_allclose(v[0, 0], c * th[0, 0] * np.cos(om[0, 0, 0] * 0.3 + b[0, 0]), rtol=1e-15)
    om, b, th, c = _functions(P=2, F=130, d=32)  # the largest dim, features over two shared-memory rounds
    x = np.random.default_rng(3).uniform(size=(3, 32))
    v, g = capi.rff_evaluate(om, b, th, c, x, grads=True)
    np.testing.assert_allclose(v[1], RP.f_values(x, om[1], b[1], th[1], c), rtol=0, atol=1e-12 * c * np.abs(th[1]).sum())
    with pytest.raises(capi.BoundsError):
        capi.rff_evaluate(np.zeros((1, 2, 33)), np.zeros((1, 2)), np.zeros((1, 2)), 1.0, np.zeros((1, 33)))
    with pytest.raises(capi.InvalidValueError):
        capi.rff_evaluate(om, b, th, np.nan, x)


def test_sample_errors_on_a_handle():
    pr, gp = _gp(MATERN, n=10, d=2)
    grid = np.full((1, 2), 0.5)
    bounds = np.array([[0.0, 1.0]] * 2)
    with pytest.raises(capi.InvalidValueError, match="spectral"):
        gp.sample_rff_optima(20, 1, bounds, grid, spectral=2)
    with pytest.raises(capi.InvalidValueError, match="spectral"):
        gp.sample_rff_functions(20, 1, spectral=-1)
    F = 20
    tab = {"omega": np.zeros((1, F, 2)), "b": np.zeros((1, F)), "z": np.zeros((1, F)), "eps": np.zeros((1, 10))}
    with pytest.raises(capi.InvalidValueError, match="chi2"):  # the Matern table needs chi2
        gp.sample_rff_functions(F, 1, table=tab, spectral=KER)
    for bad in (0.0, -1.0, np.inf, np.nan):
        chi2 = np.ones((1, F))
        chi2[0, 7] = bad
        with pytest.raises(capi.InvalidValueError, match="chi2"):
            gp.sample_rff_functions(F, 1, table=dict(tab, chi2=chi2), spectral=KER)
    gp.sample_rff_functions(F, 1, table=dict(tab, chi2=np.ones((1, F))), spectral=KER)


def _reference_wrapper(W, b, theta, c):
    """random_features.py:113-131, restated (b is a column there)."""
    def wrapper(x, gradient):
        if x.ndim == 1:
            x = x[None, :]
        if not gradient:
            result = np.dot(theta.T, c * np.cos(np.dot(W, x.T) + b[:, None]))
            if result.size == 1:
                result = float(result[0])
            return result
        return np.dot(theta.T, -c * np.sin(np.dot(W, x.T) + b[:, None]) * W)
    return wrapper


def test_gpp_names_and_the_wrapper_convention():
    import GPP as C_GP
    pr = make_problem(25, 2, (), seed=17)
    gpp = C_GP.GaussianProcess([pr["alpha"], list(pr["lengths"])], list(pr["X"].ravel()), list(pr["y"]),
                               list(pr["noise"]), [], 0, 2, 25)  # Matern-5/2, as the reference's boundary
    gp = capi.GaussianProcess(MATERN, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"])
    gpp.set_explicit_seed(123)

    class Wrapper:
        _gaussian_process = gpp

    f0 = C_GP.sample_gp_with_random_features(gpp, 60)
    f1 = C_GP.sample_gp_with_random_features(Wrapper(), 60, True)
    for f, draw, spectral in ((f0, 0, REF), (f1, 1, KER)):
        want = gp.sample_rff_functions(60, 1, seed=123, first_draw=draw, spectral=spectral)
        np.testing.assert_array_equal(f.omega, want.omega[0])
        np.testing.assert_array_equal(f.b, want.b[0])
        np.testing.assert_array_equal(f.theta, want.theta[0])
        assert f.c == want.c
        ref = _reference_wrapper(f.omega, f.b, f.theta, f.c)
        x1 = np.array([0.3, 0.6])
        xs = np.random.default_rng(1).uniform(size=(7, 2))
        v1 = f(x1, False)
        assert isinstance(v1, float) and abs(v1 - ref(x1, False)) <= 1e-13
        assert isinstance(f(x1[None], gradient=False), float)
        g1 = f(x1, True)
        assert g1.shape == ref(x1, True).shape == (2,)
        np.testing.assert_allclose(g1, ref(x1, True), rtol=1e-12, atol=1e-13)
        vs = f(xs, gradient=False)
        assert vs.shape == (7,)
        np.testing.assert_allclose(vs, ref(xs, False), rtol=1e-12, atol=1e-13)
        np.testing.assert_array_equal(vs, want(xs)[0])
        assert f(xs, gradient=True).shape == (7, 2)
    grid = np.random.default_rng(18).uniform(size=(60, 2))
    bounds = [0.0, 1.0, 0.0, 1.0]
    a = np.array(C_GP.sample_from_global_optima_kernel_matched(gpp, 50, bounds, list(grid.ravel()), 60, 3)).reshape(3, 2)
    want, _ = gp.sample_rff_optima(50, 3, bounds, grid, seed=123, first_draw=2, spectral=KER)
    np.testing.assert_array_equal(a, want)
    b = np.array(C_GP.sample_from_global_optima(gpp, 50, bounds, list(grid.ravel()), 60, 3)).reshape(3, 2)
    want_ref, _ = gp.sample_rff_optima(50, 3, bounds, grid, seed=123, first_draw=5)
    np.testing.assert_array_equal(b, want_ref)

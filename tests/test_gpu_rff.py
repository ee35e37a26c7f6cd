"""GPU tests of the random-feature sampler (cmoe_gp_sample_rff_optima, DESIGN.md K14): table mode against the unmodified
reference routine (tests/golden/reference_rff.npz) and the NumPy restatement (tests/rff_ref.py); the local optimiser's
bounds, grid-minimum, KKT and SLSQP checks; Philox against table mode; independence of the result from the run, P and
the chunking; the distribution of theta; the size limits and the front ends."""
import os
import sys

import numpy as np
import pytest
import scipy.optimize as spo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))

from cornell_moe_b200 import capi  # noqa: E402

import rff_ref as R  # noqa: E402
from synth import make_problem  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = R.golden_cases()
IDS = [n for n, _ in CASES]
# Noise 1e-8 puts entries near 1e4 into Phi, so B (or A) has a condition number near 1e8.  On the Cholesky branch the
# device and the reference then agree within 1e-6 of max|theta|.  The Woodbury branch forms theta = r - Phi A^-1 Phi^T r
# from terms about 1e8 times larger than theta, and both codes lose those digits: measured on an H100, the device and
# the reference (or the restatement) differ by up to 2.6e-5 of max|theta| there.
NOISE_FREE_TOL = {"cholesky": 1e-6, "woodbury": 1e-4}
KKT_TOL = 1e-9


def _tol(c):
    if c["noise"][0] >= 1e-6:
        return 1e-10
    return NOISE_FREE_TOL["woodbury" if _M(c) < int(c["F"]) else "cholesky"]


def _gp(c):
    return capi.GaussianProcess(0, float(c["alpha"]), c["lengths"], c["X"], c["Y"], c["noise"], c["derivs"])


def _M(c):
    return c["X"].shape[0] * (1 + len(c["derivs"]))


def _table(c, z=None, eps=None, P=1):
    F, M = int(c["F"]), _M(c)
    z = np.zeros(F) if z is None else z
    eps = np.zeros(M) if eps is None else eps
    return {"omega": np.tile(c["omega"], (P, 1, 1)), "b": np.tile(c["b"], (P, 1)), "z": np.tile(z, (P, 1)),
            "eps": np.tile(eps, (P, 1))}


def _close(a, b, tol):
    np.testing.assert_allclose(a, b, rtol=tol, atol=tol * np.abs(b).max())


@pytest.mark.parametrize("name,c", CASES, ids=IDS)
def test_table_mean_matches_the_reference(name, c):
    gp = _gp(c)
    _, _, fun = gp.sample_rff_optima(int(c["F"]), 1, c["bounds"], c["grid"], table=_table(c), return_functions=True)
    np.testing.assert_array_equal(fun["omega"][0], c["W"])
    np.testing.assert_array_equal(fun["b"][0], c["b"])
    _close(fun["theta"][0], c["m"], _tol(c))


@pytest.mark.parametrize("name,c", CASES, ids=IDS)
def test_table_draw_matches_the_reference_or_the_restatement(name, c):
    """M >= F: the reference's own draw; M < F: the restatement's pathwise draw (the reference uses eigh there)."""
    gp = _gp(c)
    F, M = int(c["F"]), _M(c)
    eps = np.random.default_rng(5).normal(size=M)
    _, _, fun = gp.sample_rff_optima(F, 1, c["bounds"], c["grid"], table=_table(c, c["z"], eps), return_functions=True)
    if M >= F:
        want = c["theta"]
    else:
        Phi, yp, _, _ = R.design(c["X"], c["Y"], c["noise"], c["derivs"], float(c["alpha"]), c["lengths"], c["omega"],
                                 c["b"])
        want = R.theta(Phi, yp, c["z"], eps)
    _close(fun["theta"][0], want, _tol(c))


@pytest.mark.parametrize("draw", ["mean", "draw"])
@pytest.mark.parametrize("name,c", CASES, ids=IDS)
def test_grid_argmin_values_and_the_local_end_point(name, c, draw):
    """Against the reference's grid evaluation, argmin and SLSQP end point: of the mean's sample function (z = eps = 0,
    both branches) and of the draw (M >= F only: on the M < F branch the device's draw is not the reference's)."""
    gp = _gp(c)
    F = int(c["F"])
    sfx = "_m" if draw == "mean" else ""
    if draw == "draw":
        if _M(c) < F:
            pytest.skip("M < F: the device's draw is the pathwise one, not the reference's eigh draw")
        tab, theta = _table(c, c["z"], np.random.default_rng(5).normal(size=_M(c))), c["theta"]
    else:
        tab, theta = _table(c), c["m"]
    grid, gvals, a = c["grid"], c["grid_vals" + sfx], int(c["grid_argmin" + sfx])
    tol = max(1e-9, _tol(c))
    # grid values: a one-point grid with a degenerate box returns f there
    for j in range(0, grid.shape[0], 25):
        x = grid[j]
        _, vals = gp.sample_rff_optima(F, 1, np.repeat(x, 2), x[None], table=tab)
        _close(vals, gvals[j:j + 1], tol)
    # argmin: a box degenerate at the reference's argmin returns that point only if the device picked it too
    gv = np.sort(gvals)
    assert gv[1] - gv[0] > 1e-6 * max(1.0, abs(gv[0]))
    pts, vals = gp.sample_rff_optima(F, 1, np.repeat(grid[a], 2), grid, table=tab)
    np.testing.assert_array_equal(pts[0], grid[a])
    _close(vals, gvals[a:a + 1], tol)
    # the end point from the same grid point: the device value is at most the reference's plus SLSQP's accuracy (and
    # the two functions' own difference, tol, on the noise-free cases)
    pts, vals = gp.sample_rff_optima(F, 1, c["bounds"], grid, table=tab)
    cc = np.sqrt(2.0 * float(c["alpha"]) / F)
    f_ref = R.f_value(c["point" + sfx], c["W"], c["b"], theta, cc)[0]
    assert vals[0] <= f_ref + max(1e-6, tol) * max(1.0, abs(f_ref)), (vals[0], f_ref)
    assert np.all(pts[0] >= 0.0) and np.all(pts[0] <= 1.0)
    if abs(vals[0] - f_ref) < 1e-7:
        np.testing.assert_allclose(pts[0], c["point" + sfx], atol=2e-3)


def _problem(n=40, d=3, derivs=(), seed=11):
    pr = make_problem(n, d, derivs, seed=seed, noise=1e-2, length=0.4)
    return pr, capi.GaussianProcess(0, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"])


def test_optimiser_bounds_grid_minimum_kkt_and_slsqp():
    # length scales near the box's width: few basins, so SLSQP and the Newton method from one start reach the same one
    pr = make_problem(40, 3, (), seed=11, noise=1e-2, length=1.0)
    gp = capi.GaussianProcess(0, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"])
    d, F, P = 3, 300, 48
    bounds = np.array([[-0.2, 1.1], [0.0, 1.0], [0.1, 0.9]])
    grid = np.random.default_rng(3).uniform(bounds[:, 0], bounds[:, 1], size=(400, d))
    pts, vals, fun = gp.sample_rff_optima(F, P, bounds, grid, seed=21, return_functions=True)
    c = np.sqrt(2.0 * pr["alpha"] / F)
    moved = 0
    for s in range(P):
        W, b, th = fun["omega"][s], fun["b"][s], fun["theta"][s]
        gvals = R.f_value(grid, W, b, th, c)
        x = pts[s]
        assert np.all(x >= bounds[:, 0]) and np.all(x <= bounds[:, 1])
        fx = R.f_value(x, W, b, th, c)[0]
        assert abs(fx - vals[s]) <= 1e-12 * (1.0 + abs(fx))
        assert vals[s] <= gvals.min() + 1e-12 * (1.0 + abs(gvals.min()))
        if not np.any(np.all(grid == x, axis=1)):
            moved += 1
            res = R.kkt_residual(x, R.f_grad(x, W, b, th, c), bounds[:, 0], bounds[:, 1])
            assert res <= KKT_TOL * (1.0 + abs(fx)) + 1e-11, (s, res)
        x0 = grid[int(np.argmin(gvals))]
        xs = spo.fmin_slsqp(lambda v: float(R.f_value(v, W, b, th, c)[0]), x0.copy(), bounds=[tuple(r) for r in bounds],
                            disp=0, fprime=lambda v: R.f_grad(v, W, b, th, c))
        f_slsqp = float(R.f_value(xs, W, b, th, c)[0])
        assert vals[s] <= f_slsqp + 1e-6, (s, vals[s], f_slsqp, x, xs, x0)
    assert moved >= P // 2


def test_philox_mode_is_table_mode_fed_the_same_numbers():
    for n, derivs, F in ((30, (), 80), (30, (1,), 40)):  # M < F, then M >= F
        pr, gp = _problem(n=n, derivs=derivs)
        M, d, P, seed = n * (1 + len(derivs)), 3, 5, 77
        grid = np.random.default_rng(4).uniform(size=(100, d))
        bounds = np.array([[0.0, 1.0]] * d)
        p1, v1, f1 = gp.sample_rff_optima(F, P, bounds, grid, seed=seed, first_draw=9, return_functions=True)
        nrm = capi.philox_normals(seed, 9, P, F * d + F + M)
        tab = {"omega": nrm[:, :F * d], "b": f1["b"], "z": nrm[:, F * d:F * d + F], "eps": nrm[:, F * d + F:]}
        p2, v2, f2 = gp.sample_rff_optima(F, P, bounds, grid, table=tab, return_functions=True)
        for k in f1:
            np.testing.assert_array_equal(f1[k], f2[k])
        np.testing.assert_array_equal(p1, p2)
        np.testing.assert_array_equal(v1, v2)
        assert np.all((f1["b"] >= 0.0) & (f1["b"] < 2.0 * np.pi))


# Samples per chunk (rff.cu): floor(2 GiB / per), per = 8 (F M + Q^2 + 64^2 ceil(Q / 64) + F (d + 4) + M + gx + 2 d + 1
# [+ F (d + 2) + M with a table]) + 4 (gx + 2) bytes, Q = min(F, M), gx = ceil(G / 256) grid CTAs.
CHUNK_CASES = [  # n, F, P: M < F with 5 samples per chunk (about 0.40 GB each), M >= F with 2 (about 0.79 GB each)
    (4096, 8192, 7),
    (20000, 4096, 3),
]


def _per_sample_bytes(F, M, d, G, table):
    Q, gx = min(F, M), -(-G // 256)
    dbl = F * M + Q * Q + 64 * 64 * -(-Q // 64) + F * (d + 4) + M + gx + 2 * d + 1 + (F * (d + 2) + M if table else 0)
    return 8 * dbl + 4 * (gx + 2)


@pytest.mark.parametrize("n,F,P", CHUNK_CASES)
def test_samples_do_not_depend_on_the_run_P_or_the_chunking(n, F, P):
    """Sample s of a P-sample call that spans chunks equals the one-sample call at draw s (Philox) or with row s of the
    table, bit for bit; so do the draw offsets, the table offsets and the output offsets of every chunk."""
    d, G = 2, 64
    pr, gp = _problem(n=n, d=d, seed=12)
    grid = np.random.default_rng(6).uniform(size=(G, d))
    bounds = np.array([[0.0, 1.0]] * d)
    M = n
    for table in (False, True):
        chunk = (2 << 30) // _per_sample_bytes(F, M, d, G, table)
        assert 1 <= chunk < P, chunk  # the call spans at least two chunks
    a = gp.sample_rff_optima(F, P, bounds, grid, seed=5, first_draw=3, return_functions=True)
    b = gp.sample_rff_optima(F, P, bounds, grid, seed=5, first_draw=3, return_functions=True)
    for x, y in zip(a[:2], b[:2]):
        np.testing.assert_array_equal(x, y)
    for s in range(P):
        one = gp.sample_rff_optima(F, 1, bounds, grid, seed=5, first_draw=3 + s, return_functions=True)
        np.testing.assert_array_equal(one[0][0], a[0][s])
        np.testing.assert_array_equal(one[1][0], a[1][s])
        for k in ("omega", "b", "theta"):
            np.testing.assert_array_equal(one[2][k][0], a[2][k][s])
    # table mode: the chunk offsets into omega, b, z and eps
    nrm = capi.philox_normals(5, 3, P, F * d + F + M)
    tab = {"omega": nrm[:, :F * d], "b": a[2]["b"], "z": nrm[:, F * d:F * d + F]}
    if M < F:
        tab["eps"] = nrm[:, F * d + F:]
    t = gp.sample_rff_optima(F, P, bounds, grid, table=tab, return_functions=True)
    np.testing.assert_array_equal(t[0], a[0])
    np.testing.assert_array_equal(t[1], a[1])
    np.testing.assert_array_equal(t[2]["theta"], a[2]["theta"])


def test_samples_do_not_depend_on_P():
    pr, gp = _problem()
    grid = np.random.default_rng(7).uniform(size=(50, 3))
    big = gp.sample_rff_optima(100, 9, np.array([[0.0, 1.0]] * 3), grid, seed=8)
    for P in (1, 4):
        small = gp.sample_rff_optima(100, P, np.array([[0.0, 1.0]] * 3), grid, seed=8)
        np.testing.assert_array_equal(small[0], big[0][:P])


@pytest.mark.parametrize("F,n", [(12, 8), (6, 8)])
def test_theta_has_the_posterior_distribution(F, n):
    pr, gp = _problem(n=n, d=2, seed=13)
    M, N = n, 4096
    rng = np.random.default_rng(F)
    om, bb = rng.normal(size=(F, 2)), rng.uniform(0.0, 2.0 * np.pi, size=F)
    tab = {"omega": np.tile(om, (N, 1, 1)), "b": np.tile(bb, (N, 1)), "z": rng.normal(size=(N, F)),
           "eps": rng.normal(size=(N, M))}
    grid = np.full((1, 2), 0.5)
    bounds = np.array([[0.5, 0.5]] * 2)
    _, _, fun = gp.sample_rff_optima(F, N, bounds, grid, table=tab, return_functions=True)
    Phi, yp, _, _ = R.design(pr["X"], pr["y"].reshape(n, 1), pr["noise"], [], pr["alpha"], pr["lengths"], om, bb)
    Sigma = R.posterior_cov(Phi)
    m = Sigma @ Phi @ yp
    T = fun["theta"] - m
    S = T.T @ T / N
    sd = np.sqrt((np.outer(np.diag(Sigma), np.diag(Sigma)) + Sigma ** 2) / N)
    assert np.all(np.abs(S - Sigma) <= 4.0 * sd), np.max(np.abs(S - Sigma) / sd)


def _rc(gp, F, P, bounds, grid, G=None):
    try:
        gp.sample_rff_optima(F, P, bounds, grid if G is None else grid[:G])
        return capi.OK
    except capi.CmoeError as e:
        return e.code


def test_size_limits_just_inside_and_just_past():
    pr, gp = _problem(n=3, d=2)
    g1 = np.full((1, 2), 0.5)
    b1 = np.array([[0.5, 0.5]] * 2)
    assert _rc(gp, 1, 1, b1, g1) == capi.OK
    assert _rc(gp, 0, 1, b1, g1) == capi.ERR_BOUNDS
    assert _rc(gp, 1, 0, b1, g1) == capi.ERR_BOUNDS
    assert _rc(gp, 1, 1, b1, np.zeros((0, 2))) == capi.ERR_BOUNDS
    bad = g1.copy()
    bad[0, 1] = np.nan
    assert _rc(gp, 4, 1, b1, bad) == capi.ERR_INVALID_VALUE
    assert _rc(gp, 4, 1, np.array([[0.0, np.inf], [0.0, 1.0]]), g1) == capi.ERR_INVALID_VALUE
    assert _rc(gp, 4, 1, np.array([[0.6, 0.5], [0.0, 1.0]]), g1) == capi.ERR_INVALID_VALUE
    # one sample's Phi plus its Gram within 2^28 doubles: with M = 8192 < F, 8192 F + 8192^2 <= 2^28 gives F <= 24576
    one, box = np.full((1, 1), 0.5), np.array([[0.5, 0.5]])
    edge = make_problem(8192, 1, (), seed=1)
    gpe = capi.GaussianProcess(0, edge["alpha"], edge["lengths"], edge["X"], edge["y"], edge["noise"])
    assert _rc(gpe, 24576, 1, box, one) == capi.OK
    assert _rc(gpe, 24577, 1, box, one) == capi.ERR_BOUNDS
    # min(F, M) <= 8192
    big = make_problem(8193, 1, (), seed=2)
    gpb = capi.GaussianProcess(0, big["alpha"], big["lengths"], big["X"], big["y"], big["noise"])
    assert _rc(gpb, 8192, 1, box, one) == capi.OK
    assert _rc(gpb, 8193, 1, box, one) == capi.ERR_BOUNDS


def test_gpp_entry_and_wrapper_use_the_gps_draws_and_leave_it_unchanged():
    import GPP as C_GP
    pr = make_problem(25, 2, (), seed=17)
    gpp = C_GP.GaussianProcess([pr["alpha"], list(pr["lengths"])], list(pr["X"].ravel()), list(pr["y"]),
                               list(pr["noise"]), [], 0, 2, 25)
    gpp.set_explicit_seed(123)
    grid = np.random.default_rng(18).uniform(size=(60, 2))
    bounds = [0.0, 1.0, 0.0, 1.0]

    class Wrapper:
        _gaussian_process = gpp

    a = np.array(C_GP.sample_from_global_optima(gpp, 50, bounds, list(grid.ravel()), 60, 3)).reshape(3, 2)
    b = np.array(C_GP.sample_from_global_optima(Wrapper(), 50, bounds, list(grid.ravel()), 60, 2)).reshape(2, 2)
    gp = capi.GaussianProcess(1, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"])
    before = gp.state()
    ref, _ = gp.sample_rff_optima(50, 5, bounds, grid, seed=123)
    np.testing.assert_array_equal(np.vstack([a, b]), ref)
    after = gp.state()
    for x, y in zip(before, after):
        np.testing.assert_array_equal(x, y)

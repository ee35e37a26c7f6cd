"""Ensemble posterior mean on the device (cmoe_posterior_mean_mcmc, cmoe_posterior_mean_mcmc_optimization, their GPP and
capi bindings): screening against the reference's answers and the CPU checker, the optimiser against every case of
tests/golden/reference_pm_mcmc.npz, bit-identity of a start or a point alone and inside a large batch, and the GPP
functions against capi on the same inputs."""
import collections
import ctypes
import os
import sys

import numpy as np
import pytest

from cornell_moe_b200 import capi
from gpu_util import checker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "reference_pm_mcmc.npz"))
CASES = [str(c) for c in GOLDEN["cases"]]
EPS = np.finfo(np.float64).eps
gpu = pytest.mark.gpu


def golden_case(name):
    return {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(name + "_")}


def _derivs(g):
    return [int(d) for d in g["derivs"]] or None


def device_ensemble(g):
    return capi.GaussianProcessEnsemble(g["hypers"], g["noises"], g["X"], g["y"], derivs=_derivs(g),
                                        kernel=int(g["kernel"]))


def checker_members(g):
    out = []
    for h, noise in zip(g["hypers"], g["noises"]):
        gp, lm = checker().gp(int(g["kernel"]), h[0], h[1:], g["X"], g["y"], noise, derivs=_derivs(g))
        assert lm == 0
        out.append(gp)
    return out


def checker_screen(cpu_gps, pts, num_fidelity):
    """-(1/M) sum_m mu_m, its gradient on the free coordinates and -mu_m, from the CPU checker."""
    dim = cpu_gps[0].dim
    ps = dim - num_fidelity
    full = np.ones((pts.shape[0], dim))
    full[:, :ps] = pts
    mus = np.array([gp.mean_additional(full) for gp in cpu_gps])
    gmus = np.array([[gp.posterior(x, want=("grad_mean",))["grad_mean"][:ps] for x in full] for gp in cpu_gps])
    return -mus.mean(axis=0), -gmus.mean(axis=0), -mus


def mean_tolerance(cpu_gps):
    """Relative tolerance of a posterior mean computed by two implementations: the solves K^-1 (y - m) agree to about
    cond(K) eps, so allow 64 cond(K) eps for the largest condition number among the members (asserted < 1e7)."""
    cond = max(np.linalg.cond(np.tril(gp.state()[0]) @ np.tril(gp.state()[0]).T) for gp in cpu_gps)
    assert cond < 1e7, cond
    return 64 * cond * EPS


def gd_params(g):
    p = g["params"]
    return capi.GDParams(int(p[0]), int(p[1]), int(p[2]), int(p[3]), float(p[4]), float(p[5]), float(p[6]),
                         float(p[7]))


@gpu
@pytest.mark.parametrize("name", ["branin", "fidelity", "derivs", "navbig"])
def test_screening_matches_reference_and_checker(name):
    g = golden_case(name)
    nf = int(g["num_fidelity"])
    ens = device_ensemble(g)
    vals, grads, members = ens.posterior_mean(g["eval_pts"], nf, grad=True, per_member=True)
    cpu = checker_members(g)
    tol = mean_tolerance(cpu)
    scale = np.abs(g["screen"]).max()
    np.testing.assert_allclose(vals, g["screen"], rtol=tol, atol=tol * scale)  # the reference's PosteriorMeanMCMC
    cv, cg, cm = checker_screen(cpu, g["eval_pts"], nf)
    np.testing.assert_allclose(vals, cv, rtol=tol, atol=tol * scale)
    np.testing.assert_allclose(members, cm, rtol=tol, atol=tol * np.abs(cm).max())
    np.testing.assert_allclose(grads, cg, rtol=tol, atol=tol * np.abs(cg).max())
    # values and gradients alone are the same numbers as with the other outputs
    np.testing.assert_array_equal(ens.posterior_mean(g["eval_pts"], nf), vals)


@gpu
def test_per_member_is_each_members_mean_and_identical_members_are_the_single_gp():
    g = golden_case("fidelity")
    nf = int(g["num_fidelity"])
    ens = device_ensemble(g)
    pts = g["eval_pts"]
    _, members = ens.posterior_mean(pts, nf, per_member=True)
    full = np.ones((pts.shape[0], ens.dim))
    full[:, :ens.dim - nf] = pts
    for m, gp in enumerate(ens.members):
        mu = gp.posterior(full[:, None, :], want=("mean",))["mean"][:, 0]
        np.testing.assert_array_equal(members[m], -mu)
    one = ens.members[0]
    same = capi.GaussianProcessEnsemble.from_members([one] * 4)
    single = capi.GaussianProcessEnsemble.from_members([one])
    np.testing.assert_allclose(same.posterior_mean(pts, nf), single.posterior_mean(pts, nf), rtol=4 * EPS, atol=0)
    np.testing.assert_array_equal(single.posterior_mean(pts, nf), members[0])


@gpu
def test_members_with_different_numbers_of_points():
    g = golden_case("branin")
    ens = device_ensemble(g)
    rng = np.random.default_rng(7)
    new = np.column_stack([rng.uniform(-5, 10, 6), rng.uniform(0, 15, 6)])
    new_y = rng.standard_normal(6)
    ens.members[1].add_sampled_points(new, new_y)
    ens.members[3].add_sampled_points(new[:2], new_y[:2])
    mixed = capi.GaussianProcessEnsemble.from_members(ens.members)
    assert sorted({gp.N for gp in mixed.members}) == [20, 22, 26]
    cpu = []
    for m, (h, noise) in enumerate(zip(g["hypers"], g["noises"])):
        k = {1: 6, 3: 2}.get(m, 0)
        gp, lm = checker().gp(int(g["kernel"]), h[0], h[1:], np.vstack([g["X"], new[:k]]),
                              np.concatenate([g["y"], new_y[:k]]), noise)
        assert lm == 0
        cpu.append(gp)
    vals, grads = mixed.posterior_mean(g["eval_pts"], grad=True)
    cv, cg, _ = checker_screen(cpu, g["eval_pts"], 0)
    tol = mean_tolerance(cpu)
    np.testing.assert_allclose(vals, cv, rtol=tol, atol=tol * np.abs(cv).max())
    np.testing.assert_allclose(grads, cg, rtol=tol, atol=tol * np.abs(cg).max())
    # the optimiser accepts the mixed ensemble, and its value at the averaged point is the screening value there
    best, bv, pts, v = mixed.posterior_mean_optimization(g["starts"], gd_params(g), g["bounds"])
    np.testing.assert_allclose(v, mixed.posterior_mean(pts), rtol=1e-13, atol=1e-13 * np.abs(v).max())


@gpu
@pytest.mark.parametrize("name", CASES)
def test_optimiser_matches_every_reference_case(name):
    """Each start runs the reference's GradientDescentOptimizer; only the rounding of grad f differs, so the averaged
    points follow the reference's to within a small multiple of the screening tolerance."""
    g = golden_case(name)
    nf = int(g["num_fidelity"])
    ens = device_ensemble(g)
    best, bv, pts, vals = ens.posterior_mean_optimization(g["starts"], gd_params(g), g["bounds"], nf)
    rel_pts = np.abs(pts - g["points"]).max() / np.abs(g["points"]).max()
    rel_vals = np.abs(vals - g["values"]).max() / np.abs(g["values"]).max()
    print(f"{name}: largest relative difference to the reference: points {rel_pts:.2e}, values {rel_vals:.2e}")
    assert rel_pts < 1e-8 and rel_vals < 1e-8
    # strict `>` in start order: the first maximum.  Starts that converge to the same optimum tie up to rounding, so the
    # reference's choice is required only among starts whose values it separates by more than the tolerance.
    first = int(np.argmax(vals))
    np.testing.assert_array_equal(best, pts[first])
    assert bv == vals[first]
    ref_best = int(g["best_index"])
    tied = np.flatnonzero(np.abs(g["values"] - g["values"][ref_best]) <= 1e-8 * np.abs(g["values"]).max())
    assert first in tied and (len(tied) > 1 or first == ref_best)
    np.testing.assert_allclose(best, g["best_point"], rtol=1e-8, atol=1e-10)
    report = ens.recommend_point(g["eval_pts"], gd_params(g), g["bounds"], nf)
    np.testing.assert_allclose(report, g["report_point"], rtol=1e-8, atol=1e-10)
    if name == "dup":  # identical starts give identical bits; the first of them is reported
        np.testing.assert_array_equal(pts[1], pts[2])
        assert first == 1
    if name in ("nav0", "navneg", "navbig"):  # a start on the upper corner with mrc * dist = 0 does not move
        np.testing.assert_array_equal(pts[2], g["starts"][2])


@gpu
def test_a_start_and_a_point_give_the_same_bits_alone_and_in_a_large_batch():
    g = golden_case("branin")
    ens = device_ensemble(g)
    rng = np.random.default_rng(11)
    lo, hi = g["bounds"][:, 0], g["bounds"][:, 1]
    starts = lo + (hi - lo) * rng.uniform(size=(1000, 2))
    _, _, pts, vals = ens.posterior_mean_optimization(starts, gd_params(g), g["bounds"])
    for i in (0, 517, 999):
        _, _, p1, v1 = ens.posterior_mean_optimization(starts[i:i + 1], gd_params(g), g["bounds"])
        np.testing.assert_array_equal(p1[0], pts[i])
        assert v1[0] == vals[i]
    screen = lo + (hi - lo) * rng.uniform(size=(10000, 2))
    v, gr = ens.posterior_mean(screen, grad=True)
    for i in (0, 4321, 9999):
        v1, g1 = ens.posterior_mean(screen[i:i + 1], grad=True)
        assert v1[0] == v[i]
        np.testing.assert_array_equal(g1[0], gr[i])


@gpu
def test_gpp_functions_agree_with_capi():
    import GPP  # noqa: E402

    g = golden_case("fidelity")
    nf = int(g["num_fidelity"])
    X, y, dim = g["X"], g["y"], g["X"].shape[1]
    ps = dim - nf
    ens = device_ensemble(g)
    mcmc = GPP.GaussianProcessMCMC(list(g["hypers"].ravel()), list(g["noises"].ravel()), list(X.ravel()), list(y), [],
                                   len(g["hypers"]), 0, dim, X.shape[0])
    as_list = [GPP.GaussianProcess([h[0], list(h[1:])], list(X.ravel()), list(y), list(noise), [], 0, dim, X.shape[0])
               for h, noise in zip(g["hypers"], g["noises"])]
    pts = g["eval_pts"]
    vals, grads = ens.posterior_mean(pts, nf, grad=True)
    p = gd_params(g)
    best, _, _, fvals = ens.posterior_mean_optimization(g["starts"], p, g["bounds"], nf)
    PyParams = collections.namedtuple("GradientDescentParameters", ["max_num_steps", "max_num_restarts",
                                                                    "num_steps_averaged", "gamma", "pre_mult",
                                                                    "max_relative_change", "tolerance"])
    for gps in (mcmc, as_list):
        v = GPP.compute_posterior_mean_mcmc_of_points(gps, nf, list(pts.ravel()), pts.shape[0])
        np.testing.assert_array_equal(v, vals)
        gr = GPP.compute_grad_posterior_mean_mcmc_of_points(gps, nf, list(pts.ravel()), pts.shape[0])
        np.testing.assert_array_equal(np.reshape(gr, (-1, ps)), grads)
        for params in (GPP.GradientDescentParameters(1, p.max_num_steps, 3, p.num_steps_averaged, p.gamma, p.pre_mult,
                                                     p.max_relative_change, 1e-10),
                       PyParams(p.max_num_steps, 3, p.num_steps_averaged, p.gamma, p.pre_mult, p.max_relative_change,
                                1e-10)):
            bp, fv = GPP.posterior_mean_mcmc_optimization(gps, nf, params, list(g["bounds"].ravel()),
                                                          list(g["starts"].ravel()), g["starts"].shape[0])
            np.testing.assert_array_equal(bp, best)
            np.testing.assert_array_equal(fv, fvals)


@gpu
def test_input_checks_that_need_a_handle():
    g = golden_case("branin")
    ens = device_ensemble(g)
    buf, info = np.zeros(8), ctypes.c_int()
    for nf in (2, 3):  # num_fidelity >= dim leaves no free coordinate
        rc = capi.lib().cmoe_posterior_mean_mcmc(ens._handles(), len(ens), nf, capi._d(buf), 1, capi._d(buf), None,
                                                 None, ctypes.byref(info))
        assert rc == capi.ERR_BOUNDS and "num_fidelity" in capi.lib().cmoe_last_error().decode()
        p = gd_params(g)
        rc = capi.lib().cmoe_posterior_mean_mcmc_optimization(ens._handles(), len(ens), nf, ctypes.byref(p),
                                                              capi._d(buf), capi._d(buf), 1, None, None, None, None,
                                                              ctypes.byref(info))
        assert rc == capi.ERR_BOUNDS and "num_fidelity" in capi.lib().cmoe_last_error().decode()
    with pytest.raises(capi.BoundsError, match="EMPTY"):
        ens.posterior_mean_optimization(g["starts"], gd_params(g), [[-5.0, 10.0], [15.0, 0.0]])
    p = gd_params(g)
    p.max_num_steps = 0
    with pytest.raises(capi.BoundsError, match="max_num_steps"):
        ens.posterior_mean_optimization(g["starts"], p, g["bounds"])
    # a mismatched member is refused as for the other ensemble calls
    other = capi.GaussianProcess(capi.MATERN_NU_2P5, 1.0, [0.5] * 3, np.zeros((2, 3)) + [[0.0], [1.0]], [0.0, 1.0],
                                 [0.01])
    with pytest.raises(capi.InvalidValueError):
        capi.GaussianProcessEnsemble.from_members([ens.members[0], other]).posterior_mean(np.zeros((1, 2)))

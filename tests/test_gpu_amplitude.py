"""GPU parity at signal variances far from 1: alpha = 2^14 and 2^-14.

The SquareExponential q-KG kernels fold ln(alpha) into the exponent of every kernel value (kg.cu, kg_mc.cuh), the other
builds multiply by alpha; at alpha = 1 both are invisible.  Each case scales a unit-alpha problem exactly, with a power of
two c: alpha -> c alpha, noise -> c noise, y -> sqrt(c) y (sqrt(c) = 2^(+-7)).  K, its Cholesky factor and every
posterior quantity then scale exactly by powers of two, so the device result at c alpha is compared

* with the CPU checker, at the tolerances of the case's unit-alpha test (absolute tolerances scaled with the result), and
* with the same device call at alpha = 1 through the scale identity: mean, analytic EI, discrete-only q-KG and its
  gradient scale by sqrt(c), variance by c, the Cholesky factor of K or of the variance by sqrt(c), K^-1 (y - m) by
  1/sqrt(c); LCB selections are unchanged.  Joint posterior draws from the same normals scale by sqrt(c) and keep
  their argmins.  The random-feature weights theta are unchanged (the design matrix sqrt(2 alpha / F) cos(W x + b) /
  sqrt(noise) and y / sqrt(noise) do not move), so the sample functions' values scale by sqrt(c) and their argmins stay.
  The ensemble's discrete-only q-KG scales by sqrt(c) like the single GP's.

Three entry points are compared with the checker only, because their result is not scale-equivariant:
* full q-KG, single and ensemble: the inner descent's step is pre_mult i^-gamma times the gradient, so its path and
  end point depend on the gradient's size;
* posterior-mean optimisation: the same descent on the posterior mean;
* Monte-Carlo q-EI: the reference's q-EI is not invariant under this scaling (at c = 2^-14 its value differs from
  sqrt(c) times the unit-alpha value by ~6 %, in the checker as on the device).

Only the rounding of ln(c alpha) inside the exponent differs between the two calls, so the identity holds far tighter
than the checker tolerance: SCALE_RTOL (below) is set from the spread measured on an H100."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.stats import norm

from gpu_util import checker, tril_close
from synth import DISCRETE_ONLY_GD, EXAMPLE_INNER_GD, make_problem, unit_bounds
import rff_ref as R
from test_gpu_offset_domain import KG_CASES, KG_PATHS, kg_inputs

pytestmark = pytest.mark.gpu

AMPS = [2.0 ** 14, 2.0 ** -14]
AMP_IDS = ["2^14", "2^-14"]
KG_V, KG_G = dict(rtol=1e-7, atol=1e-10), dict(rtol=1e-5, atol=1e-8)  # tests/test_gpu_kg.py
# Scale identity: the alpha = 1 result times the exact power of two, relative to the largest entry of the result (and,
# for q-KG, at least to sqrt(c) max|y|: a discrete-only q-KG value can be 0 up to rounding).  Where alpha is a factor the
# two calls are the same arithmetic on scaled operands, and on an H100 (80 GB HBM3, 700 W) they were bit-identical for
# every posterior, fit, LCB, analytic-EI and Matern q-KG case.  Where ln(alpha) enters the exponent (SE q-KG) each
# kernel value moves by ~u |t|, u = 2^-53; the largest measured spread was 2.3e-15 (SE q-KG gradients), so the bound
# keeps a factor ~40 above it and stays 6 orders below the checker tolerance.
SCALE_RTOL = 1e-13


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def scaled(prob, c):
    out = dict(prob)
    out["alpha"] = prob["alpha"] * c
    out["noise"] = prob["noise"] * c
    out["y"] = prob["y"] * np.sqrt(c)
    return out


def device_gp(capi, kernel, prob):
    return capi.GaussianProcess(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                                prob["derivs"])


def checker_gp(kernel, prob):
    ref, lm = checker().gp(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    return ref


def close_scaled(got, base, factor, what, floor=0.0):
    """got == factor * base to SCALE_RTOL of max(largest |entry|, factor * floor); prints the measured spread."""
    got, want = np.asarray(got, dtype=np.float64), factor * np.asarray(base, dtype=np.float64)
    scale = max(np.abs(want).max(), factor * floor, 1e-300)
    dev = float(np.abs(got - want).max() / scale)
    print(f"\n  scale identity {what}: {dev:.2e}")
    assert dev <= SCALE_RTOL, (what, dev)


def tol(t, s):
    return dict(rtol=t["rtol"], atol=t["atol"] * s)


# ---- q-KG: one case per build --------------------------------------------------------------------------------------

def kg_case_inputs(case, c):
    label, kernel, N, dim, q, p, g_idx, mc, length, nf = case
    prob, cands, Xp, disc, table = kg_inputs(kernel, N, dim, q, p, g_idx, mc, length, nf, seed=900 + N + dim + q)
    best1 = 0.1 if nf else float(checker_gp(kernel, prob).mean_additional(disc).min())
    return prob, scaled(prob, c), cands, Xp, disc, table, best1


def tile_kernel_names(label, c):
    """Names of the CUDA kernels the q-KG call of case `label` at amplitude c launches (torch.profiler)."""
    import torch
    from cornell_moe_b200 import capi
    from torch.profiler import ProfilerActivity, profile
    case = next(k for k in KG_CASES if k[0] == label)
    kernel, nf = case[1], case[9]
    _, sprob, cands, Xp, disc, table, best1 = kg_case_inputs(case, c)
    gp = device_gp(capi, kernel, sprob)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gp.kg(cands, Xp, case[7], np.sqrt(c) * best1, EXAMPLE_INNER_GD, unit_bounds(case[3] - nf), disc,
              num_fidelity=nf, table=table, grad=True)
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events()})


@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("label", [k[0] for k in KG_CASES if KG_PATHS[k[0]] == "tile"])
def test_kg_amplitude_runs_the_tile_path(label, c):
    """The tile cases of test_kg_amplitude run kg_acc_tile_kernel, whose exp_tab2k rounds carry ln(alpha).  The profiler
    runs in a child process: a profiling session in this process leaves CUPTI state behind that makes the next
    sessions of the suite (tests/test_gpu_offset_domain.py) miss kernel records."""
    tests = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys, json; sys.path[:0] = [{os.path.dirname(tests)!r}, {tests!r}]; import test_gpu_amplitude as t; "
            f"print(json.dumps(t.tile_kernel_names({label!r}, {c!r})))")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().splitlines()[-1])
    assert any("kg_acc_tile_kernel" in n for n in names), names


@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("case", KG_CASES, ids=[k[0] for k in KG_CASES])
def test_kg_amplitude(capi, case, c):
    label, kernel, N, dim, q, p, g_idx, mc, length, nf = case
    prob, sprob, cands, Xp, disc, table, best1 = kg_case_inputs(case, c)
    sc = np.sqrt(c)
    bounds = unit_bounds(dim - nf)
    ref = checker_gp(kernel, sprob)
    best = sc * best1
    gp, gp1 = device_gp(capi, kernel, sprob), device_gp(capi, kernel, prob)
    # the tile cases' build is confirmed by test_kg_amplitude_runs_the_tile_path
    kg, grad = gp.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, bounds, disc, num_fidelity=nf, table=table, grad=True)
    for i in range(1 if N * dim >= 2000 else 2):
        v, g = ref.kg(cands[i], Xp, mc, best, table, EXAMPLE_INNER_GD, bounds, disc, num_fidelity=nf, grad=True)
        np.testing.assert_allclose(kg[i], v, **tol(KG_V, sc))
        np.testing.assert_allclose(grad[i], g, **tol(KG_G, sc))
    # discrete-only: the inner minimum is a posterior-mean value at a fixed point, so value and gradient scale exactly
    kd, gd = gp.kg(cands, Xp, mc, best, DISCRETE_ONLY_GD, bounds, disc, num_fidelity=nf, table=table, grad=True)
    kd1, gd1 = gp1.kg(cands, Xp, mc, best1, DISCRETE_ONLY_GD, bounds, disc, num_fidelity=nf, table=table, grad=True)
    ymax = float(np.abs(prob["y"]).max())
    close_scaled(kd, kd1, sc, f"{label} q-KG value", ymax)
    close_scaled(gd, gd1, sc, f"{label} q-KG gradient", ymax)


# ---- q-EI ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("kernel", [0, 1])
def test_qei_amplitude(capi, kernel, c):
    dim, q, p, mc = 3, 3, 1, 64
    prob = make_problem(40, dim, seed=14, noise=0.05)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    gp, ref = device_gp(capi, kernel, sprob), checker_gp(kernel, sprob)
    rng = np.random.default_rng(15)
    cands, Xp = rng.uniform(size=(2, q, dim)), rng.uniform(size=(p, dim))
    table = rng.standard_normal(mc * (q + p))
    best1 = float(prob["y"].min()) + 0.3
    ei, grad = gp.ei(cands, Xp, mc, sc * best1, table=table, grad=True)
    for i in range(2):
        v, g = ref.ei(cands[i], Xp, mc, sc * best1, table, grad=True)
        np.testing.assert_allclose(ei[i], v, rtol=1e-9, atol=1e-12 * sc)
        np.testing.assert_allclose(grad[i], g, rtol=1e-6, atol=1e-9 * sc)


@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
def test_ei_analytic_amplitude(capi, c):
    dim = 3
    prob = make_problem(40, dim, seed=16, noise=0.05)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    pts = np.random.default_rng(17).uniform(size=(20, dim))
    best1 = float(prob["y"].min()) + 0.3
    v, g = capi.ei_analytic(device_gp(capi, 0, sprob), pts, sc * best1, grad=True)
    v1, g1 = capi.ei_analytic(device_gp(capi, 0, prob), pts, best1, grad=True)
    ref = checker_gp(0, sprob)
    for i in range(3):  # closed form on the checker's posterior
        r = ref.posterior(pts[i:i + 1], (), ("mean", "var"))
        mu, sd = float(np.ravel(r["mean"])[0]), float(np.sqrt(np.ravel(r["var"])[0]))
        z = (sc * best1 - mu) / sd
        np.testing.assert_allclose(v[i], (sc * best1 - mu) * norm.cdf(z) + sd * norm.pdf(z), rtol=1e-9,
                                   atol=1e-12 * sc)
    close_scaled(v, v1, sc, "analytic EI")
    close_scaled(g, g1, sc, "analytic EI gradient")


# ---- posterior and fit ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("kernel", [0, 1])
def test_posterior_amplitude(capi, kernel, c):
    """mean, variance, its Cholesky factor and their gradients (tolerances of tests/test_gpu_posterior_ei.py)."""
    dim = 4
    prob = make_problem(60, dim, g_idx=(1,), seed=12, noise=0.05)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    gp, gp1, ref = device_gp(capi, kernel, sprob), device_gp(capi, kernel, prob), checker_gp(kernel, sprob)
    sets = np.random.default_rng(13).uniform(size=(3, 3, dim))
    want = ("mean", "grad_mean", "var", "chol_var", "grad_var", "grad_chol")
    out, out1 = gp.posterior(sets, (1,), want), gp1.posterior(sets, (1,), want)
    Q = 6
    for s in range(3):
        r = ref.posterior(sets[s], (1,), want)
        np.testing.assert_allclose(out["mean"][s], r["mean"], rtol=1e-9, atol=1e-10 * sc)
        np.testing.assert_allclose(out["grad_mean"][s], r["grad_mean"], rtol=1e-8, atol=1e-9 * sc)
        tril_close(out["var"][s].reshape(Q, Q).T, r["var"].reshape(Q, Q).T, rtol=1e-8, atol=1e-10 * c)
        tril_close(out["chol_var"][s].reshape(Q, Q).T, r["chol_var"].reshape(Q, Q).T, rtol=1e-7, atol=1e-9 * sc)
        np.testing.assert_allclose(out["grad_var"][s], r["grad_var"], rtol=1e-7, atol=1e-8 * c)
        np.testing.assert_allclose(out["grad_chol"][s], r["grad_chol"], rtol=1e-6, atol=1e-7 * sc)
    for key, f in (("mean", sc), ("grad_mean", sc), ("var", c), ("chol_var", sc), ("grad_var", c), ("grad_chol", sc)):
        close_scaled(out[key], out1[key], f, key)


# (label, N, dim, derivative indices, cov_tma): the g = 0 build, the TMA build, the derivative build, and the
# cooperative factorisation (n >= 1024)
FIT_CASES = [("g0", 200, 5, (), 0), ("tma", 300, 5, (), 1), ("deriv", 60, 4, (0, 2), 0), ("coop", 1100, 6, (), 0)]


@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("fit", FIT_CASES, ids=[f[0] for f in FIT_CASES])
def test_fit_amplitude(capi, fit, kernel, c):
    """The Cholesky factor of K and K^-1 (y - m) (tolerances of tests/test_gpu_gp.py)."""
    label, N, dim, g_idx, tma = fit
    prob = make_problem(N, dim, g_idx=g_idx, seed=40 + N, noise=0.05)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    capi.set_option("cov_tma", tma)
    try:
        gp, gp1 = device_gp(capi, kernel, sprob), device_gp(capi, kernel, prob)
    finally:
        capi.set_option("cov_tma", 0)
    L, kinvy, mean = gp.state()
    L1, kinvy1, mean1 = gp1.state()
    Lr, kr, mr = checker_gp(kernel, sprob).state()
    assert mean == mr
    tril_close(L, Lr, rtol=1e-9, atol=1e-11 * sc)
    np.testing.assert_allclose(kinvy, kr, rtol=1e-7, atol=1e-8 / sc)
    close_scaled(np.tril(L), np.tril(L1), sc, f"{label} Cholesky factor")
    close_scaled(kinvy, kinvy1, 1 / sc, f"{label} K^-1 (y - m)")


# ---- LCB -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("kernel", [0, 1])
def test_lcb_amplitude(capi, kernel, c):
    """cmoe_lcb_select: selections, mean and sd (tests/test_gpu_lcb.py) against the checker loop and the alpha = 1 call."""
    import lcb_ref
    dim, q = 3, 4
    prob = make_problem(30, dim, seed=21, noise=0.05)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    cand = np.random.default_rng(22).uniform(size=(64, dim))
    idx, mean, sd = device_gp(capi, kernel, sprob).lower_confidence_bound(cand, q)
    idx1, mean1, sd1 = device_gp(capi, kernel, prob).lower_confidence_bound(cand, q)
    r = lcb_ref.reference_loop(checker(), kernel, sprob["alpha"], sprob["lengths"], sprob["X"], sprob["y"],
                               sprob["noise"], sprob["derivs"], cand, q)
    np.testing.assert_array_equal(idx, r["selected"])
    np.testing.assert_allclose(mean, r["mean"], rtol=1e-10, atol=1e-13 * sc)
    np.testing.assert_allclose(sd, r["sd"], rtol=1e-10)
    np.testing.assert_array_equal(idx, idx1)
    close_scaled(mean, mean1, sc, "LCB mean")
    close_scaled(sd, sd1, sc, "LCB sd")


# ---- joint sampling ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("kernel", [0, 1])
def test_sample_joint_amplitude(capi, kernel, c):
    """cmoe_gp_sample_joint from a normals table: mean and factor against the checker's posterior (the 1e-10 norm bounds
    of tests/test_gpu_sampling.py), the draw against mean + L z, and every output against the alpha = 1 call."""
    dim, Q = 4, 40
    prob = make_problem(60, dim, seed=61, noise=0.05)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    rng = np.random.default_rng(62)
    sets = rng.uniform(size=(2, Q, dim))
    z = rng.standard_normal((2, Q))
    want = ("samples", "argmin", "mean", "chol")
    out = device_gp(capi, kernel, sprob).sample_joint(sets, table=z, want=want)
    out1 = device_gp(capi, kernel, prob).sample_joint(sets, table=z, want=want)
    ref = checker_gp(kernel, sprob)
    for s in range(2):
        post = ref.posterior(sets[s], want=("mean", "chol_var"))
        L_ref = np.tril(post["chol_var"].reshape(Q, Q).T)
        assert np.linalg.norm(out["chol"][s] - L_ref) <= 1e-10 * np.linalg.norm(L_ref)
        assert np.linalg.norm(out["mean"][s] - post["mean"]) <= 1e-10 * np.linalg.norm(post["mean"])
        draw = post["mean"] + L_ref @ z[s]
        assert np.linalg.norm(out["samples"][s] - draw) <= 1e-10 * np.linalg.norm(draw)
    np.testing.assert_array_equal(out["argmin"], out1["argmin"])
    for key in ("samples", "mean", "chol"):
        close_scaled(out[key], out1[key], sc, f"joint {key}")


# ---- random-feature sample functions and their optima --------------------------------------------------------------

@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("N", [30, 80], ids=["pathwise", "cholesky"])
def test_rff_amplitude(capi, N, c):
    """cmoe_gp_sample_rff_optima_ex and cmoe_gp_sample_rff_functions from a table, on both posterior branches (M < F:
    pathwise; M >= F: Cholesky).  theta against the NumPy restatement (tests/rff_ref.py, the 1e-10 of tests/test_gpu_rff.py
    at this noise), the optima values against the restatement's f; theta, omega, b and the argmins equal to the alpha = 1
    call's, values scaled by sqrt(c)."""
    dim, F, P = 3, 64, 3
    prob = make_problem(N, dim, seed=71, noise=0.05)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    rng = np.random.default_rng(72)
    M = N
    tab = {"omega": rng.standard_normal((P, F, dim)), "b": rng.uniform(0, 2 * np.pi, (P, F)),
           "z": rng.standard_normal((P, F)), "eps": rng.standard_normal((P, M))}
    bounds = unit_bounds(dim)
    grid = rng.uniform(size=(200, dim))
    gp, gp1 = device_gp(capi, 0, sprob), device_gp(capi, 0, prob)
    pts, vals, fun = gp.sample_rff_optima(F, P, bounds, grid, table=tab, return_functions=True)
    pts1, vals1, fun1 = gp1.sample_rff_optima(F, P, bounds, grid, table=tab, return_functions=True)
    for s in range(P):
        Phi, yp, W, cc = R.design(sprob["X"], sprob["y"].reshape(N, 1), sprob["noise"], [], sprob["alpha"],
                                  sprob["lengths"], tab["omega"][s], tab["b"][s])
        th = R.theta(Phi, yp, tab["z"][s], tab["eps"][s])
        np.testing.assert_allclose(fun["theta"][s], th, rtol=1e-10, atol=1e-10 * np.abs(th).max())
        want = R.f_value(pts[s], W, tab["b"][s], fun["theta"][s], cc)
        np.testing.assert_allclose(vals[s], want[0], rtol=1e-10, atol=1e-12 * sc)
    for key in ("omega", "b", "theta"):
        np.testing.assert_array_equal(fun[key], fun1[key])
    np.testing.assert_array_equal(pts, pts1)
    close_scaled(vals, vals1, sc, "rff optima values")
    x = rng.uniform(size=(50, dim))
    f, f1 = gp.sample_rff_functions(F, P, table=tab), gp1.sample_rff_functions(F, P, table=tab)
    np.testing.assert_array_equal(f.theta, f1.theta)
    (v, g), (v1, g1) = f(x, gradient=True), f1(x, gradient=True)
    close_scaled(v, v1, sc, "rff function values")
    close_scaled(g, g1, sc, "rff function gradients")


# ---- posterior-mean optimisation -----------------------------------------------------------------------------------

@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
@pytest.mark.parametrize("kernel", [0, 1])
def test_posterior_mean_optimization_amplitude(capi, kernel, c):
    """Against the checker at the tolerances of tests/test_gpu_mcmc.py::test_posterior_mean_optimization (end point to
    1e-7: the descent stops on a 1e-8 step tolerance).  No scale identity: the step is proportional to the gradient."""
    dim = 3
    prob = make_problem(40, dim, seed=3)
    sprob, sc = scaled(prob, c), np.sqrt(c)
    gp, ref = device_gp(capi, kernel, sprob), checker_gp(kernel, sprob)
    gd = [1, 50, 3, 0, 0.7, 1.0, 0.2, 1e-8]
    for x0 in ([0.3, 0.6, 0.5], [0.9, 0.1, 0.2]):
        b, v, found = capi.posterior_mean_optimization(gp, x0, gd, unit_bounds(dim))
        br, vr = ref.posterior_mean_optimization(np.array(x0), gd, unit_bounds(dim))
        assert found
        np.testing.assert_allclose(b, br, rtol=1e-7, atol=1e-7)
        np.testing.assert_allclose(v, vr, rtol=1e-9, atol=1e-12 * sc)


# ---- ensemble q-KG -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c", AMPS, ids=AMP_IDS)
def test_kg_mcmc_amplitude(capi, c):
    """cmoe_kg_eval_mcmc over 3 Matern-5/2 members with every member's alpha and noise scaled: full q-KG against the
    checker's member average (tolerances of tests/test_gpu_mcmc.py), discrete-only q-KG against the alpha = 1 call."""
    M, dim, q, p, mc = 3, 3, 2, 1, 16
    prob = make_problem(30, dim, seed=31, noise=0.1)
    rng = np.random.default_rng(5)
    hypers = np.concatenate([rng.uniform(0.8, 1.5, size=(M, 1)), rng.uniform(0.4, 0.9, size=(M, dim))], axis=1)
    noises = rng.uniform(0.05, 0.15, size=(M, 1))
    shypers, snoises, sy, sc = hypers.copy(), noises * c, prob["y"] * np.sqrt(c), np.sqrt(c)
    shypers[:, 0] *= c
    rng = np.random.default_rng(6)
    Xq, Xp = rng.uniform(size=(q, dim)), rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, 4, dim))
    best1 = rng.uniform(-0.5, 0.5, size=M)
    table = rng.standard_normal((mc // 2) * (q + p))
    bounds = unit_bounds(dim)
    vr, gr = checker().kg_mcmc(shypers, snoises, prob["X"], sy, prob["derivs"], Xq, Xp, mc, sc * best1, table,
                               EXAMPLE_INNER_GD, bounds, disc, grad=True)
    ens = capi.GaussianProcessEnsemble(shypers, snoises, prob["X"], sy, prob["derivs"])
    ens1 = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"])
    v, g = ens.kg(Xq, Xp, mc, sc * best1, EXAMPLE_INNER_GD, bounds, disc, table=table, grad=True)
    np.testing.assert_allclose(v[0], vr, **tol(KG_V, sc))
    np.testing.assert_allclose(g[0], gr, **tol(KG_G, sc))
    vd, gd = ens.kg(Xq, Xp, mc, sc * best1, DISCRETE_ONLY_GD, bounds, disc, table=table, grad=True)
    vd1, gd1 = ens1.kg(Xq, Xp, mc, best1, DISCRETE_ONLY_GD, bounds, disc, table=table, grad=True)
    ymax = float(np.abs(prob["y"]).max())
    close_scaled(vd, vd1, sc, "ensemble q-KG value", ymax)
    close_scaled(gd, gd1, sc, "ensemble q-KG gradient", ymax)

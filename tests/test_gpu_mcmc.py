"""GPU parity tests of the widened rows (SURVEY.md 8f): MCMC-averaged q-KG / q-EI over an ensemble of GPs, and
posterior_mean_optimization — all through the C ABI, checked against the compiled reference (or the pinned C oracle)."""
import os
import sys

import numpy as np
import pytest

import oracle as orc
from gpu_util import checker
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def _ensemble_inputs(M, dim, g, seed):
    rng = np.random.default_rng(seed)
    hypers = np.concatenate([rng.uniform(0.8, 1.5, size=(M, 1)), rng.uniform(0.4, 0.9, size=(M, dim))], axis=1)
    noises = rng.uniform(0.05, 0.15, size=(M, 1 + g))
    return hypers, noises


@pytest.mark.parametrize("q,p,g_idx,nf", [(1, 0, (), 0), (2, 1, (), 0), (2, 0, (0,), 0), (1, 0, (), 1), (2, 1, (), 1)])
def test_kg_mcmc_table_fed(capi, q, p, g_idx, nf):
    M, dim, mc, num_pts = 3, 3, 8, 4
    prob = make_problem(12, dim, g_idx=g_idx, seed=31, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, len(g_idx), 5)
    rng = np.random.default_rng(6)
    Xq, Xp = rng.uniform(0.2, 0.9, size=(q, dim)), rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, num_pts, dim - nf))
    best = rng.uniform(-0.5, 0.5, size=M)
    table = rng.standard_normal((mc // 2) * (q + p) * (1 + len(g_idx)))
    vr, gr = checker().kg_mcmc(hypers, noises, prob["X"], prob["y"], prob["derivs"], Xq, Xp, mc, best, table,
                               EXAMPLE_INNER_GD, unit_bounds(dim - nf), disc, num_fidelity=nf, grad=True)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"])
    v, g = ens.kg(Xq, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim - nf), disc, num_fidelity=nf, table=table,
                  grad=True)
    np.testing.assert_allclose(v[0], vr, rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(g[0], gr, rtol=1e-5, atol=1e-8)
    # the value-only call and the Philox-fed call agree with the table that holds the same stream
    np.testing.assert_allclose(ens.kg(Xq, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim - nf), disc, num_fidelity=nf,
                                      table=table), v, rtol=1e-12)
    t2 = orc.philox_normals(41, 0, mc // 2, (q + p) * (1 + len(g_idx)))
    a = ens.kg(Xq, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim - nf), disc, num_fidelity=nf, seed=41)
    b = ens.kg(Xq, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim - nf), disc, num_fidelity=nf, table=t2)
    np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("q,p", [(1, 0), (3, 2)])
def test_ei_mcmc_table_fed(capi, q, p):
    M, dim, mc = 4, 3, 16
    prob = make_problem(15, dim, seed=32, noise=0.05)
    hypers, noises = _ensemble_inputs(M, dim, 0, 7)
    rng = np.random.default_rng(8)
    Xq, Xp = rng.uniform(size=(q, dim)), rng.uniform(size=(p, dim))
    best = rng.uniform(0.5, 1.5, size=M)
    table = rng.standard_normal(mc * (q + p))
    vr, gr = checker().ei_mcmc(hypers, noises, prob["X"], prob["y"], prob["derivs"], Xq, Xp, mc, best, table, grad=True)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    v, g = ens.ei(Xq, Xp, mc, best, table=table, grad=True)
    np.testing.assert_allclose(v[0], vr, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(g[0], gr, rtol=1e-7, atol=1e-10)
    if q == 1 and p == 0:
        # analytic_single = mean of the members' closed-form 1-EI
        a = ens.ei(Xq, Xp, mc, best, analytic_single=True)
        want = np.mean([capi.ei_analytic(m, Xq, b) for m, b in zip(ens.members, best)])
        np.testing.assert_allclose(a[0], want, rtol=1e-13)


def test_multistart_mcmc_drivers(capi):
    M, dim, q, mc = 3, 2, 2, 32
    prob = make_problem(25, dim, seed=12, noise=0.05)
    hypers, noises = _ensemble_inputs(M, dim, 0, 3)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    rng = np.random.default_rng(14)
    starts = rng.uniform(size=(30, q, dim))
    disc = rng.uniform(size=(M, 6, dim))
    best = np.array([float(m.posterior(disc[i][:, None, :], (), ("mean",))["mean"].min())
                     for i, m in enumerate(ens.members)])
    outer = [30, 3, 1, 0, 0.7, 0.3, 0.2, 1e-7]
    bp, bv, found, sv = ens.multistart_kg(starts, None, mc, best, outer, EXAMPLE_INNER_GD, unit_bounds(dim),
                                          unit_bounds(dim), disc, seed=5)
    assert found and np.isfinite(bv) and np.all(bp >= 0.0) and np.all(bp <= 1.0)
    # the screening values are the ensemble evaluation, which is the mean of the members' q-KG
    np.testing.assert_array_equal(sv, ens.kg(starts, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, seed=5))
    per = np.mean([m.kg(starts, None, mc, best[i], EXAMPLE_INNER_GD, unit_bounds(dim), disc[i], seed=5)
                   for i, m in enumerate(ens.members)], axis=0)
    np.testing.assert_allclose(sv, per, rtol=1e-12, atol=1e-14)
    # one outer step from a single start reproduces the reference's update rule on the averaged gradient
    one = [1, 1, 1, 0, 0.7, 0.3, 0.2, 1e-7]
    bp1, bv1, _, _ = ens.multistart_kg(starts[:1], None, mc, best, one, EXAMPLE_INNER_GD, unit_bounds(dim),
                                       unit_bounds(dim), disc, seed=5)
    _, g = ens.kg(starts[:1], None, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, seed=5, grad=True)
    backend = checker()
    want = starts[0].copy()
    step = 0.3 * g[0]
    for k in range(q):
        step[k] = backend.limit_update(unit_bounds(dim), 0.2, starts[0][k], step[k])
    want += step
    v_want = ens.kg(want, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, seed=5)[0]
    if v_want > -np.inf:
        np.testing.assert_allclose(bp1, want, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(bv1, v_want, rtol=1e-12)
    # EI drivers: MC for q = 2 and analytic for q = 1
    ybest = np.full(M, float(prob["y"].min()))
    for qq in (1, 2):
        st = rng.uniform(size=(25, qq, dim))
        bp, bv, found, sv = ens.multistart_ei(st, None, 256, ybest, [25, 4, 2, 0, 0.7, 0.2, 0.2, 1e-8],
                                              unit_bounds(dim), seed=3)
        assert np.all(bp >= 0.0) and np.all(bp <= 1.0) and bv >= 0.0
        np.testing.assert_array_equal(sv, ens.ei(st, None, 256, ybest, seed=3, analytic_single=True))


@pytest.mark.parametrize("kernel,g_idx,nf", [(0, (), 0), (1, (0, 2), 0), (1, (), 1), (0, (), 2)])
def test_posterior_mean_optimization(capi, kernel, g_idx, nf):
    dim = 4 if nf == 2 else 3
    prob = make_problem(40, dim, g_idx=g_idx, seed=3)
    gp = capi.GaussianProcess(kernel, 1.0, prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    ref, _ = checker().gp(kernel, 1.0, prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    gd = [1, 50, 3, 0, 0.7, 1.0, 0.2, 1e-8]
    for x0 in ([0.3, 0.6, 0.5, 0.4][: dim - nf], [0.9, 0.1, 0.2, 0.7][: dim - nf]):
        b, v, found = capi.posterior_mean_optimization(gp, x0, gd, unit_bounds(dim - nf), nf)
        br, vr = ref.posterior_mean_optimization(np.array(x0), gd, unit_bounds(dim - nf), nf)
        assert found
        # the descent stops once a step is shorter than its 1e-8 tolerance: the end point is defined to ~1e-8 only, and
        # which iteration stops it depends on last-bit differences of K^-1 y (seen when the covariance build moved to
        # centred coordinates: 1.6e-8 on one coordinate); the value at the optimum is flat there and keeps its 1e-9
        np.testing.assert_allclose(b, br, rtol=1e-7, atol=1e-7)
        np.testing.assert_allclose(v, vr, rtol=1e-9)
    # max_num_restarts = 0: the reference returns without touching its outputs
    b, v, found = capi.posterior_mean_optimization(gp, x0, [1, 50, 0, 0, 0.7, 1.0, 0.2, 1e-8], unit_bounds(dim - nf), nf)
    assert not found


def test_gpp_mcmc_surface(capi):
    sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
    import GPP as C_GP
    M, dim, q, mc, num_pts = 3, 3, 2, 16, 4
    prob = make_problem(18, dim, seed=44, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, 0, 2)
    gpm = C_GP.GaussianProcessMCMC(list(hypers.ravel()), list(noises.ravel()), list(prob["X"].ravel()),
                                   list(prob["y"]), [], M, 0, dim, 18)
    assert gpm.num_mcmc == M and gpm.dim == dim
    rnd = C_GP.RandomnessSourceContainer(2)
    rnd.SetExplicitNormalRNGSeed(99)
    rng = np.random.default_rng(3)
    Xq = rng.uniform(size=(q, dim))
    disc = rng.uniform(size=(M, num_pts, dim))
    best = list(rng.uniform(-0.3, 0.3, size=M))

    class Inner:
        domain_type = C_GP.DomainTypes.tensor_product
        optimizer_type = C_GP.OptimizerTypes.gradient_descent
        num_random_samples = 12
        optimizer_parameters = C_GP.GradientDescentParameters(*EXAMPLE_INNER_GD)

    kg = C_GP.compute_knowledge_gradient_mcmc(gpm, 0, Inner, list(unit_bounds(dim)), list(disc.ravel()), list(Xq.ravel()),
                                              [], num_pts, q, 0, mc, best, rnd)
    gkg = C_GP.compute_grad_knowledge_gradient_mcmc(gpm, 0, Inner, list(unit_bounds(dim)), list(disc.ravel()),
                                                    list(Xq.ravel()), [], num_pts, q, 0, mc, best, rnd)
    table = orc.philox_normals(99, 0, mc // 2, q)
    vr, gr = checker().kg_mcmc(hypers, noises, prob["X"], prob["y"], None, Xq, None, mc, best, table, EXAMPLE_INNER_GD,
                               unit_bounds(dim), disc, grad=True)
    np.testing.assert_allclose(kg, vr, rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(np.array(gkg).reshape(q, dim), gr, rtol=1e-5, atol=1e-8)
    ei = C_GP.compute_expected_improvement_mcmc(gpm, list(Xq.ravel()), [], q, 0, mc, best, rnd)
    gei = C_GP.compute_grad_expected_improvement_mcmc(gpm, list(Xq.ravel()), [], q, 0, mc, best, rnd)
    t2 = orc.philox_normals(99, 0, mc, q)
    er, ger = checker().ei_mcmc(hypers, noises, prob["X"], prob["y"], None, Xq, None, mc, best, t2, grad=True)
    np.testing.assert_allclose(ei, er, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(np.array(gei).reshape(q, dim), ger, rtol=1e-7, atol=1e-10)
    status = {}
    outer = type("P", (), dict(domain_type=C_GP.DomainTypes.tensor_product,
                               optimizer_type=C_GP.OptimizerTypes.gradient_descent, num_random_samples=12,
                               optimizer_parameters=C_GP.GradientDescentParameters(22, 2, 1, 0, 0.7, 0.3, 0.2, 1e-7)))
    pts = C_GP.multistart_knowledge_gradient_mcmc_optimization(outer, Inner, gpm, 0, list(unit_bounds(dim)),
                                                               list(disc.ravel()), [], num_pts, q, 0, best, mc, 2, rnd,
                                                               status)
    assert status["gradient_descent_tensor_product_domain_found_update"] is True
    assert len(pts) == q * dim and all(0.0 <= x <= 1.0 for x in pts)
    null = type("P", (), dict(domain_type=C_GP.DomainTypes.tensor_product, optimizer_type=C_GP.OptimizerTypes.null,
                              num_random_samples=12, optimizer_parameters=None))
    pts = C_GP.multistart_expected_improvement_mcmc_optimization(null, gpm, list(unit_bounds(dim)), [], q, 0, best, mc,
                                                                 2, rnd, status)
    assert "lhc_tensor_product_domain_found_update" in status and len(pts) == q * dim
    pts = C_GP.multistart_expected_improvement_mcmc_optimization(outer, gpm, list(unit_bounds(dim)), [], 1, 0, best, mc,
                                                                 2, rnd, status)
    assert len(pts) == dim
    vals = C_GP.evaluate_KG_mcmc_at_point_list(gpm, 0, Inner, list(unit_bounds(dim)), list(Xq.ravel()),
                                               list(disc.ravel()), 1, num_pts, q, 0, best, mc, 2, rnd, status)
    np.testing.assert_allclose(vals[0], kg, rtol=0, atol=0)
    vals = C_GP.evaluate_EI_mcmc_at_point_list(gpm, list(Xq.ravel()), [], 1, q, 0, best, mc, 2, rnd, status)
    np.testing.assert_allclose(vals[0], ei, rtol=0, atol=0)
    with pytest.raises(C_GP.BoundsException):
        C_GP.evaluate_EI_mcmc_at_point_list(gpm, list(Xq.ravel()), [], 1, q, 0, best, mc, 3, rnd, status)
    # posterior_mean_optimization on one member GP through the module
    gp = C_GP.GaussianProcess([1.0, list(prob["lengths"])], list(prob["X"].ravel()), list(prob["y"]),
                              list(prob["noise"]), [], 0, dim, 18)
    ref, _ = checker().gp(1, 1.0, prob["lengths"], prob["X"], prob["y"], prob["noise"])
    sgd = type("P", (), dict(optimizer_parameters=C_GP.GradientDescentParameters(1, 40, 2, 0, 0.7, 1.0, 0.2, 1e-8)))
    got = C_GP.posterior_mean_optimization(gp, 0, sgd, list(unit_bounds(dim)), [0.4, 0.5, 0.6], status)
    want, _ = ref.posterior_mean_optimization(np.array([0.4, 0.5, 0.6]), [1, 40, 2, 0, 0.7, 1.0, 0.2, 1e-8],
                                              unit_bounds(dim), 0)
    np.testing.assert_allclose(got, want, rtol=1e-7, atol=1e-9)

"""GPU parity on domains far from the origin.  Every device entry point is compared with the CPU checker (which forms
coordinate differences first) at the tolerances of its unit-box test, and with its own result on the unshifted problem
(the kernels are translation invariant).

The q-KG kernels form -r^2/2 in the expanded form x.y - |x|^2/2 - |y|^2/2, whose absolute error is about
eps (|x|^2 + |y|^2) in length-scale units; they only keep full accuracy here because their operands are taken relative to
the GP's centre.  One case per build of the q-KG path (kg_select): the small fast-path instantiation, the DMMA tile
instantiation <SE,8,8>, the global-memory body, Matern-5/2, the general and the wide derivative paths, a fidelity
coordinate, both sides of the fast path's radius and a plan that re-selects its path per upload.  Which case lands on
which path is restated on the host in tests/test_offset_domain_cpu.py, together with a check that these inputs do lose
digits in the expanded form."""
import numpy as np
import pytest

from gpu_util import checker, tril_close
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

pytestmark = pytest.mark.gpu

KG_V, KG_G = dict(rtol=1e-7, atol=1e-10), dict(rtol=1e-5, atol=1e-8)  # tests/test_gpu_kg.py, table-fed


def offset(dim, free=None):
    """c_d = (-1)^d 1000 (1 + d/10): both signs and a different size per axis, so that no cancellation is shared by all
    axes; fidelity coordinates (d >= free) stay put, they enter the cost, which does not translate."""
    c = np.array([(-1.0) ** d * 1000.0 * (1.0 + 0.1 * d) for d in range(dim)])
    if free is not None:
        c[free:] = 0.0
    return c


# (label, kernel, N, dim, q, p, derivative indices, num_mc, length scale or None (make_problem's), fidelity coords)
KG_CASES = [
    ("fast_small", 0, 60, 3, 2, 1, (), 64, None, 0),
    ("tile", 0, 300, 8, 8, 0, (), 100, None, 0),
    ("tile_padded", 0, 300, 7, 5, 2, (), 70, None, 0),
    ("global", 0, 1500, 8, 8, 0, (), 32, None, 0),
    ("matern", 1, 200, 6, 4, 0, (), 64, None, 0),
    ("general_se", 0, 40, 4, 2, 0, (0, 2), 32, None, 0),
    ("general_matern", 1, 40, 4, 2, 0, (0, 2), 32, None, 0),
    ("wide", 0, 12, 10, 1, 0, tuple(range(10)), 32, None, 0),
    ("fidelity", 0, 40, 3, 2, 0, (), 32, None, 1),
]
# expected build per label (tests/test_offset_domain_cpu.py restates the host's rule)
KG_PATHS = {"fast_small": "fast", "tile": "tile", "tile_padded": "tile", "global": "global", "matern": "fast",
            "general_se": "general", "general_matern": "general", "wide": "wide", "fidelity": "fast"}


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def kg_inputs(kernel, N, dim, q, p, g_idx, mc, length, nf, seed):
    """Unshifted problem and evaluation inputs (unit box); the caller adds the offset."""
    prob = make_problem(N, dim, g_idx=g_idx, seed=seed, noise=0.05)
    if length is not None:
        prob["lengths"] = np.full(dim, length)
    rng = np.random.default_rng(seed + 1)
    ps = dim - nf
    cands = rng.uniform(size=(2, q, dim))
    Xp = rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(6, ps))
    Q = (q + p) * (1 + len(g_idx))
    table = rng.standard_normal((mc // 2) * Q)
    return prob, cands, Xp, disc, table


def shifted(prob, c):
    out = dict(prob)
    out["X"] = prob["X"] + c  # unit scale: derivative observations stay consistent
    return out


def device_gp(capi, kernel, prob):
    return capi.GaussianProcess(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                                prob["derivs"])


def checker_gp(kernel, prob):
    ref, lm = checker().gp(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    return ref


def kg_pair(capi, case, with_profile=False):
    """(device value, device grad, checker values, checker grads, device value/grad of the unshifted problem, kernels
    that ran on the shifted call)."""
    label, kernel, N, dim, q, p, g_idx, mc, length, nf = case
    prob, cands, Xp, disc, table = kg_inputs(kernel, N, dim, q, p, g_idx, mc, length, nf, seed=500 + N + dim + q)
    ps = dim - nf
    c = offset(dim, ps)
    ps_c = c[:ps]
    sprob = shifted(prob, c)
    ref = checker_gp(kernel, sprob)
    best = 0.1 if nf else float(ref.mean_additional(disc + ps_c).min())
    bounds = unit_bounds(ps)
    sbounds = bounds + np.repeat(ps_c, 2)
    gp_s = device_gp(capi, kernel, sprob)
    args_s = (cands + c, Xp + c, mc, best, EXAMPLE_INNER_GD, sbounds, disc + ps_c)
    names = set()
    if with_profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            kg_s, grad_s = gp_s.kg(*args_s, num_fidelity=nf, table=table, grad=True)
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
    else:
        kg_s, grad_s = gp_s.kg(*args_s, num_fidelity=nf, table=table, grad=True)
    gp_0 = device_gp(capi, kernel, prob)
    kg_0, grad_0 = gp_0.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, bounds, disc, num_fidelity=nf, table=table, grad=True)
    # the checker at full size is the slow part: one candidate on the largest shapes
    ncheck = 1 if N * dim >= 2000 else 2
    vr, gr = [], []
    for i in range(ncheck):
        v, g = ref.kg(cands[i] + c, Xp + c, mc, best, table, EXAMPLE_INNER_GD, sbounds, disc + ps_c, num_fidelity=nf,
                      grad=True)
        vr.append(v)
        gr.append(g)
    return kg_s, grad_s, vr, gr, kg_0, grad_0, names


@pytest.mark.parametrize("case", KG_CASES, ids=[c[0] for c in KG_CASES])
def test_kg_offset_domain(capi, case):
    tile = KG_PATHS[case[0]] == "tile"
    kg_s, grad_s, vr, gr, kg_0, grad_0, names = kg_pair(capi, case, with_profile=tile)
    for i in range(len(vr)):
        np.testing.assert_allclose(kg_s[i], vr[i], **KG_V)
        np.testing.assert_allclose(grad_s[i], gr[i], **KG_G)
    np.testing.assert_allclose(kg_s, kg_0, **KG_V)
    np.testing.assert_allclose(grad_s, grad_0, **KG_G)
    if tile:
        # the tile accumulation only runs on the tile instantiation's shared-memory fast path
        assert any("kg_acc_tile_kernel" in n for n in names), sorted(names)


def radius_case(target):
    """Tile instantiation (d = 8, q + p = 5 -> QP = 8) with a length scale that puts the largest centred scaled radius the
    host checks (training, discrete, pending points, inner-domain corners, candidates) at `target` length scales."""
    dim, N, q, mc = 8, 40, 5, 32
    prob, cands, Xp, disc, table = kg_inputs(0, N, dim, q, 0, (), mc, None, 0, seed=77)
    c = offset(dim)
    centre = prob["X"].mean(axis=0)
    corners = np.maximum(np.abs(0.0 - centre), np.abs(1.0 - centre))
    pts = np.concatenate([prob["X"], disc, cands.reshape(-1, dim)])
    r1 = max(np.sqrt((corners ** 2).sum()), np.sqrt(((pts - centre) ** 2).sum(axis=1)).max())
    prob["lengths"] = np.full(dim, r1 / target)
    return prob, cands, disc, table, c, mc


@pytest.mark.parametrize("side,target", [("fast", 1990.0), ("guarded", 2010.0)])
def test_kg_offset_radius_edge(capi, side, target):
    """Just inside and just outside kFastPathRadius = 2000, measured in the centred frame.  Inside, the table exps and
    the tile path run (kg_acc_tile_kernel); outside, the guarded build (kg_acc_kernel).  Both match the checker."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    prob, cands, disc, table, c, mc = radius_case(target)
    sprob = shifted(prob, c)
    ref = checker_gp(0, sprob)
    best = float(ref.mean_additional(disc + c).min())
    sb = unit_bounds(8) + np.repeat(c, 2)
    gp = device_gp(capi, 0, sprob)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        kg, grad = gp.kg(cands + c, None, mc, best, EXAMPLE_INNER_GD, sb, disc + c, table=table, grad=True)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    assert any("kg_acc_tile_kernel" in n for n in names) == (side == "fast"), sorted(names)
    for i in range(2):
        v, g = ref.kg(cands[i] + c, None, mc, best, table, EXAMPLE_INNER_GD, sb, disc + c, grad=True)
        np.testing.assert_allclose(kg[i], v, **KG_V)
        np.testing.assert_allclose(grad[i], g, **KG_G)
    kg0, grad0 = device_gp(capi, 0, prob).kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(8), disc, table=table,
                                             grad=True)
    np.testing.assert_allclose(kg, kg0, **KG_V)
    np.testing.assert_allclose(grad, grad0, **KG_G)


def test_kg_plan_reselects_path_per_upload(capi):
    """One plan, three uploads: candidates inside the fast path's radius, then a batch with a candidate ~2200 length
    scales from the centre (guarded build), then inside again.  Each batch matches the checker."""
    dim, q, mc = 3, 2, 32
    prob, cands, _, disc, table = kg_inputs(0, 30, dim, q, 0, (), mc, None, 0, seed=88)
    c = offset(dim)
    sprob = shifted(prob, c)
    ref = checker_gp(0, sprob)
    best = float(ref.mean_additional(disc + c).min())
    sb = unit_bounds(dim) + np.repeat(c, 2)
    gp = device_gp(capi, 0, sprob)
    far = cands.copy()
    far[1, 0, 0] += 1100.0  # l = 0.5: 2200 length scales
    plan = capi.KGPlan(gp, mc, best, EXAMPLE_INNER_GD, sb, disc + c, 2, q, table=table)
    for batch in (cands, far, cands):
        plan.upload(batch + c)
        plan.run()
        plan.sync()
        kg, grad, _ = plan.download()
        for i in range(2):
            v, g = ref.kg(batch[i] + c, None, mc, best, table, EXAMPLE_INNER_GD, sb, disc + c, grad=True)
            np.testing.assert_allclose(kg[i], v, **KG_V)
            np.testing.assert_allclose(grad[i], g, **KG_G)


def _ensemble_inputs(M, dim, seed):
    rng = np.random.default_rng(seed)
    hypers = np.concatenate([rng.uniform(0.8, 1.5, size=(M, 1)), rng.uniform(0.4, 0.9, size=(M, dim))], axis=1)
    noises = rng.uniform(0.05, 0.15, size=(M, 1))
    return hypers, noises


def test_kg_mcmc_offset_domain(capi):
    """cmoe_kg_eval_mcmc over 3 members: the average of the members' checker values (tests/test_gpu_mcmc.py)."""
    M, dim, q, p, mc = 3, 3, 2, 1, 16
    prob = make_problem(30, dim, seed=31, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, 5)
    rng = np.random.default_rng(6)
    Xq, Xp = rng.uniform(size=(q, dim)), rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, 4, dim))
    best = rng.uniform(-0.5, 0.5, size=M)
    table = rng.standard_normal((mc // 2) * (q + p))
    c = offset(dim)
    vr, gr = checker().kg_mcmc(hypers, noises, prob["X"] + c, prob["y"], prob["derivs"], Xq + c, Xp + c, mc, best, table,
                               EXAMPLE_INNER_GD, unit_bounds(dim) + np.repeat(c, 2), disc + c, grad=True)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"] + c, prob["y"], prob["derivs"])
    v, g = ens.kg(Xq + c, Xp + c, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim) + np.repeat(c, 2), disc + c, table=table,
                  grad=True)
    np.testing.assert_allclose(v[0], vr, **KG_V)
    np.testing.assert_allclose(g[0], gr, **KG_G)
    ens0 = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"])
    v0, g0 = ens0.kg(Xq, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, table=table, grad=True)
    np.testing.assert_allclose(v, v0, **KG_V)
    np.testing.assert_allclose(g, g0, **KG_G)


def test_multistart_kg_offset_domain(capi):
    """cmoe_multistart_kg on the shifted problem against the unshifted one: best_point - c, best_value, found_flag."""
    dim, q, mc = 2, 2, 32
    prob = make_problem(30, dim, seed=3, noise=0.05)
    c = offset(dim)
    rng = np.random.default_rng(4)
    starts = rng.uniform(0.1, 0.9, size=(12, q, dim))
    disc = rng.uniform(size=(8, dim))
    table = rng.standard_normal((mc // 2) * q)
    outer = [12, 3, 1, 0, 0.7, 0.3, 0.2, 1e-7]
    out = []
    for shift in (np.zeros(dim), c):
        gp = device_gp(capi, 0, shifted(prob, shift))
        best = float(gp.posterior((disc + shift)[:, None, :], (), ("mean",))["mean"].min())
        b = unit_bounds(dim) + np.repeat(shift, 2)
        out.append(capi.multistart_kg(gp, starts + shift, None, mc, best, outer, EXAMPLE_INNER_GD, b, b, disc + shift,
                                      table=table))
    (bp0, bv0, f0, sv0), (bp, bv, f, sv) = out
    assert f == f0
    np.testing.assert_allclose(sv, sv0, **KG_V)
    np.testing.assert_allclose(bv, bv0, **KG_V)
    np.testing.assert_allclose(bp - c, bp0, rtol=1e-6, atol=1e-8)


# ---- difference-form entry points: regression guards ----------------------------------------------------------------

@pytest.mark.parametrize("kernel", [0, 1])
def test_posterior_offset_domain(capi, kernel):
    """mean, variance, its Cholesky factor and their gradients (tolerances of tests/test_gpu_posterior_ei.py)."""
    dim = 4
    prob = make_problem(60, dim, g_idx=(1,), seed=12, noise=0.05)
    c = offset(dim)
    sprob = shifted(prob, c)
    gp, gp0, ref = device_gp(capi, kernel, sprob), device_gp(capi, kernel, prob), checker_gp(kernel, sprob)
    sets = np.random.default_rng(13).uniform(size=(3, 3, dim))
    want = ("mean", "grad_mean", "var", "chol_var", "grad_var", "grad_chol")
    out, out0 = gp.posterior(sets + c, (1,), want), gp0.posterior(sets, (1,), want)
    Q = 6
    for s in range(3):
        r = ref.posterior(sets[s] + c, (1,), want)
        for o in (out, out0):
            np.testing.assert_allclose(o["mean"][s], r["mean"], rtol=1e-9, atol=1e-10)
            np.testing.assert_allclose(o["grad_mean"][s], r["grad_mean"], rtol=1e-8, atol=1e-9)
            tril_close(o["var"][s].reshape(Q, Q).T, r["var"].reshape(Q, Q).T, rtol=1e-8, atol=1e-10)
            tril_close(o["chol_var"][s].reshape(Q, Q).T, r["chol_var"].reshape(Q, Q).T, rtol=1e-7, atol=1e-9)
            np.testing.assert_allclose(o["grad_var"][s], r["grad_var"], rtol=1e-7, atol=1e-8)
            np.testing.assert_allclose(o["grad_chol"][s], r["grad_chol"], rtol=1e-6, atol=1e-7)


def test_qei_offset_domain(capi):
    dim, q, p, mc = 3, 3, 1, 64
    prob = make_problem(40, dim, seed=14, noise=0.05)
    c = offset(dim)
    sprob = shifted(prob, c)
    gp, gp0, ref = device_gp(capi, 0, sprob), device_gp(capi, 0, prob), checker_gp(0, sprob)
    rng = np.random.default_rng(15)
    cands, Xp = rng.uniform(size=(2, q, dim)), rng.uniform(size=(p, dim))
    table = rng.standard_normal(mc * (q + p))
    best = float(prob["y"].min()) + 0.3
    ei, grad = gp.ei(cands + c, Xp + c, mc, best, table=table, grad=True)
    ei0, grad0 = gp0.ei(cands, Xp, mc, best, table=table, grad=True)
    for i in range(2):
        v, g = ref.ei(cands[i] + c, Xp + c, mc, best, table, grad=True)
        np.testing.assert_allclose(ei[i], v, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(grad[i], g, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(ei, ei0, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(grad, grad0, rtol=1e-6, atol=1e-9)


def test_posterior_mean_optimization_offset_domain(capi):
    dim = 3
    prob = make_problem(40, dim, seed=3)
    c = offset(dim)
    sprob = shifted(prob, c)
    gp, ref = device_gp(capi, 0, sprob), checker_gp(0, sprob)
    gd = [1, 50, 3, 0, 0.7, 1.0, 0.2, 1e-8]
    x0 = np.array([0.3, 0.6, 0.5])
    b, v, found = capi.posterior_mean_optimization(gp, x0 + c, gd, unit_bounds(dim) + np.repeat(c, 2))
    br, vr = ref.posterior_mean_optimization(x0 + c, gd, unit_bounds(dim) + np.repeat(c, 2))
    assert found
    # tests/test_gpu_mcmc.py::test_posterior_mean_optimization: the end point is defined to ~1e-8 by the step tolerance
    np.testing.assert_allclose(b - c, br - c, rtol=1e-7, atol=1e-7)
    np.testing.assert_allclose(v, vr, rtol=1e-9)
    b0, v0, _ = capi.posterior_mean_optimization(device_gp(capi, 0, prob), x0, gd, unit_bounds(dim))
    np.testing.assert_allclose(b - c, b0, rtol=1e-7, atol=1e-7)
    np.testing.assert_allclose(v, v0, rtol=1e-9)


def test_posterior_mean_optima_mcmc_offset_domain(capi):
    """cmoe_posterior_mean_optima_mcmc: against the checker restatement (tests/pm_optima_ref.py) and the unshifted call."""
    import pm_optima_ref
    M, dim, kernel = 3, 3, 1
    prob = make_problem(30, dim, seed=3, noise=0.05)
    rng = np.random.default_rng(103)
    hypers = np.concatenate([rng.uniform(0.8, 1.5, size=(M, 1)), rng.uniform(0.4, 0.9, size=(M, dim))], axis=1)
    noises = np.full((M, 1), 0.05)
    c = offset(dim)
    gd = [1, 50, 3, 0, 0.7, 1.0, 0.2, 1e-8]
    pts, shared = rng.uniform(size=(100, dim)), rng.uniform(size=(4, dim))
    res = []
    for shift in (np.zeros(dim), c):
        ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"] + shift, prob["y"], kernel=kernel)
        res.append(ens.posterior_mean_optima(pts + shift, gd, unit_bounds(dim) + np.repeat(shift, 2), 0, True,
                                             shared + shift))
    out0, out = res
    members = [checker_gp(kernel, dict(shifted(prob, c), alpha=h[0], lengths=h[1:])) for h in hypers]
    ref = pm_optima_ref.optima(members, prob["X"] + c, pts + c, gd, unit_bounds(dim) + np.repeat(c, 2), 0, True,
                               shared + c)
    # tolerances of tests/test_gpu_pm_optima.py::test_against_the_checker, on the optima relative to the offset
    for r, r_shift in ((ref, c), (out0, np.zeros(dim))):
        np.testing.assert_array_equal(out.start_index, r.start_index)
        np.testing.assert_array_equal(out.kept_start, r.kept_start)
        np.testing.assert_allclose(out.optima - c, r.optima - r_shift, rtol=1e-7, atol=1e-7)
        np.testing.assert_allclose(out.means, r.means, rtol=1e-9)
        np.testing.assert_allclose(out.best_so_far, r.best_so_far, rtol=1e-9)


def test_lcb_offset_domain(capi):
    """cmoe_lcb_select: selections, mean and sd (tests/test_gpu_lcb.py) against the checker loop and the unshifted call."""
    import lcb_ref
    dim, q = 3, 4
    prob = make_problem(30, dim, seed=21, noise=0.05)
    c = offset(dim)
    sprob = shifted(prob, c)
    cand = np.random.default_rng(22).uniform(size=(64, dim))
    idx, mean, sd = device_gp(capi, 1, sprob).lower_confidence_bound(cand + c, q)
    idx0, mean0, sd0 = device_gp(capi, 1, prob).lower_confidence_bound(cand, q)
    r = lcb_ref.reference_loop(checker(), 1, sprob["alpha"], sprob["lengths"], sprob["X"], sprob["y"], sprob["noise"],
                               sprob["derivs"], cand + c, q)
    np.testing.assert_array_equal(idx, r["selected"])
    np.testing.assert_allclose(mean, r["mean"], rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(sd, r["sd"], rtol=1e-10)
    np.testing.assert_array_equal(idx, idx0)
    np.testing.assert_allclose(mean, mean0, rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(sd, sd0, rtol=1e-10)


@pytest.mark.parametrize("kernel", [0, 1])
def test_log_marginal_likelihood_offset_domain(capi, kernel):
    dim = 4
    prob = make_problem(80, dim, g_idx=(0,), seed=23, noise=0.05)
    c = offset(dim)
    sprob = shifted(prob, c)
    args = lambda pr: (kernel, pr["alpha"], pr["lengths"], pr["X"], pr["y"], pr["noise"], pr["derivs"])  # noqa: E731
    v, v0 = capi.log_marginal_likelihood(*args(sprob)), capi.log_marginal_likelihood(*args(prob))
    g, g0 = capi.grad_log_marginal_likelihood(*args(sprob)), capi.grad_log_marginal_likelihood(*args(prob))
    vr = checker().log_marginal_likelihood(*args(sprob))
    gr = checker().grad_log_marginal_likelihood(*args(sprob))
    # the unit-box parity tests compare the likelihood at 1e-8 and its gradient at 1e-7 (tests/test_gpu_reference_drivers.py)
    gtol = dict(rtol=1e-7, atol=1e-9 * np.abs(gr).max())
    np.testing.assert_allclose(v, vr, rtol=1e-8)
    np.testing.assert_allclose(g, gr, **gtol)
    np.testing.assert_allclose(v, v0, rtol=1e-8)
    np.testing.assert_allclose(g, g0, **gtol)

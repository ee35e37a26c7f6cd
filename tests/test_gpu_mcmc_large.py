"""GPU tests of the ensemble q-KG / d-KG and q-EI past the per-set row bounds (DESIGN.md K18), through the C ABI: exact
decomposition into the members' single-GP large calls, the reference's ensemble evaluators on table-fed normals, the
unchanged boundary, the drivers, the memory contract, a singular member, batch / chunk invariance and the GPP module."""
import os
import subprocess
import sys

import numpy as np
import pytest

from gpu_util import checker
from synth import DISCRETE_ONLY_GD, EXAMPLE_INNER_GD, make_problem, unit_bounds

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


def _fidelity_cost(pts, nf, M, values, grads):
    """apply_fidelity_cost (multistart.cu) in its operation order: values / (M cost), the quotient rule per coordinate."""
    nc, q, dim = pts.shape
    v_out, g_out = values.copy(), grads.copy() if grads is not None else None
    for c in range(nc):
        x = pts[c]
        cost, index = 1.0, -1
        if nf > 0:
            cost = 0.0
            for i in range(q):
                pc = 1.0
                for j in range(dim - nf, dim):
                    pc *= x[i, j]
                if cost < pc:
                    cost, index = pc, i
        kg_avg = values[c] / float(M)
        v_out[c] = values[c] / (float(M) * cost)
        if grads is not None:
            for i in range(q):
                for d in range(dim):
                    gradcost = cost / x[i, d] if (i == index and d >= dim - nf) else 0.0
                    ga = grads[c, i, d] / float(M)
                    g_out[c, i, d] = (ga * cost - kg_avg * gradcost) / (cost * cost)
    return v_out, g_out


def _member_sum(parts):
    """the member-ordered sum from 0.0, as the ensemble reduces"""
    acc = np.zeros_like(parts[0])
    for x in parts:
        acc = acc + x
    return acc


# (id, kernel, dim, g_idx, q, p, nf): Q = (q + p)(1 + g) from 33 to about 100
KG_CASES = [
    ("se-g0-q10p30", 0, 3, (), 10, 30, 0),
    ("matern-g2-u12", 1, 3, (0, 2), 4, 8, 0),
    ("se-g2-u17-nf1", 0, 3, (1, 2), 5, 12, 1),
    ("matern-g0-q5p90-nf1", 1, 3, (), 5, 90, 1),
]


@pytest.mark.parametrize("case", KG_CASES, ids=[c[0] for c in KG_CASES])
def test_kg_mcmc_is_the_sum_of_member_large_calls(capi, case):
    _, kernel, dim, g_idx, q, p, nf = case
    M, mc, num_pts = 3, 32, 5
    assert 32 < (q + p) * (1 + len(g_idx)) <= 100
    prob = make_problem(20, dim, g_idx=g_idx, seed=21, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, len(g_idx), 4)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"], kernel=kernel)
    rng = np.random.default_rng(8)
    cands = rng.uniform(0.2, 0.9, size=(3, q, dim))
    Xp = rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, num_pts, dim - nf))
    best = rng.uniform(-0.3, 0.3, size=M)
    ib = unit_bounds(dim - nf)
    v, g = ens.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, ib, disc, num_fidelity=nf, seed=9, grad=True)
    parts = [m.kg_large(cands, Xp, mc, best[i], EXAMPLE_INNER_GD, ib, disc[i], num_fidelity=nf, seed=9, grad=True)
             for i, m in enumerate(ens.members)]
    vw, gw = _fidelity_cost(cands, nf, M, _member_sum([x[0] for x in parts]), _member_sum([x[1] for x in parts]))
    np.testing.assert_array_equal(v, vw)
    np.testing.assert_array_equal(g, gw)
    # the value-only call is the same evaluation, and one member at a time gives the same bits
    np.testing.assert_array_equal(ens.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, ib, disc, num_fidelity=nf, seed=9), v)
    capi.set_option("ensemble_members_in_flight", 1)
    try:
        v1, g1 = ens.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, ib, disc, num_fidelity=nf, seed=9, grad=True)
    finally:
        capi.set_option("ensemble_members_in_flight", 0)
    np.testing.assert_array_equal(v1, v)
    np.testing.assert_array_equal(g1, g)


@pytest.mark.parametrize("kernel,g_idx,q,p", [(0, (), 97, 0), (1, (), 40, 80), (1, (1,), 20, 180)])
def test_ei_mcmc_is_the_mean_of_member_large_calls(capi, kernel, g_idx, q, p):
    M, dim, mc = 3, 3, 128
    prob = make_problem(24, dim, g_idx=g_idx, seed=31, noise=0.05, length=0.3)
    hypers, noises = _ensemble_inputs(M, dim, len(g_idx), 6)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"], kernel=kernel)
    rng = np.random.default_rng(9)
    cands = rng.uniform(size=(3, q, dim))
    Xp = rng.uniform(size=(p, dim))
    best = np.full(M, float(prob["y"][:: 1 + len(g_idx)].min()) + 0.3)
    v, g = ens.ei(cands, Xp, mc, best, seed=5, grad=True)
    parts = [m.ei_large(cands, Xp, mc, best[i], seed=5, grad=True) for i, m in enumerate(ens.members)]
    np.testing.assert_array_equal(v, _member_sum([x[0] for x in parts]) / float(M))
    np.testing.assert_array_equal(g, _member_sum([x[1] for x in parts]) / float(M))
    table = rng.standard_normal(mc * (q + p))
    vt = ens.ei(cands, Xp, mc, best, table=table)
    wt = _member_sum([m.ei_large(cands, Xp, mc, best[i], table=table) for i, m in enumerate(ens.members)]) / float(M)
    np.testing.assert_array_equal(vt, wt)


@pytest.mark.parametrize("gd", ["discrete", "inner"])
@pytest.mark.parametrize("g_idx,q,p,nf", [((), 8, 26, 0), ((0, 1), 3, 9, 0), ((), 30, 4, 1)])
def test_kg_mcmc_matches_reference_past_32_rows(capi, g_idx, q, p, nf, gd):
    """the reference's KnowledgeGradientMCMCEvaluator (Matern 5/2 members) on the same table-fed normals"""
    M, dim, num_pts = 3, 3, 5
    prob = make_problem(16, dim, g_idx=g_idx, seed=29, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, len(g_idx), 5)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"])
    Q = (q + p) * (1 + len(g_idx))
    assert Q > 32
    rng = np.random.default_rng(17)
    Xq = rng.uniform(0.2, 0.9, size=(q, dim))
    Xp = rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, num_pts, dim - nf))
    best = rng.uniform(-0.3, 0.3, size=M)
    mc = 16 if gd == "discrete" else 32
    inner = DISCRETE_ONLY_GD if gd == "discrete" else EXAMPLE_INNER_GD
    table = rng.standard_normal((mc // 2) * Q)
    v, g = ens.kg(Xq, Xp, mc, best, inner, unit_bounds(dim - nf), disc, num_fidelity=nf, table=table, grad=True)
    vr, gr = checker().kg_mcmc(hypers, noises, prob["X"], prob["y"], prob["derivs"], Xq, Xp, mc, best, table, inner,
                               unit_bounds(dim - nf), disc, num_fidelity=nf, grad=True)
    rv, rg = (1e-8, 1e-6) if gd == "discrete" else (1e-7, 1e-5)
    np.testing.assert_allclose(v[0], vr, rtol=rv, atol=1e-11)
    np.testing.assert_allclose(g[0], gr, rtol=rg, atol=1e-8)


@pytest.mark.parametrize("q,p", [(97, 0), (30, 90)])
def test_ei_mcmc_matches_reference_past_96_rows(capi, q, p):
    M, dim, mc = 3, 3, 64
    prob = make_problem(30, dim, seed=12, noise=1e-2, length=0.3)
    hypers, noises = _ensemble_inputs(M, dim, 0, 7)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    rng = np.random.default_rng(40 + q)
    Xq, Xp = rng.uniform(size=(q, dim)), rng.uniform(size=(p, dim))
    best = np.full(M, float(prob["y"].min()) + 0.3)
    table = rng.standard_normal(mc * (q + p))
    v, g = ens.ei(Xq, Xp, mc, best, table=table, grad=True)
    vr, gr = checker().ei_mcmc(hypers, noises, prob["X"], prob["y"], None, Xq, Xp, mc, best, table, grad=True)
    assert abs(v[0] - vr) <= 1e-10 * max(1.0, abs(vr)), (v[0], vr)
    np.testing.assert_allclose(g[0], gr, rtol=1e-7, atol=1e-9 * max(1.0, np.abs(gr).max()))


def test_boundary_is_unchanged(capi):
    M, dim = 3, 3
    prob = make_problem(20, dim, seed=2, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, 0, 9)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    rng = np.random.default_rng(1)
    # q-KG at Q = 32: the members' cmoe_kg_eval
    q, p, mc = 4, 28, 32
    cands, Xp = rng.uniform(size=(3, q, dim)), rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, 4, dim))
    best = rng.uniform(-0.3, 0.3, size=M)
    v, g = ens.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, seed=3, grad=True)
    parts = [m.kg(cands, Xp, mc, best[i], EXAMPLE_INNER_GD, unit_bounds(dim), disc[i], seed=3, grad=True)
             for i, m in enumerate(ens.members)]
    vw, gw = _fidelity_cost(cands, 0, M, _member_sum([x[0] for x in parts]), _member_sum([x[1] for x in parts]))
    np.testing.assert_array_equal(v, vw)
    np.testing.assert_array_equal(g, gw)
    # q-EI at q + p = 96: the members' per-set kernels
    q, p = 6, 90
    cands, Xp = rng.uniform(size=(3, q, dim)), rng.uniform(size=(p, dim))
    bei = np.full(M, float(prob["y"].min()) + 0.3)
    v, g = ens.ei(cands, Xp, 256, bei, seed=3, grad=True)
    parts = [m.ei(cands, Xp, 256, bei[i], seed=3, grad=True) for i, m in enumerate(ens.members)]
    np.testing.assert_array_equal(v, _member_sum([x[0] for x in parts]) / float(M))
    np.testing.assert_array_equal(g, _member_sum([x[1] for x in parts]) / float(M))


def test_multistart_mcmc_drivers_past_the_bounds(capi):
    from cornell_moe_b200 import multigpu
    M, dim, mc = 3, 2, 32
    prob = make_problem(25, dim, seed=12, noise=0.05)
    hypers, noises = _ensemble_inputs(M, dim, 0, 3)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    rng = np.random.default_rng(14)
    q, p = 3, 31  # Q = 34
    starts = rng.uniform(size=(24, q, dim))
    Xp = rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, 6, dim))
    best = np.array([float(m.posterior(disc[i][:, None, :], (), ("mean",))["mean"].min())
                     for i, m in enumerate(ens.members)])
    outer = [24, 3, 1, 0, 0.7, 0.3, 0.2, 1e-7]
    args = (starts, Xp, mc, best, outer, EXAMPLE_INNER_GD, unit_bounds(dim), unit_bounds(dim), disc)
    bp, bv, found, sv = ens.multistart_kg(*args, seed=5)
    assert found and np.isfinite(bv) and np.all(bp >= 0.0) and np.all(bp <= 1.0)
    np.testing.assert_array_equal(sv, ens.kg(starts, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, seed=5))
    per = np.mean([m.kg_large(starts, Xp, mc, best[i], EXAMPLE_INNER_GD, unit_bounds(dim), disc[i], seed=5)
                   for i, m in enumerate(ens.members)], axis=0)
    np.testing.assert_allclose(sv, per, rtol=1e-12, atol=1e-14)
    # one outer step of the descent driver reproduces the update rule on the averaged gradient
    one = [1, 1, 1, 0, 0.7, 0.3, 0.2, 1e-7]
    vals, pts = ens.kg_gradient_descent(starts[:2], Xp, mc, best, one, EXAMPLE_INNER_GD, unit_bounds(dim),
                                        unit_bounds(dim), disc, seed=5)
    _, g = ens.kg(starts[:2], Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, seed=5, grad=True)
    backend = checker()
    for s in range(2):
        want = starts[s].copy()
        step = 0.3 * g[s]
        for k in range(q):
            step[k] = backend.limit_update(unit_bounds(dim), 0.2, starts[s][k], step[k])
        want += step
        np.testing.assert_allclose(pts[s], want, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(vals[s], ens.kg(want, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc,
                                                   seed=5)[0], rtol=1e-10)
    # the multi-GPU layer without a process group is the C driver
    bp_s, bv_s, found_s, sv_s = multigpu.multistart_kg_mcmc(ens, *args, seed=5)
    np.testing.assert_allclose(sv_s, sv, rtol=1e-13, atol=1e-15)
    assert found_s == found
    np.testing.assert_allclose(bv_s, bv, rtol=1e-12)
    np.testing.assert_allclose(bp_s, bp, rtol=1e-12, atol=1e-14)
    # q-EI past 96 rows
    q, p = 2, 100
    st = rng.uniform(size=(22, q, dim))
    Xp = rng.uniform(size=(p, dim))
    ybest = np.full(M, float(prob["y"].min()))
    bp, bv, found, sv = ens.multistart_ei(st, Xp, 128, ybest, [22, 3, 1, 0, 0.7, 0.2, 0.2, 1e-8], unit_bounds(dim),
                                          seed=3)
    assert np.all(bp >= 0.0) and np.all(bp <= 1.0) and bv >= 0.0
    np.testing.assert_array_equal(sv, ens.ei(st, Xp, 128, ybest, seed=3))
    per = np.mean([m.ei_large(st, Xp, 128, ybest[i], seed=3) for i, m in enumerate(ens.members)], axis=0)
    np.testing.assert_allclose(sv, per, rtol=1e-12, atol=1e-15)
    vals, pts = ens.ei_gradient_descent(st[:2], Xp, 128, ybest, [1, 1, 1, 0, 0.7, 0.2, 0.2, 1e-8], unit_bounds(dim),
                                        seed=3)
    _, g = ens.ei(st[:2], Xp, 128, ybest, seed=3, grad=True)
    for s in range(2):
        want = st[s].copy()
        step = 0.2 * g[s]
        for k in range(q):
            step[k] = backend.limit_update(unit_bounds(dim), 0.2, st[s][k], step[k])
        want += step
        np.testing.assert_allclose(pts[s], want, rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(vals[s], ens.ei(want, Xp, 128, ybest, seed=3)[0], rtol=1e-10)


def _used_mib():
    """this process's device memory from a read-only nvidia-smi query; None where the pid is not visible"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=60).stdout
    except (OSError, subprocess.SubprocessError):
        return None
    for line in out.splitlines():
        parts = [x.strip() for x in line.split(",")]
        if len(parts) == 2 and parts[0] == str(os.getpid()):
            return float(parts[1])
    return None


def _device_used_mib():
    """the device's used memory (cudaMemGetInfo through torch, whose context is made before the first reading)"""
    import torch
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2**20


def test_memory_does_not_grow_with_the_members(capi):
    """Value-only q-KG at Q = 40 with 2^20 samples: one candidate's chunk is about 1.3 GB, so 16 members run one at a
    time on the one 2 GiB region of the first member's handle; per-member workspaces would add over 15 GiB.  Both
    readings are taken before any call, after the M = 1 call and after the first M = 16 call: this process's memory
    where nvidia-smi lists its pid, else the device's used memory.  The M = 1 call must show its workspace (>= 1 GiB),
    so the reading sees workspaces, and the M = 16 call must add less than 512 MiB."""
    M, dim, q, p, mc = 16, 3, 10, 30, 1 << 20
    prob = make_problem(20, dim, seed=5, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, 0, 12)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    one = capi.GaussianProcessEnsemble.from_members(ens.members[:1])
    rng = np.random.default_rng(3)
    cand, Xp = rng.uniform(size=(1, q, dim)), rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, 5, dim))
    best = np.zeros(M)

    def readings():
        return _used_mib(), _device_used_mib()

    r0 = readings()
    v1 = one.kg(cand, Xp, mc, best[:1], DISCRETE_ONLY_GD, unit_bounds(dim), disc[:1], seed=1)
    r1 = readings()
    v16 = ens.kg(cand, Xp, mc, best, DISCRETE_ONLY_GD, unit_bounds(dim), disc, seed=1)
    r16 = readings()
    assert np.isfinite(v1).all() and np.isfinite(v16).all()
    k = 0 if all(r[0] is not None for r in (r0, r1, r16)) else 1
    assert r1[k] - r0[k] >= 1024.0, ("the M = 1 workspace is not visible in the reading", r0, r1)
    assert r16[k] - r1[k] < 512.0, (r1, r16)


def test_singular_member_reports_its_leading_minor(capi):
    M, dim, q, p = 4, 3, 3, 31  # Q = 34
    prob = make_problem(12, dim, seed=8, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, 0, 13)
    noises[2] = 0.0  # member 2: noise-free, so a union point on a training point has a singular covariance
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    rng = np.random.default_rng(4)
    cands = rng.uniform(size=(3, q, dim))
    cands[1, 2] = prob["X"][5]
    Xp = rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, 4, dim))
    best = np.zeros(M)
    with pytest.raises(capi.SingularMatrixError) as single:
        ens.members[2].kg_large(cands, Xp, 16, 0.0, DISCRETE_ONLY_GD, unit_bounds(dim), disc[2], seed=1)
    with pytest.raises(capi.SingularMatrixError) as err:
        ens.kg(cands, Xp, 16, best, DISCRETE_ONLY_GD, unit_bounds(dim), disc, seed=1, grad=True)
    assert err.value.info == single.value.info and err.value.info > 0
    # the other members and candidates are untouched: the ensemble still evaluates without the duplicate
    ok = cands[[0, 2]]
    v = ens.kg(ok, Xp, 16, best, DISCRETE_ONLY_GD, unit_bounds(dim), disc, seed=1)
    assert np.isfinite(v).all()


def test_batch_and_chunk_invariance(capi):
    """2^17 samples with gradients make one candidate's chunk workspace about 270 MB: three members in flight get two
    candidates per chunk, so a batch of five spans three chunks."""
    M, dim, q, p, mc = 3, 3, 10, 30, 1 << 17
    prob = make_problem(20, dim, seed=6, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, 0, 14)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    rng = np.random.default_rng(5)
    cands, Xp = rng.uniform(size=(5, q, dim)), rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, 5, dim))
    best = np.zeros(M)
    args = (Xp, mc, best, DISCRETE_ONLY_GD, unit_bounds(dim), disc)
    v, g = ens.kg(cands, *args, seed=2, grad=True)
    for c in (0, 3, 4):
        vc, gc = ens.kg(cands[c:c + 1], *args, seed=2, grad=True)
        np.testing.assert_array_equal(vc[0], v[c])
        np.testing.assert_array_equal(gc[0], g[c])


def test_gpp_mcmc_entries_past_the_bounds(capi):
    sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
    import GPP as C_GP
    M, dim, mc, num_pts = 3, 3, 16, 4
    prob = make_problem(18, dim, seed=44, noise=0.1)
    hypers, noises = _ensemble_inputs(M, dim, 0, 2)
    gpm = C_GP.GaussianProcessMCMC(list(hypers.ravel()), list(noises.ravel()), list(prob["X"].ravel()),
                                   list(prob["y"]), [], M, 0, dim, 18)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"])
    rnd = C_GP.RandomnessSourceContainer(2)
    rnd.SetExplicitNormalRNGSeed(99)
    rng = np.random.default_rng(3)
    q, p = 4, 30  # Q = 34
    Xq, Xp = rng.uniform(size=(q, dim)), rng.uniform(size=(p, dim))
    disc = rng.uniform(size=(M, num_pts, dim))
    best = rng.uniform(-0.3, 0.3, size=M)

    class Inner:
        domain_type = C_GP.DomainTypes.tensor_product
        optimizer_type = C_GP.OptimizerTypes.gradient_descent
        num_random_samples = 12
        optimizer_parameters = C_GP.GradientDescentParameters(*EXAMPLE_INNER_GD)

    kg = C_GP.compute_knowledge_gradient_mcmc(gpm, 0, Inner, list(unit_bounds(dim)), list(disc.ravel()),
                                              list(Xq.ravel()), list(Xp.ravel()), num_pts, q, p, mc, list(best), rnd)
    gkg = C_GP.compute_grad_knowledge_gradient_mcmc(gpm, 0, Inner, list(unit_bounds(dim)), list(disc.ravel()),
                                                    list(Xq.ravel()), list(Xp.ravel()), num_pts, q, p, mc, list(best),
                                                    rnd)
    v, g = ens.kg(Xq, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(dim), disc, seed=99, grad=True)
    assert kg == v[0]
    np.testing.assert_array_equal(np.array(gkg).reshape(q, dim), g[0])
    status = {}
    vals = C_GP.evaluate_KG_mcmc_at_point_list(gpm, 0, Inner, list(unit_bounds(dim)), list(Xq.ravel()),
                                               list(disc.ravel()) + list(Xp.ravel()), 1, num_pts, q, p, list(best), mc,
                                               2, rnd, status)
    assert vals[0] == v[0]
    qe, pe = 10, 90  # q + p = 100
    Xq, Xp = rng.uniform(size=(qe, dim)), rng.uniform(size=(pe, dim))
    bei = list(np.full(M, float(prob["y"].min()) + 0.3))
    ei = C_GP.compute_expected_improvement_mcmc(gpm, list(Xq.ravel()), list(Xp.ravel()), qe, pe, mc, bei, rnd)
    gei = C_GP.compute_grad_expected_improvement_mcmc(gpm, list(Xq.ravel()), list(Xp.ravel()), qe, pe, mc, bei, rnd)
    v, g = ens.ei(Xq, Xp, mc, np.array(bei), seed=99, grad=True)
    assert ei == v[0]
    np.testing.assert_array_equal(np.array(gei).reshape(qe, dim), g[0])
    vals = C_GP.evaluate_EI_mcmc_at_point_list(gpm, list(Xq.ravel()), list(Xp.ravel()), 1, qe, pe, bei, mc, 2, rnd,
                                               status)
    assert vals[0] == v[0]

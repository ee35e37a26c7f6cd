"""GPU tests of q-KG on GPs with more than eight derivative observations per point (d-KG with full gradients up to 31
dimensions): the wide instantiations of kg_mc_gen_kernel (CMOE_KG_WIDE_ENTRIES_FOR_DIM, kg_mc_wide_*.cu) against the
CPU checker on identical table-fed normals, their dispatch, the size limits, determinism, the ensemble entry point and
the reference's multistart driver.

Which case reaches which branch of the wide weight ring (stream_point_weights_wide) and of the operand staging:
* a point's rows wrapping around the end of the ring: every case with 1 + g not dividing 80 (g = 10, 11, 12, 16, 20, 31);
  never wrapping: g = 9 and g = 15 (10 and 16 rows per point);
* a partial last stage (N (1 + g) not a multiple of 8): the cases with an odd N;
* training points staged in shared memory (stage_ops): every case with N (DIMP + 2) doubles <= 20 KiB; read through the
  read-only path instead: `d9-g9-unstaged` (N = 200);
* own-lane weight fill: every case (all lanes take their first sample together); warp-cooperative fill of stragglers:
  test_wide_many_samples_per_lane (1024 samples per candidate, several per lane)."""
import os
import re

import numpy as np
import pytest

import oracle as orc
from gpu_util import checker
from synth import DISCRETE_ONLY_GD, EXAMPLE_INNER_GD, make_problem, unit_bounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cornell-moe_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_dkg_wide.npz")

KG_DIMS = (2, 4, 6, 8, 12, 16, 32)
KG_GEN_WIDTHS = (8, 16, 24, 32)
KG_MAX_G = 8       # narrow derivative-observation kernel
KG_MAX_G_WIDE = 31

# (id, d, g_idx, q, p, num_fidelity, N)
WIDE_CASES = [
    ("d9-g9", 9, tuple(range(9)), 1, 0, 0, 11),                 # Q 10, DIM 12, width 16
    ("d10-g10-q2", 10, tuple(range(10)), 2, 0, 0, 9),           # Q 22, width 24
    ("d12-g9-q2p1", 12, (0, 2, 3, 5, 6, 7, 9, 10, 11), 2, 1, 0, 8),  # Q 30, width 32, a subset
    ("d16-g16", 16, tuple(range(16)), 1, 0, 0, 9),              # DIM 16, width 24
    ("d20-g15", 20, tuple(range(1, 20, 4)) + tuple(range(2, 20, 2)) + (0,), 1, 0, 0, 9),  # DIM 32, width 16
    ("d31-g31", 31, tuple(range(31)), 1, 0, 0, 7),              # Q 32, the largest accepted
    ("d10-g9-nf1", 10, tuple(range(9)), 1, 0, 1, 10),           # num_fidelity = 1
    ("d13-g12", 13, tuple(range(12, -1, -1))[:12], 1, 0, 0, 9),  # DIM 16, width 16; indices in descending order
    ("d16-g12-q2", 16, tuple(range(0, 16, 4)) + tuple(range(1, 16, 2)), 2, 0, 0, 7),  # DIM 16, width 32
    ("d24-g20", 24, tuple(range(2, 22)), 1, 0, 0, 7),           # DIM 32, width 24
    ("d9-g9-unstaged", 9, tuple(range(9)), 1, 0, 0, 200),       # operands through the read-only path
]


def _padded(sizes, v):
    return min(s for s in sizes if s >= v)


def _compiled_wide_entries():
    """{(kernel, padded dim, width)} of the wide derivative-observation kernel as compiled: CMOE_KG_WIDE_ENTRIES_FOR_DIM in
    kg_mc.cuh over the dimensions of the kg_mc_wide_*.cu translation units."""
    with open(os.path.join(CSRC, "kg_mc.cuh")) as f:
        src = f.read()
    m = re.search(r"#define CMOE_KG_WIDE_ENTRIES_FOR_DIM\(D\)((?:.*\\\n)*.*)", src)
    assert m, "CMOE_KG_WIDE_ENTRIES_FOR_DIM not found in kg_mc.cuh"
    per_dim = [(int(k), int(qp)) for k, qp in re.findall(r"kg_entry<(\d+),\s*D,\s*(\d+),\s*kKgWide>\(\)", m.group(1))]
    dims = []
    for name in sorted(os.listdir(CSRC)):
        if re.fullmatch(r"kg_mc_wide_\d+\.cu", name):
            with open(os.path.join(CSRC, name)) as f:
                dims += [int(v) for v in re.findall(r"CMOE_KG_WIDE_ENTRIES_FOR_DIM\((\d+)\)", f.read())]
    return {(k, dim, qp) for dim in dims for k, qp in per_dim}


def test_wide_cases_reach_every_compiled_wide_instantiation():
    """CPU: the cases above reach every compiled wide (kernel, dim, width) entry with shapes the C ABI accepts, and only
    g > 8 can reach a wide entry (g <= 8 dispatches exactly as without them)."""
    compiled = _compiled_wide_entries()
    assert len(compiled) == 18, sorted(compiled)
    reached = set()
    for _, d, g_idx, q, p, nf, _ in WIDE_CASES:
        g = len(g_idx)
        assert KG_MAX_G < g <= min(d, KG_MAX_G_WIDE) and len(set(g_idx)) == g and all(0 <= a < d for a in g_idx)
        assert 0 <= nf < d
        Q = (q + p) * (1 + g)
        assert Q <= 32
        for kernel in (0, 1):
            e = (kernel, _padded(KG_DIMS, d), _padded(KG_GEN_WIDTHS, Q))
            assert e in compiled, e
            reached.add(e)
    assert reached == compiled
    # every (dim, width) a wide entry serves is only reachable with g >= 9: dim >= 9 and Q = U (1 + g) >= 10
    assert all(dim >= 12 and qp >= 16 for _, dim, qp in compiled)


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


def _pair(capi, kernel, prob):
    gp = capi.GaussianProcess(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                              prob["derivs"])
    ref, lm = checker().gp(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    return gp, ref


def _inputs(case, mc, seed=27):
    _, d, g_idx, q, p, nf, _ = case
    rng = np.random.default_rng(seed + d)
    cands = rng.uniform(size=(2, q, d))
    Xp = rng.uniform(size=(p, d))
    disc = rng.uniform(size=(5, d - nf))
    table = rng.standard_normal((mc // 2) * (q + p) * (1 + len(g_idx)))
    return cands, Xp, disc, table


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("gd", [DISCRETE_ONLY_GD, EXAMPLE_INNER_GD], ids=["discrete", "inner"])
@pytest.mark.parametrize("case", WIDE_CASES, ids=[c[0] for c in WIDE_CASES])
def test_wide_dkg_table_fed(capi, case, gd, kernel):
    _, d, g_idx, q, p, nf, N = case
    prob = make_problem(N, d, g_idx=g_idx, seed=9 + d, noise=0.1)
    gp, ref = _pair(capi, kernel, prob)
    mc = 32
    cands, Xp, disc, table = _inputs(case, mc)
    best = float(ref.mean_additional(np.concatenate([disc, np.ones((len(disc), nf))], axis=1)).min())
    kg, grad = gp.kg(cands, Xp, mc, best, gd, unit_bounds(d - nf), disc, num_fidelity=nf, table=table, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], Xp, mc, best, table, gd, unit_bounds(d - nf), disc, num_fidelity=nf, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [0, 1])
def test_wide_many_samples_per_lane(capi, kernel):
    """1024 samples per candidate: lanes take several samples each, so columns are filled by cohorts of lanes (own-lane
    fill) and for stragglers (warp-cooperative fill)."""
    case = WIDE_CASES[1]
    _, d, g_idx, q, p, nf, N = case
    prob = make_problem(N, d, g_idx=g_idx, seed=9 + d, noise=0.1)
    gp, ref = _pair(capi, kernel, prob)
    mc = 1024
    cands, Xp, disc, table = _inputs(case, mc)
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(d), disc, table=table, grad=True)
    v, g = ref.kg(cands[1], Xp, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(d), disc, grad=True)
    np.testing.assert_allclose(kg[1], v, rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(grad[1], g, rtol=1e-5, atol=1e-8)


@pytest.mark.gpu
def test_wide_bounds(capi):
    rng = np.random.default_rng(3)
    for d, g, q in ((32, 32, 1), (10, 10, 3)):  # Q = 33 both times
        prob = make_problem(4, d, g_idx=tuple(range(g)), seed=d, noise=0.1)
        gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
        with pytest.raises(capi.BoundsError):
            gp.kg(rng.uniform(size=(1, q, d)), None, 4, 0.0, DISCRETE_ONLY_GD, unit_bounds(d), rng.uniform(size=(3, d)),
                  seed=1)
    # g > 8 with a partial derivative observed twice per point is refused
    prob = make_problem(4, 10, g_idx=(0, 1, 2, 3, 4, 5, 6, 7, 8, 8), seed=5, noise=0.1)
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    with pytest.raises(capi.BoundsError):
        gp.kg(rng.uniform(size=(1, 1, 10)), None, 4, 0.0, DISCRETE_ONLY_GD, unit_bounds(10), rng.uniform(size=(3, 10)),
              seed=1)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [0, 1])
def test_wide_deterministic_and_permutation_invariant(capi, kernel):
    d, g_idx = 12, tuple(range(11))
    prob = make_problem(13, d, g_idx=g_idx, seed=41, noise=0.1)
    gp = capi.GaussianProcess(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                              prob["derivs"])
    rng = np.random.default_rng(8)
    cands = rng.uniform(size=(7, 1, d))
    disc = rng.uniform(size=(6, d))
    args = (None, 256, 0.1, EXAMPLE_INNER_GD, unit_bounds(d), disc)
    kg, grad = gp.kg(cands, *args, seed=17, grad=True)
    assert np.all(np.isfinite(kg)) and np.all(np.isfinite(grad))
    k2, g2 = gp.kg(cands, *args, seed=17, grad=True)
    np.testing.assert_array_equal(k2, kg)
    np.testing.assert_array_equal(g2, grad)
    perm = rng.permutation(7)
    k3, g3 = gp.kg(cands[perm], *args, seed=17, grad=True)
    np.testing.assert_array_equal(k3, kg[perm])
    np.testing.assert_array_equal(g3, grad[perm])


@pytest.mark.gpu
def test_wide_ensemble_kg(capi):
    """GaussianProcessEnsemble.kg at g = 10: the mean of the members' q-KG, each against the checker."""
    M, d, g_idx, q, mc = 2, 10, tuple(range(10)), 1, 32
    prob = make_problem(8, d, g_idx=g_idx, seed=31, noise=0.1)
    rng = np.random.default_rng(5)
    hypers = np.concatenate([rng.uniform(0.8, 1.5, size=(M, 1)), rng.uniform(0.6, 1.2, size=(M, d))], axis=1)
    noises = rng.uniform(0.05, 0.15, size=(M, 1 + len(g_idx)))
    Xq = rng.uniform(0.2, 0.9, size=(q, d))
    disc = rng.uniform(size=(M, 4, d))
    best = rng.uniform(-0.5, 0.5, size=M)
    table = rng.standard_normal((mc // 2) * q * (1 + len(g_idx)))
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], prob["derivs"])
    v = ens.kg(Xq, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(d), disc, table=table)
    want = []
    for m in range(M):
        ref, lm = checker().gp(1, hypers[m, 0], hypers[m, 1:], prob["X"], prob["y"], noises[m], prob["derivs"])
        assert lm == 0
        want.append(ref.kg(Xq, None, mc, best[m], table, EXAMPLE_INNER_GD, unit_bounds(d), disc[m]))
    np.testing.assert_allclose(v[0], np.mean(want), rtol=1e-7, atol=1e-10)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's multistart driver at g = 9 (tests/golden/reference_dkg_wide.npz, tests/golden/make_dkg_wide_golden.py)
# ---------------------------------------------------------------------------------------------------------------------
MS_OUTER1 = [12, 1, 1, 0, 0.7, 0.4, 0.2, 1e-7]


def _ms_problem():
    d, g_idx = 9, tuple(range(9))
    prob = make_problem(10, d, g_idx=g_idx, seed=77, noise=0.05)
    rng = np.random.default_rng(78)
    starts = rng.uniform(0.1, 0.9, size=(12, 1, d))
    disc = rng.uniform(size=(5, d))
    return prob, starts, disc


def reference_values(backend):
    """The reference side of test_wide_multistart_kg_matches_reference_driver, from the compiled reference `backend`."""
    prob, starts, disc = _ms_problem()
    d = prob["dim"]
    ref, lm = backend.gp(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    assert lm == 0
    mc, seed = 32, 4243
    best = float(ref.mean_additional(disc).min())
    bd = unit_bounds(d)
    table = orc.normal_draws(seed, (mc // 2) * (1 + len(prob["derivs"])))
    bp, found = orc.ref_multistart_kg(ref, starts, None, mc, best, MS_OUTER1, EXAMPLE_INNER_GD, bd, bd, disc, seed)
    value = ref.kg_reused_state(starts[0], bp, None, mc, best, table, EXAMPLE_INNER_GD, bd, disc)
    return {k: np.asarray(v) for k, v in dict(best=best, table=table, bp=bp, found=found, value=value).items()}


@pytest.mark.gpu
def test_wide_multistart_kg_matches_reference_driver(capi):
    """cmoe_multistart_kg at g = 9 against the reference's unmodified driver on identical normals (one descent step per
    start, so the comparison is exact), then the GPP entry point on the same GP."""
    golden = np.load(GOLDEN)
    prob, starts, disc = _ms_problem()
    d = prob["dim"]
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    bd = unit_bounds(d)
    mc = 32
    bp, bv, found, _ = capi.multistart_kg(gp, starts, None, mc, float(golden["best"]), MS_OUTER1, EXAMPLE_INNER_GD, bd,
                                          bd, disc, seed=1, table=golden["table"])
    assert found == bool(golden["found"])
    np.testing.assert_allclose(bp, golden["bp"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(bv, golden["value"], rtol=1e-7, atol=1e-10)

    import sys
    sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
    import GPP as C_GP
    gpp = C_GP.GaussianProcess([1.0, list(prob["lengths"])], list(prob["X"].ravel()), list(prob["y"]),
                               list(prob["noise"]), [int(a) for a in prob["derivs"]], len(prob["derivs"]), d, prob["N"])
    Params = type("I", (), dict(domain_type=C_GP.DomainTypes.tensor_product,
                                optimizer_type=C_GP.OptimizerTypes.gradient_descent, num_random_samples=8,
                                optimizer_parameters=C_GP.GradientDescentParameters(*EXAMPLE_INNER_GD)))
    outer = type("P", (), dict(domain_type=C_GP.DomainTypes.tensor_product,
                               optimizer_type=C_GP.OptimizerTypes.gradient_descent, num_random_samples=8,
                               optimizer_parameters=C_GP.GradientDescentParameters(*MS_OUTER1)))
    rnd = C_GP.RandomnessSourceContainer(1)
    rnd.SetExplicitNormalRNGSeed(123)
    status = {}
    pts = C_GP.multistart_knowledge_gradient_optimization(outer, Params, gpp, 0, list(bd), list(disc.ravel()), [], 5, 1,
                                                          0, float(golden["best"]), mc, 1, rnd, status)
    assert status["gradient_descent_tensor_product_domain_found_update"] is True
    assert len(pts) == d and all(0.0 <= x <= 1.0 for x in pts)

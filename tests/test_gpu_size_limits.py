"""The batched kernels at the edges of their size contracts.

* Union sizes up to the 96-row bound of the per-set posterior and q-EI kernels, against the CPU checker and a plain
  80-bit restatement of Var = K(P,P) - K*^T K^-1 K* and its Cholesky factor; clean bounds errors just past each limit.
* Every compiled instantiation of the fused q-KG kernels (`CMOE_KG_ENTRIES_FOR_DIM` x the `kg_mc_inst_*.cu` dimensions),
  one case each, against the checker; a CPU test parses the compiled table so that a new instantiation without a case
  fails on any machine.  Plus the global-memory body of `kg_mc_kernel` past the shared-memory fast path.
* Batch, chunk and grid boundaries: more than 65535 candidates (grid.y of the per-candidate launches), more than
  8 x 65535 points in one K(X, P) build, the 2 GiB q-EI chunks and the 3 GiB q-KG batches.  Each result is compared bit
  for bit with the same candidates or sets in a small call (every candidate / set has its own fixed-order reductions).
"""
import glob
import os
import re

import numpy as np
import pytest
from scipy.stats import norm

from gpu_util import checker
from synth import DISCRETE_ONLY_GD, EXAMPLE_INNER_GD, make_problem, unit_bounds

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cornell-moe_b200", "csrc")
LD = np.longdouble
MAX_Q = 96  # kMaxQ: (q+p)(1+num_derivatives) of the per-set posterior / q-EI kernels


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


# ---------------------------------------------------------------------------------------------------------------------
# 80-bit restatement of the posterior covariance and its Cholesky factor
# ---------------------------------------------------------------------------------------------------------------------
def _cov_ld(kernel, alpha, lengths, P1, d1, P2, d2):
    """Covariance between the rows of two point sets in long double.  Rows are point-major: (point i, m) with m = 0 the
    value and m > 0 the derivative along coordinate d[m-1].  With u_a = (p2_a - p1_a) / l_a^2 the block of a point pair
    is  [A, -B u_b ; B u_a, -C u_a u_b + [a == b] B / l_a^2],  (A, B, C) = (k, k, k) for SquareExponential and
    (k, 5/3 alpha e (1 + sqrt5 r), 25/3 alpha e) for Matern-5/2 (e = exp(-sqrt5 r))."""
    P1, P2 = np.asarray(P1, LD), np.asarray(P2, LD)
    lsq = np.asarray(lengths, LD) ** 2
    diff = P2[None, :, :] - P1[:, None, :]
    r2 = (diff * diff / lsq).sum(axis=-1)
    alpha = LD(alpha)
    if kernel == 0:
        A = alpha * np.exp(-r2 / 2)
        B = C = A
    else:
        arg = np.sqrt(LD(5)) * np.sqrt(r2)
        e = np.exp(-arg)
        A = alpha * e * (1 + arg + LD(5) / 3 * r2)
        B = LD(5) / 3 * alpha * e * (arg + 1)
        C = LD(25) / 3 * alpha * e
    u = diff / lsq
    b1, b2 = 1 + len(d1), 1 + len(d2)
    out = np.empty((P1.shape[0], b1, P2.shape[0], b2), dtype=LD)
    out[:, 0, :, 0] = A
    for m, a in enumerate(d1):
        out[:, m + 1, :, 0] = B * u[:, :, a]
    for k, b in enumerate(d2):
        out[:, 0, :, k + 1] = -B * u[:, :, b]
        for m, a in enumerate(d1):
            out[:, m + 1, :, k + 1] = -C * u[:, :, a] * u[:, :, b] + (B / lsq[a] if a == b else 0)
    return out.reshape(P1.shape[0] * b1, P2.shape[0] * b2)


def _chol_ld(A):
    """Lower Cholesky factor, column by column (no pivoting), in long double."""
    A = np.array(A, dtype=LD)
    n = A.shape[0]
    L = np.zeros_like(A)
    for j in range(n):
        s = A[j:, j] - L[j:, :j] @ L[j, :j]
        L[j, j] = np.sqrt(s[0])
        L[j + 1:, j] = s[1:] / L[j, j]
    return L


def _fwd_ld(L, B):
    """L^-1 B by forward substitution, all columns of B at once."""
    X = np.array(B, dtype=LD)
    for i in range(L.shape[0]):
        X[i] = (X[i] - L[i, :i] @ X[:i]) / L[i, i]
    return X


def _posterior_var_ld(kernel, prob, P, ds):
    """Var = K(P,P) - K*^T K^-1 K* with K = K(X,X) + diag(noise by row type), K* = K(X, P), and its Cholesky factor."""
    X, g_idx, lengths, alpha = prob["X"], tuple(prob["derivs"]), prob["lengths"], prob["alpha"]
    K = _cov_ld(kernel, alpha, lengths, X, g_idx, X, g_idx)
    K += np.diag(np.tile(np.asarray(prob["noise"], LD), X.shape[0]))
    V = _fwd_ld(_chol_ld(K), _cov_ld(kernel, alpha, lengths, X, g_idx, P, ds))
    var = _cov_ld(kernel, alpha, lengths, P, ds, P, ds) - V.T @ V
    return var, _chol_ld(var)


def test_posterior_restatement_matches_checker_at_small_shape():
    """The 80-bit restatement itself, against the CPU checker at a small shape with derivative rows on both sides (so the
    tolerances derived from it in the GPU tests rest on a restatement of the same quantity)."""
    for kernel in (0, 1):
        prob = make_problem(12, 3, g_idx=(0, 2), seed=5, noise=1e-2)
        ref, lm = checker().gp(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                               prob["derivs"])
        assert lm == 0
        P = np.random.default_rng(2).uniform(size=(4, 3))
        ds = (1, 2)
        var, L = _posterior_var_ld(kernel, prob, P, ds)
        Q = var.shape[0]
        r = ref.posterior(P, ds, ("var", "chol_var"))
        assert r["rc"] == 0
        np.testing.assert_allclose(r["var"].reshape(Q, Q).T, var.astype(np.float64), rtol=1e-9, atol=1e-11)
        np.testing.assert_allclose(np.tril(r["chol_var"].reshape(Q, Q).T), L.astype(np.float64), rtol=1e-8, atol=1e-10)


# ---------------------------------------------------------------------------------------------------------------------
# A. union sizes up to the 96-row bound
# ---------------------------------------------------------------------------------------------------------------------
# (N, dim, GP derivative observations, set derivative rows, points per set, sets, length scale, gradients)
POSTERIOR_BOUND_CASES = {
    "num96": (40, 3, (), (), 96, 2, 0.08, True),
    # derivative rows have prior variance alpha / l^2: a short length scale keeps cond(Var) near that ratio
    "num32_two_derivative_rows": (40, 3, (0, 2), (0, 2), 32, 2, 0.06, True),
    # the largest post_var_kernel footprint: (96 * 97 + 96 * 32) doubles = 99 KB of the 100 KB opt-in
    "dim32_num96": (40, 32, (), (), 96, 1, 0.5, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("case", list(POSTERIOR_BOUND_CASES))
def test_posterior_at_96_rows(capi, kernel, case):
    N, dim, g_idx, ds, num, nsets, length, grads = POSTERIOR_BOUND_CASES[case]
    prob = make_problem(N, dim, g_idx=g_idx, seed=7 + dim, noise=1e-2, length=length)
    gp, ref = _pair(capi, kernel, prob)
    sets = np.random.default_rng(19).uniform(size=(nsets, num, dim))
    Q = num * (1 + len(ds))
    assert Q == MAX_Q
    want = ("mean", "var", "chol_var") + (("grad_mean", "grad_var", "grad_chol") if grads else ())
    out = gp.posterior(sets, ds, want)
    for s in range(nsets):
        var_ld, L_ld = _posterior_var_ld(kernel, prob, sets[s], ds)
        var64, L64 = var_ld.astype(np.float64), L_ld.astype(np.float64)
        cond = np.linalg.cond(var64)
        assert cond < 1e4, cond  # a well-conditioned Q x Q problem: the comparisons below measure the kernels
        r = ref.posterior(sets[s], ds, want)
        assert r["rc"] == 0
        # tolerance = a small multiple of the checker's own distance from the 80-bit result (floored at a few ulps)
        for name, mine, exact in (("var", out["var"][s], var64), ("chol_var", out["chol_var"][s], L64)):
            theirs = r[name].reshape(Q, Q).T
            mine = mine.reshape(Q, Q).T
            scale = np.abs(exact).max()
            ref_err = np.abs(np.tril(theirs) - np.tril(exact)).max()
            tol = 4.0 * max(ref_err, 16 * np.finfo(np.float64).eps * scale)
            err = np.abs(np.tril(mine) - np.tril(exact)).max()
            assert err <= tol, (name, err, ref_err, tol)
        V = out["var"][s].reshape(Q, Q).T
        np.testing.assert_allclose(V, V.T, rtol=1e-9, atol=1e-11)
        assert np.all(np.triu(out["chol_var"][s].reshape(Q, Q).T, 1) == 0.0)
        np.testing.assert_allclose(out["mean"][s], r["mean"], rtol=1e-9, atol=1e-10)
        if grads:
            np.testing.assert_allclose(out["grad_mean"][s], r["grad_mean"], rtol=1e-8, atol=1e-9)
            np.testing.assert_allclose(out["grad_var"][s], r["grad_var"], rtol=1e-7, atol=1e-8)
            np.testing.assert_allclose(out["grad_chol"][s], r["grad_chol"], rtol=1e-6, atol=1e-7)


# U = q + p: 77 is the last union whose (U^2 + U) doubles fit the default 48 KiB of dynamic shared memory
@pytest.mark.gpu
@pytest.mark.parametrize("q,p", [(77, 0), (70, 8), (90, 6)])
def test_ei_union_up_to_96(capi, q, p):
    prob = make_problem(30, 3, seed=4, length=0.08)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(3141 + q)
    cands = rng.uniform(size=(2, q, 3))
    Xp = rng.uniform(size=(p, 3))
    mc = 64
    table = rng.standard_normal(mc * (q + p))
    best = float(prob["y"].min()) + 0.3
    ei, grad = gp.ei(cands, Xp, mc, best, table=table, grad=True)
    for c in range(2):
        var_ld, _ = _posterior_var_ld(0, prob, np.concatenate([cands[c], Xp]), ())
        assert np.linalg.cond(var_ld.astype(np.float64)) < 1e4
        v, g = ref.ei(cands[c], Xp, mc, best, table, grad=True)
        np.testing.assert_allclose(ei[c], v, rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(grad[c], g, rtol=1e-6, atol=1e-9)
    np.testing.assert_array_equal(gp.ei(cands, Xp, mc, best, table=table), ei)


@pytest.mark.gpu
def test_bounds_errors_just_past_each_limit(capi):
    prob = make_problem(20, 3, seed=2, length=0.1)
    gp, _ = _pair(capi, 0, prob)
    rng = np.random.default_rng(1)
    with pytest.raises(capi.BoundsError):
        gp.posterior(rng.uniform(size=(1, MAX_Q + 1, 3)), (), ("var",))
    with pytest.raises(capi.BoundsError):
        gp.posterior(rng.uniform(size=(1, 33, 3)), (0, 1), ("chol_var",))  # 33 * 3 = 99 rows
    with pytest.raises(capi.BoundsError):
        gp.ei(rng.uniform(size=(1, 90, 3)), rng.uniform(size=(7, 3)), 16, 0.0, seed=1)
    disc = rng.uniform(size=(4, 3))
    with pytest.raises(capi.BoundsError):  # union width 33: no compiled q-KG instantiation
        gp.kg(rng.uniform(size=(1, 33, 3)), None, 4, 0.0, DISCRETE_ONLY_GD, unit_bounds(3), disc, seed=1)
    with pytest.raises(capi.BoundsError):
        gp.kg(rng.uniform(size=(1, 30, 3)), rng.uniform(size=(3, 3)), 4, 0.0, DISCRETE_ONLY_GD, unit_bounds(3), disc,
              seed=1)
    prob_g = make_problem(12, 3, g_idx=(0, 1), seed=3)
    gp_g, _ = _pair(capi, 0, prob_g)
    with pytest.raises(capi.BoundsError):  # 11 * (1 + 2) = 33 rows of the derivative-observation kernel
        gp_g.kg(rng.uniform(size=(1, 11, 3)), None, 4, 0.0, DISCRETE_ONLY_GD, unit_bounds(3), disc, seed=1)
    # the limits themselves are accepted
    gp.posterior(rng.uniform(size=(1, MAX_Q, 3)), (), ("var",))
    gp.kg(rng.uniform(size=(1, 32, 3)), None, 4, 0.0, DISCRETE_ONLY_GD, unit_bounds(3), disc, seed=1)


# the covariance build without derivative observations stages (128 + 64)(dim + 1) + 64 doubles: 51200 B at dim = 32,
# past the default 48 KiB from dim = 31 on (it failed to launch there, so such a GP could not be created)
@pytest.mark.gpu
@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("dim", [30, 31, 32])
def test_gp_fit_up_to_dim_32(capi, kernel, dim):
    prob = make_problem(300, dim, seed=dim, noise=1e-2)
    gp, ref = _pair(capi, kernel, prob)
    K, kinvy, mean = gp.state()
    Kr, kr, mr = ref.state()
    assert mean == mr
    np.testing.assert_allclose(np.tril(K), np.tril(Kr), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(kinvy, kr, rtol=1e-7, atol=1e-8)


# ---------------------------------------------------------------------------------------------------------------------
# B. every compiled q-KG instantiation
# ---------------------------------------------------------------------------------------------------------------------
KG_DIMS = (2, 4, 6, 8, 12, 16, 32)         # padded dimensions, one kg_mc_inst_<D>.cu each
KG_WIDTHS = (2, 4, 8, 16, 24, 32)          # union widths of kg_mc_kernel (no derivative observations)
KG_GEN_WIDTHS = (8, 16, 24, 32)            # union widths that also have kg_mc_gen_kernel
KG_MAX_G = 8


def _below(sizes, v):
    i = sizes.index(v)
    return sizes[i - 1] if i else 0


def _sweep_cases():
    """One case per compiled entry and path.  Even cases use d = the padded dimension (no padding), odd ones the next
    lower padded dimension + 1 (the most padding); the union rows Q = U (1 + g) alternate between the entry's width and
    the next lower compiled width + 1 in the same way, and every other pair of cases has points being sampled."""
    cases = []
    for gen in (False, True):
        widths = KG_GEN_WIDTHS if gen else KG_WIDTHS
        for kernel in (0, 1):
            for dimp in KG_DIMS:
                for width in widths:
                    k = len(cases)
                    d = dimp if k % 2 == 0 else _below(KG_DIMS, dimp) + 1
                    lo = _below(widths, width)
                    target = width if (k // 2) % 2 == 0 else lo + 1
                    if gen:
                        # the derivative path needs g >= 1 observed partials, at most min(d, 8)
                        opts = [(abs(u * (1 + g) - target), -g if k % 3 else g, u, g)
                                for g in range(1, min(d, KG_MAX_G) + 1) for u in range(1, width + 1)
                                if lo < u * (1 + g) <= width]
                        _, _, U, g = min(opts)
                    else:
                        U, g = target, 0
                    p = U // 3 if (k // 4) % 2 == 1 else 0
                    g_idx = tuple(int(v) for v in sorted(np.random.default_rng(k).choice(d, g, replace=False)))
                    cases.append(dict(id=f"{'gen' if gen else 'mc'}-k{kernel}-D{dimp}-W{width}", kernel=kernel, d=d,
                                      q=U - p, p=p, g_idx=g_idx))
    # the five shapes the suite ran before this sweep existed
    for d, q in ((2, 2), (5, 3), (6, 4), (10, 2), (13, 1)):
        cases.append(dict(id=f"d{d}-q{q}", kernel=d % 2, d=d, q=q, p=0, g_idx=()))
    return cases


KG_SWEEP = _sweep_cases()


def _compiled_kg_entries():
    """{(kernel, padded dim, union width, has the derivative-observation kernel)} as compiled: the entry list of
    CMOE_KG_ENTRIES_FOR_DIM in kg_mc.cuh, expanded over the dimensions of the kg_mc_inst_*.cu translation units."""
    with open(os.path.join(CSRC, "kg_mc.cuh")) as f:
        src = f.read()
    m = re.search(r"#define CMOE_KG_ENTRIES_FOR_DIM\(D\)((?:.*\\\n)*.*)", src)
    assert m, "CMOE_KG_ENTRIES_FOR_DIM not found in kg_mc.cuh"
    per_dim = [(builds == "kKgFastGen", int(kern), int(qp)) for kern, qp, builds in
               re.findall(r"kg_entry<(\d+),\s*D,\s*(\d+),\s*(kKgFast|kKgFastGen)>\(\)", m.group(1))]
    dims = []
    for path in glob.glob(os.path.join(CSRC, "kg_mc_inst_*.cu")):
        with open(path) as f:
            dims += [int(v) for v in re.findall(r"CMOE_KG_ENTRIES_FOR_DIM\((\d+)\)", f.read())]
    # every entry has kg_mc_kernel; the kKgFastGen ones add kg_mc_gen_kernel
    return ({(kern, dim, qp, False) for dim in dims for _, kern, qp in per_dim} |
            {(kern, dim, qp, True) for dim in dims for gen, kern, qp in per_dim if gen})


def _dispatch(table, kernel, d, Q, need_gen):
    """find_kg_entry (kg.cu): the smallest compiled (dim, width) >= (d, Q) for the kernel, with the derivative kernel if
    needed.  Returns (kernel, dim, width, path)."""
    fits = [(dim, qp) for kern, dim, qp, gen in table if kern == kernel and dim >= d and qp >= Q and (gen or not need_gen)]
    if not fits:
        return None
    dim, qp = min(fits)
    return kernel, dim, qp, need_gen


def test_kg_sweep_covers_every_compiled_instantiation():
    """CPU: the sweep below reaches every compiled (kernel, dim, width) entry on each of its paths, exactly the compiled
    set, with shapes the C ABI accepts."""
    compiled = _compiled_kg_entries()
    mc_entries = {e for e in compiled if not e[3]}
    gen_entries = {e for e in compiled if e[3]}
    assert len(mc_entries) == 84 and len(gen_entries) == 56, (len(mc_entries), len(gen_entries))
    assert {e[1] for e in compiled} == set(KG_DIMS)
    assert {e[2] for e in compiled} == set(KG_WIDTHS) and {e[2] for e in gen_entries} == set(KG_GEN_WIDTHS)
    reached = []
    for c in KG_SWEEP:
        g = len(c["g_idx"])
        assert c["q"] >= 1 and c["p"] >= 0 and 1 <= c["d"] <= 32 and g <= min(c["d"], KG_MAX_G)
        assert len(set(c["g_idx"])) == g and all(0 <= a < c["d"] for a in c["g_idx"])
        e = _dispatch(compiled, c["kernel"], c["d"], (c["q"] + c["p"]) * (1 + g), g > 0)
        assert e is not None, c
        reached.append(e)
    assert set(reached) == mc_entries | gen_entries
    assert sum(1 for c in KG_SWEEP if c["p"] > 0) >= 20
    # both edges of the padding are exercised for every dimension and width
    assert {c["d"] for c in KG_SWEEP} >= {1, 3, 5, 7, 9, 13, 17} | set(KG_DIMS)


@pytest.mark.gpu
@pytest.mark.parametrize("case", KG_SWEEP, ids=[c["id"] for c in KG_SWEEP])
def test_kg_instantiation_sweep(capi, case):
    kernel, d, q, p, g_idx = case["kernel"], case["d"], case["q"], case["p"], case["g_idx"]
    prob = make_problem(20, d, g_idx=g_idx, seed=100 + d, noise=0.05)
    gp, ref = _pair(capi, kernel, prob)
    rng = np.random.default_rng(d + 7 * q + 3 * p)
    cands = rng.uniform(size=(2, q, d))
    Xp = rng.uniform(size=(p, d))
    disc = rng.uniform(size=(6, d))
    mc = 32
    table = rng.standard_normal((mc // 2) * (q + p) * (1 + len(g_idx)))
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, Xp, mc, best, EXAMPLE_INNER_GD, unit_bounds(d), disc, table=table, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], Xp, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(d), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


# N (DIMP + QP + 2) doubles past 200 KiB: the MC kernel reads its operands from global memory, and the accumulation
# kernel evaluates exp with its range guards
@pytest.mark.gpu
@pytest.mark.parametrize("kernel,N,d,q", [(0, 1500, 8, 8), (0, 400, 32, 32), (1, 400, 32, 32)])
def test_kg_global_memory_body(capi, kernel, N, d, q):
    assert N * (d + q + 2) * 8 > 200 * 1024
    prob = make_problem(N, d, seed=N + d, noise=0.05)
    gp, ref = _pair(capi, kernel, prob)
    rng = np.random.default_rng(q)
    cands = rng.uniform(size=(2, q, d))
    disc = rng.uniform(size=(6, d))
    mc = 32
    table = rng.standard_normal((mc // 2) * q)
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, None, mc, best, EXAMPLE_INNER_GD, unit_bounds(d), disc, table=table, grad=True)
    for c in range(2):
        v, g = ref.kg(cands[c], None, mc, best, table, EXAMPLE_INNER_GD, unit_bounds(d), disc, grad=True)
        np.testing.assert_allclose(kg[c], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(grad[c], g, rtol=1e-5, atol=1e-8)


# ---------------------------------------------------------------------------------------------------------------------
# C. batch, chunk and grid boundaries: bit for bit against the same candidates / sets in a small call
# ---------------------------------------------------------------------------------------------------------------------
def _subsets(n):
    """Index ranges of 5 at the start, across the 65535 boundary when there is one, and at the end."""
    out = [np.arange(0, 5), np.arange(n - 5, n)]
    if n > 65540:
        out.insert(1, np.arange(65532, 65537))
    return out


@pytest.mark.gpu
def test_ei_more_than_65535_candidates(capi):
    prob = make_problem(20, 3, seed=11, length=0.3)
    gp, _ = _pair(capi, 0, prob)
    cands = np.random.default_rng(1).uniform(size=(70000, 1, 3))
    best = float(prob["y"].min()) + 0.3
    ei = gp.ei(cands, None, 64, best, seed=5)
    assert np.all(np.isfinite(ei)) and np.all(ei >= 0)
    for idx in _subsets(70000):
        np.testing.assert_array_equal(gp.ei(cands[idx], None, 64, best, seed=5), ei[idx])


@pytest.mark.gpu
def test_kg_more_than_65535_candidates(capi):
    prob = make_problem(20, 2, seed=12, noise=0.05)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(2)
    cands = rng.uniform(size=(70000, 1, 2))
    disc = rng.uniform(size=(5, 2))
    best = float(ref.mean_additional(disc).min())
    kg, grad = gp.kg(cands, None, 2, best, DISCRETE_ONLY_GD, unit_bounds(2), disc, seed=3, grad=True)
    assert np.all(np.isfinite(kg)) and np.all(np.isfinite(grad))
    for idx in _subsets(70000):
        k2, g2 = gp.kg(cands[idx], None, 2, best, DISCRETE_ONLY_GD, unit_bounds(2), disc, seed=3, grad=True)
        np.testing.assert_array_equal(k2, kg[idx])
        np.testing.assert_array_equal(g2, grad[idx])


@pytest.mark.gpu
def test_posterior_more_than_524280_points(capi):
    """90000 sets x 6 points: 540000 columns of K(X, P) in one build."""
    prob = make_problem(30, 3, seed=13, length=0.3)
    gp, _ = _pair(capi, 1, prob)
    sets = np.random.default_rng(3).uniform(size=(90000, 6, 3))
    want = ("mean", "var", "chol_var")
    out = gp.posterior(sets, (), want)
    for idx in _subsets(90000) + [np.arange(45000, 45005)]:
        small = gp.posterior(sets[idx], (), want)
        for k in want:
            np.testing.assert_array_equal(small[k], out[k][idx])


@pytest.mark.gpu
def test_ei_and_kg_more_than_524280_union_points(capi):
    """17000 candidates x q = 32: 544000 union points in one K(X, P) build (values only: the Smith gradients of that
    many 32-point sets would need about 10 GB)."""
    prob = make_problem(20, 3, seed=14, noise=0.05, length=0.1)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(4)
    cands = rng.uniform(size=(17000, 32, 3))
    best = float(prob["y"].min()) + 0.3
    ei = gp.ei(cands, None, 16, best, seed=9)
    disc = rng.uniform(size=(5, 3))
    kbest = float(ref.mean_additional(disc).min())
    kg = gp.kg(cands, None, 2, kbest, DISCRETE_ONLY_GD, unit_bounds(3), disc, seed=9)
    assert np.all(np.isfinite(ei)) and np.all(np.isfinite(kg))
    for idx in _subsets(17000) + [np.arange(8500, 8505)]:
        np.testing.assert_array_equal(gp.ei(cands[idx], None, 16, best, seed=9), ei[idx])
        np.testing.assert_array_equal(gp.kg(cands[idx], None, 2, kbest, DISCRETE_ONLY_GD, unit_bounds(3), disc, seed=9),
                                      kg[idx])


@pytest.mark.gpu
def test_sample_joint_524288_points_in_one_chunk(capi):
    """4096 sets x 128 points at N = 50: one chunk of kMaxChunkSets sets, 524288 points in one K(X, P) build.  The last
    sets must match a call that starts at their draw."""
    prob = make_problem(50, 3, seed=15, noise=1e-2, length=0.1)
    gp, _ = _pair(capi, 0, prob)
    sets = np.random.default_rng(5).uniform(size=(4096, 128, 3))
    want = ("samples", "argmin", "mean")
    out = gp.sample_joint(sets, seed=21, first_draw=0, jitter=1e-8, want=want)
    tail = gp.sample_joint(sets[4090:], seed=21, first_draw=4090, jitter=1e-8, want=want)
    head = gp.sample_joint(sets[:3], seed=21, first_draw=0, jitter=1e-8, want=want)
    for k in want:
        np.testing.assert_array_equal(tail[k], out[k][4090:])
        np.testing.assert_array_equal(head[k], out[k][:3])
    assert np.all(np.isfinite(out["samples"]))
    np.testing.assert_array_equal(out["argmin"], np.argmin(out["samples"], axis=1))


@pytest.mark.gpu
def test_kg_3gib_batch_split(capi):
    """d = 32, q = 32, 2^20 samples: (32 + 32 + 2) * 8 B * 2^20 of per-sample records per candidate put 5 candidates in
    a 3 GiB batch, so 12 candidates run as 5 + 5 + 2."""
    prob = make_problem(20, 32, seed=16, noise=0.05)
    gp, ref = _pair(capi, 0, prob)
    rng = np.random.default_rng(6)
    cands = rng.uniform(size=(12, 32, 32))
    disc = rng.uniform(size=(5, 32))
    best = float(ref.mean_additional(disc).min())
    mc = 1 << 20
    kg = gp.kg(cands, None, mc, best, DISCRETE_ONLY_GD, unit_bounds(32), disc, seed=17)
    assert np.all(np.isfinite(kg))
    for idx in (np.arange(4, 7), np.arange(9, 12)):
        np.testing.assert_array_equal(gp.kg(cands[idx], None, mc, best, DISCRETE_ONLY_GD, unit_bounds(32), disc,
                                            seed=17), kg[idx])


@pytest.mark.gpu
def test_ei_2gib_chunk_split_and_closed_form(capi):
    """q = 1, 2^23 samples: 3 * 8 B * 2^23 of per-sample scratch per candidate put 10 candidates in a 2 GiB chunk, so 25
    candidates run as 10 + 10 + 5.  The MC value is also checked against the closed-form expected improvement of the
    same (posterior + 1e-6) normal, within 4 standard errors."""
    prob = make_problem(30, 3, seed=17, length=0.3)
    gp, _ = _pair(capi, 0, prob)
    cands = np.random.default_rng(7).uniform(size=(25, 1, 3))
    best = float(prob["y"].min()) + 0.3
    mc = 1 << 23
    ei = gp.ei(cands, None, mc, best, seed=23)
    for idx in (np.arange(8, 12), np.arange(20, 25)):
        np.testing.assert_array_equal(gp.ei(cands[idx], None, mc, best, seed=23), ei[idx])
    post = gp.posterior(cands, (), ("mean", "var"))
    mu = post["mean"][:, 0]
    sigma = np.sqrt(post["var"][:, 0] + 1e-6)
    z = (best - mu) / sigma
    exact = (best - mu) * norm.cdf(z) + sigma * norm.pdf(z)
    second = ((best - mu) ** 2 + sigma ** 2) * norm.cdf(z) + (best - mu) * sigma * norm.pdf(z)  # E[(b - Y)_+^2]
    se = np.sqrt(np.maximum(second - exact ** 2, 0.0) / mc)
    assert np.all(np.abs(ei - exact) <= 4.0 * se + 1e-15), np.max(np.abs(ei - exact) / se)

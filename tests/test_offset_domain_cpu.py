"""Host-side checks of the offset-domain GPU tests (tests/test_gpu_offset_domain.py), no device needed:

* the inputs are hard: the expanded form of -r^2/2 that the q-KG kernels use, evaluated on uncentred scaled coordinates,
  loses more than 1e-9 in the posterior mean on every offset case, so the GPU file cannot quietly turn into a unit-box test;
* each GPU case runs the build its label names, by a restatement of the host's selection rule (find_kg_entry and
  kg_select in kg_mc.cuh): the 200 KiB operand limit of the shared-memory fast path, and its radius contract
  (kFastPathRadius) measured in the frame of the kernels' operands, centred on the mean of the training points."""
import numpy as np
import pytest

import test_gpu_offset_domain as T

DIMS = (2, 4, 6, 8, 12, 16, 32)  # padded dimensions of the compiled q-KG instantiations (kg_mc_inst_*.cu)
QPS = (2, 4, 8, 16, 24, 32)      # union-row widths
FAST_PATH_RADIUS = 2000.0
SMEM_LIMIT = 200 * 1024


def select_path(kernel, N, dim, U, g, rmax):
    """The build kg_select picks for N training points, U union points, g derivative observations and the largest
    centred scaled radius rmax of the operands."""
    Q = U * (1 + g)
    if g > 8:
        return "wide"
    if g > 0:
        return "general"
    DIMP = min(d for d in DIMS if d >= dim)
    QP = min(w for w in QPS if w >= Q)
    smem = (N * (DIMP + QP + 2) + U * (DIMP + 2)) * 8
    if smem > SMEM_LIMIT:
        return "global"
    if not rmax < FAST_PATH_RADIUS:
        return "guarded"
    return "tile" if (kernel == 0 and DIMP == 8 and QP == 8) else "fast"


def centred_rmax(X, lengths, pts, lo, hi, nf):
    """kg.cu's rmax in the frame of the operands: training, discrete, pending and candidate points and the farthest
    corner of the inner domain (fidelity coordinates at 1.0), all relative to the mean of the training points."""
    centre = X.mean(axis=0)
    r = max(np.sqrt((((p - centre) / lengths) ** 2).sum(axis=1)).max() for p in [X] + pts if len(p))
    ps = X.shape[1] - nf
    lo = np.concatenate([lo, np.ones(nf)])
    hi = np.concatenate([hi, np.ones(nf)])
    corner = np.maximum(np.abs(lo - centre), np.abs(hi - centre)) / lengths
    assert corner.size == ps + nf
    return max(r, np.sqrt((corner ** 2).sum()))


def case_inputs(case):
    label, kernel, N, dim, q, p, g_idx, mc, length, nf = case
    prob, cands, Xp, disc, _ = T.kg_inputs(kernel, N, dim, q, p, g_idx, mc, length, nf, seed=500 + N + dim + q)
    ps = dim - nf
    c = T.offset(dim, ps)
    full_disc = np.concatenate([disc, np.ones((len(disc), nf))], axis=1) + c
    pts = [full_disc, Xp + c, cands.reshape(-1, dim) + c]
    return prob, c, pts, np.zeros(ps) + c[:ps], np.ones(ps) + c[:ps]


@pytest.mark.parametrize("case", T.KG_CASES, ids=[c[0] for c in T.KG_CASES])
def test_case_runs_the_build_its_label_names(case):
    label, kernel, N, dim, q, p, g_idx, mc, length, nf = case
    prob, c, pts, lo, hi = case_inputs(case)
    rmax = centred_rmax(prob["X"] + c, prob["lengths"], pts, lo, hi, nf)
    assert select_path(kernel, N, dim, q + p, len(g_idx), rmax) == T.KG_PATHS[label]


@pytest.mark.parametrize("side,target", [("fast", 1990.0), ("guarded", 2010.0)])
def test_radius_edge_cases_straddle_the_fast_path_radius(side, target):
    prob, cands, disc, _, c, _ = T.radius_case(target)
    rmax = centred_rmax(prob["X"] + c, prob["lengths"], [disc + c, cands.reshape(-1, 8) + c], np.zeros(8) + c,
                        np.ones(8) + c, 0)
    assert abs(rmax - target) < 1.0
    assert select_path(0, prob["N"], 8, 5, 0, rmax) == ("tile" if side == "fast" else "guarded")


def _kernel(kernel, alpha, t):
    """k from t = -r^2/2 (SquareExponential) or from r^2 = -2t (Matern-5/2)."""
    if kernel == 0:
        return alpha * np.exp(t)
    r = np.sqrt(np.maximum(-2.0 * t, 0.0)) * np.sqrt(5.0)
    return alpha * (1.0 + r + r * r / 3.0) * np.exp(-r)


def mean_errors(kernel, prob, queries):
    """max |mu_expanded - mu_difference| over the queries, with beta = K^-1 (y - mean) of the value observations (the
    derivative rows, where present, are left out: the kernel values are what the expanded form gets wrong)."""
    X, L, alpha = prob["X"], prob["lengths"], prob["alpha"]
    b = 1 + len(prob["derivs"])
    y = prob["y"].reshape(-1, b)[:, 0]
    Xs, Qs = X / L, queries / L

    def diff_t(A, B):
        return -0.5 * (((A[:, None, :] - B[None, :, :]) ** 2).sum(axis=2))

    def expanded_t(A, B):
        return A @ B.T - 0.5 * (A * A).sum(axis=1)[:, None] - 0.5 * (B * B).sum(axis=1)[None, :]

    K = _kernel(kernel, alpha, diff_t(Xs, Xs)) + prob["noise"][0] * np.eye(len(X))
    beta = np.linalg.solve(K, y - y.mean())
    mu_d = _kernel(kernel, alpha, diff_t(Qs, Xs)) @ beta
    mu_e = _kernel(kernel, alpha, expanded_t(Qs, Xs)) @ beta
    return np.abs(mu_e - mu_d).max()


@pytest.mark.parametrize("case", T.KG_CASES, ids=[c[0] for c in T.KG_CASES])
def test_offset_inputs_defeat_the_uncentred_expanded_form(case):
    label, kernel, N, dim, q, p, g_idx, mc, length, nf = case
    prob, c, pts, lo, hi = case_inputs(case)
    queries = np.random.default_rng(1).uniform(size=(64, dim)) + c
    sprob = T.shifted(prob, c)
    assert mean_errors(kernel, sprob, queries) > 1e-9
    # and the centred frame removes the loss (what the kernels now use)
    centred = dict(sprob, X=sprob["X"] - sprob["X"].mean(axis=0))
    assert mean_errors(kernel, centred, queries - sprob["X"].mean(axis=0)) < 1e-12


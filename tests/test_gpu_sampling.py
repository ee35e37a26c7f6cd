"""Joint posterior sampling on the device (cmoe_gp_sample_joint, cmoe_latin_hypercube, cmoe_gp_sample_global_optima and
the GPP methods on top of them): factor parity beyond the 96-row limit of cmoe_gp_posterior, sample parity with the
reference's answers, the distribution of the draws, the Latin hypercube bit for bit, composition, chunking
invariance, failure reporting, and the SASS of the new DMMA kernels."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from cornell_moe_b200 import capi
from gpu_util import checker
from sampling_ref import latin_hypercube

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "reference_sampling.npz"))
gpu = pytest.mark.gpu


def _gp(kernel, N, dim, lengths, seed=0, noise=1e-2, derivs=None):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, dim))
    g = 0 if derivs is None else len(derivs)
    y = np.sin(3 * X).sum(axis=1)
    if g:
        y = np.column_stack([y] + [3 * np.cos(3 * X[:, d]) for d in derivs]).ravel()
    lens = np.full(dim, lengths)
    args = (kernel, 1.0, lens, X, y, np.full(1 + g, noise))
    return capi.GaussianProcess(*args, derivs=derivs), args, derivs


@gpu
@pytest.mark.parametrize("kernel", [capi.SQUARE_EXPONENTIAL, capi.MATERN_NU_2P5])
@pytest.mark.parametrize("Q", [300, 1000])
def test_factor_and_mean_match_the_checker_beyond_the_old_cap(kernel, Q):
    dim, lengths = 8, (0.25 if kernel == capi.SQUARE_EXPONENTIAL else 0.15)
    gp, args, _ = _gp(kernel, 200, dim, lengths, seed=Q)
    pts = np.random.default_rng(Q + 1).uniform(size=(Q, dim))
    ref, lm = checker().gp(*args)
    assert lm == 0
    post = ref.posterior(pts, want=("mean", "var", "chol_var"))
    var = post["var"].reshape(Q, Q)
    cond = np.linalg.cond(var)
    assert cond < 1e4, cond  # the 1e-10 bound below relies on it
    L_ref = np.tril(post["chol_var"].reshape(Q, Q).T)
    out = gp.sample_joint(pts, want=("mean", "chol"))
    L = out["chol"][0]
    assert np.all(np.triu(L, 1) == 0.0)
    assert np.linalg.norm(L - L_ref) <= 1e-10 * np.linalg.norm(L_ref)
    assert np.linalg.norm(out["mean"][0] - post["mean"]) <= 1e-10 * np.linalg.norm(post["mean"])


def _golden(name):
    return {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(name + "_")}


@gpu
@pytest.mark.parametrize("name", [str(c) for c in GOLDEN["cases"]])
def test_samples_match_the_reference(name):
    g = _golden(name)
    derivs = [int(d) for d in g["derivs"]]
    gp = capi.GaussianProcess(int(g["kernel"]), 1.0, g["lengths"], g["X"], g["y"], g["noise"], derivs=derivs or None)
    out = gp.sample_joint(g["pts"], derivs_s=derivs or None, table=g["normals"][None], want=("samples", "argmin"))
    np.testing.assert_allclose(out["samples"][0], g["samples"], rtol=1e-9, atol=1e-12)
    # the reference's -1 (minimum at point 0) is 0 here; the one-point case has a single candidate
    assert out["argmin"][0] == (max(0, int(g["argmin_ref"])) if g["has_argmin"] else 0)


@gpu
def test_gpp_sample_point_from_gp_is_the_one_point_joint_draw():
    import GPP

    g = _golden("point")
    derivs = [int(d) for d in g["derivs"]]
    X, dim = g["X"], g["X"].shape[1]
    gpp = GPP.GaussianProcess([1.0, list(g["lengths"])], list(X.ravel()), list(g["y"]), list(g["noise"]), derivs,
                              len(derivs), dim, X.shape[0])
    gp = capi.GaussianProcess(capi.MATERN_NU_2P5, 1.0, g["lengths"], X, g["y"], g["noise"], derivs=derivs)
    gpp.set_explicit_seed(77)
    first = gpp.sample_point_from_gp(list(g["pts"][0]))
    second = gpp.sample_point_from_gp(list(g["pts"][0]))
    assert len(first) == 1 + len(derivs)
    want = gp.sample_joint(g["pts"], derivs_s=derivs, seed=77, first_draw=0)["samples"][0]
    np.testing.assert_array_equal(first, want)
    want2 = gp.sample_joint(g["pts"], derivs_s=derivs, seed=77, first_draw=1)["samples"][0]
    np.testing.assert_array_equal(second, want2)


@gpu
def test_draws_have_the_posterior_mean_and_covariance():
    gp, _, _ = _gp(capi.SQUARE_EXPONENTIAL, 50, 3, 0.4, seed=5)
    pts = np.random.default_rng(6).uniform(size=(8, 3))
    M = 8192
    ys = gp.sample_joint(np.broadcast_to(pts, (M, 8, 3)), seed=123, want=("samples",))["samples"]
    post = gp.posterior(pts[None], want=("mean", "var"))
    mu, var = post["mean"][0], post["var"][0].reshape(8, 8)
    se_mean = np.sqrt(np.diag(var) / M)
    assert np.all(np.abs(ys.mean(axis=0) - mu) <= 5 * se_mean)
    cov = np.cov(ys, rowvar=False)
    d = np.diag(var)
    se_cov = np.sqrt((np.outer(d, d) + var ** 2) / M)
    assert np.all(np.abs(cov - var) <= 5 * se_cov)


@gpu
@pytest.mark.parametrize("num_sets,num_pts,seed,draw", [(1, 1, 0, 0), (3, 7, 5, 11), (4, 1000, 0xC0FFEE, 2**40),
                                                        (2, 8192, 1, 2)])
def test_latin_hypercube_is_bit_identical_to_the_restatement(num_sets, num_pts, seed, draw):
    bounds = np.array([[0.0, 1.0], [-2.0, 3.0], [5.0, 5.5], [1.0, 1.0], [-1e3, 1e3]])
    dev = capi.latin_hypercube(num_sets, num_pts, bounds, seed=seed, first_draw=draw)
    for b in range(num_sets):
        np.testing.assert_array_equal(dev[b], latin_hypercube(seed, draw + b, num_pts, bounds))


@gpu
def test_global_optima_compose_and_do_not_depend_on_chunking():
    gp, _, _ = _gp(capi.SQUARE_EXPONENTIAL, 60, 3, 0.3, seed=9)
    bounds = np.array([[0.0, 1.0], [-1.0, 2.0], [0.5, 0.75]])
    B1, B2, inner = 3, 4, 300
    opt = gp.sample_global_optima(B1 + B2, inner, bounds, seed=42, first_draw=10)
    assert opt.shape == (B1 + B2, 3)
    pts = capi.latin_hypercube(B1 + B2, inner, bounds, seed=42, first_draw=10)
    amin = gp.sample_joint(pts, seed=42, first_draw=10, want=("argmin",))["argmin"]
    np.testing.assert_array_equal(opt, pts[np.arange(B1 + B2), amin])
    split = np.vstack([gp.sample_global_optima(B1, inner, bounds, seed=42, first_draw=10),
                       gp.sample_global_optima(B2, inner, bounds, seed=42, first_draw=10 + B1)])
    np.testing.assert_array_equal(opt, split)
    np.testing.assert_array_equal(opt, gp.sample_global_optima(B1 + B2, inner, bounds, seed=42, first_draw=10))
    assert np.all(opt >= bounds[:, 0]) and np.all(opt <= bounds[:, 1])
    # sample_joint: one call over all sets == per-set calls (a set's draw is independent of its neighbours)
    full = gp.sample_joint(pts[:3], seed=7, first_draw=100, want=("samples", "argmin"))
    for b in range(3):
        one = gp.sample_joint(pts[b], seed=7, first_draw=100 + b, want=("samples", "argmin"))
        np.testing.assert_array_equal(one["samples"][0], full["samples"][b])
        assert one["argmin"][0] == full["argmin"][b]


@gpu
def test_sets_on_both_sides_of_a_chunk_boundary_match_single_set_calls():
    # 4097 sets of 2 points: a chunk holds at most 4096 sets, so set 4096 is drawn in a second chunk
    gp, _, _ = _gp(capi.SQUARE_EXPONENTIAL, 40, 2, 0.3, seed=12)
    sets = np.random.default_rng(13).uniform(size=(4097, 2, 2))
    full = gp.sample_joint(sets, seed=99, first_draw=5, want=("samples", "argmin", "mean", "chol"))
    for b in (0, 4095, 4096):
        one = gp.sample_joint(sets[b], seed=99, first_draw=5 + b, want=("samples", "argmin", "mean", "chol"))
        for k in ("samples", "argmin", "mean", "chol"):
            np.testing.assert_array_equal(one[k][0], full[k][b])
    table = np.random.default_rng(14).standard_normal((4097, 2))
    full_t = gp.sample_joint(sets, table=table)["samples"]
    np.testing.assert_array_equal(full_t[4096], gp.sample_joint(sets[4096], table=table[4096:])["samples"][0])


@gpu
def test_singular_set_reports_the_leading_minor_and_jitter_recovers():
    gp, args, _ = _gp(capi.SQUARE_EXPONENTIAL, 40, 3, 0.3, seed=3, noise=1e-8)
    X = args[3]
    rng = np.random.default_rng(4)
    near = X[0] + 1e-3
    pts = np.vstack([near, near, rng.uniform(size=(6, 3))])
    var = gp.posterior(pts[None], want=("var",))["var"][0].reshape(8, 8)
    rc, _ = checker().cholesky(var)
    assert rc > 0
    with pytest.raises(capi.SingularMatrixError) as e:
        gp.sample_joint(np.stack([pts, rng.uniform(size=(8, 3))])[::-1].copy())
    assert e.value.info == rc
    out = gp.sample_joint(pts, jitter=1e-6, want=("samples", "argmin"))
    assert np.all(np.isfinite(out["samples"]))
    with pytest.raises(capi.InvalidValueError):
        gp.sample_joint(pts, jitter=-1.0)
    with pytest.raises(capi.InvalidValueError):
        gp.sample_joint(pts, jitter=np.nan)
    with pytest.raises(capi.BoundsError):
        gp.sample_joint(np.zeros((1, 8193, 3)))
    with pytest.raises(capi.BoundsError):
        gp.sample_joint(pts, derivs_s=[3])


@gpu
def test_gpp_seeds_replay_and_advance():
    import GPP

    rng = np.random.default_rng(8)
    X = rng.uniform(size=(30, 2))
    y = np.sin(3 * X).sum(axis=1)
    gpp = GPP.GaussianProcess([1.0, [0.3, 0.3]], list(X.ravel()), list(y), [1e-2], [], 0, 2, 30)
    bounds = [0.0, 1.0, -1.0, 1.0]
    gpp.set_explicit_seed(5)
    a = gpp.sample_global_optima(4, 200, bounds)
    b = gpp.sample_global_optima(4, 200, bounds)
    assert len(a) == 8 and a != b
    gpp.set_explicit_seed(5)
    assert gpp.sample_global_optima(4, 200, bounds) == a
    gpp.reset_to_most_recent_seed()
    assert gpp.sample_global_optima(4, 200, bounds) == a
    opt = np.array(a).reshape(4, 2)
    assert np.all(opt[:, 0] >= 0.0) and np.all(opt[:, 0] <= 1.0)
    assert np.all(opt[:, 1] >= -1.0) and np.all(opt[:, 1] <= 1.0)
    p1 = gpp.sample_point_from_gp([0.5, 0.5])
    p2 = gpp.sample_point_from_gp([0.5, 0.5])
    assert p1 != p2
    with pytest.raises(GPP.BoundsException):
        gpp.sample_global_optima(2, 10, [0.0, 1.0])
    with pytest.raises(GPP.SingularMatrixException):
        gpp2 = GPP.GaussianProcess([1.0, [0.3, 0.3]], list(X.ravel()), list(y), [0.0], [], 0, 2, 30)
        gpp2.sample_point_from_gp(list(X[0]))


def _kernel_sass(name):
    obj = os.path.join(ROOT, "cornell-moe_b200", "build", "sample.o")
    if not os.path.exists(obj) or shutil.which("cuobjdump") is None:
        pytest.skip("object file or cuobjdump not available (run __graft_entry__.build() first)")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    parts = [p for p in sass.split("Function : ")[1:] if name in p.split("\n", 1)[0]]
    assert parts, name
    return "".join(parts)


@pytest.mark.parametrize("kernel", ["cov_tile_kernel", "chol_update_kernel"])
def test_tile_kernels_issue_full_rate_dmma(kernel):
    sass = _kernel_sass(kernel)
    assert "DMMA.16x8x4" in sass
    assert "DMMA.8x8x4" not in sass

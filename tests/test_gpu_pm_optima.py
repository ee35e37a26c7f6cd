"""Per-member posterior-mean optima on the device (cmoe_posterior_mean_optima_mcmc, capi and GPP bindings): against the
CPU checker through tests/pm_optima_ref.py, against cmoe_posterior_mean_mcmc for the screen (bit for bit), against the
loop of single-GP calls it replaces, batch and chunk invariance, members of different sizes, the q-KG hand-over and
the edges of the argument contract."""
import ctypes
import os
import sys

import numpy as np
import pytest

import pm_optima_ref
from cornell_moe_b200 import capi
from gpu_util import checker
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
gpu = pytest.mark.gpu
LONG_GD = [1, 50, 3, 0, 0.7, 1.0, 0.2, 1e-8]


def make_ensemble(kernel, g_idx, M=4, N=30, dim=3, seed=3):
    """(problem, device ensemble, hyper-parameters [M, 1 + dim]); the members share the data."""
    prob = make_problem(N, dim, g_idx=g_idx, seed=seed, noise=0.05)
    rng = np.random.default_rng(seed + 100)
    hypers = np.concatenate([rng.uniform(0.8, 1.5, size=(M, 1)), rng.uniform(0.4, 0.9, size=(M, dim))], axis=1)
    noises = np.full((M, 1 + len(g_idx)), 0.05)
    ens = capi.GaussianProcessEnsemble(hypers, noises, prob["X"], prob["y"], derivs=prob["derivs"], kernel=kernel)
    return prob, ens, hypers


def checker_members(kernel, prob, hypers, Xs=None, ys=None):
    out = []
    for m, h in enumerate(hypers):
        gp, lm = checker().gp(kernel, h[0], h[1:], prob["X"] if Xs is None else Xs[m],
                              prob["y"] if ys is None else ys[m], prob["noise"], prob["derivs"])
        assert lm == 0
        out.append(gp)
    return out


def loop_of_single_calls(members, sampled, pts, gd, bounds, nf, include_sampled, shared):
    """What the call replaces: per member one posterior call for the screen, one posterior_mean_optimization, the
    fallback, and one posterior call for best_so_far (stage 2 of profiles/suggest_probe.py)."""
    dim = members[0].dim
    ps = dim - nf

    def mean(gp, p):
        full = np.ones((len(p), dim))
        full[:, :ps] = p
        return gp.posterior(full[:, None, :], (), ("mean",))["mean"].ravel()

    rows = []
    for m, gp in enumerate(members):
        p = pts[m] if pts.ndim == 3 else pts
        if include_sampled:
            p = np.concatenate([p, sampled[m][:, :ps]])
        mu = mean(gp, p)
        i0 = int(np.argmin(mu))
        point, kept = p[i0].copy(), True
        if gd[2] > 0:
            end, val, _ = capi.posterior_mean_optimization(gp, p[i0], gd, bounds, nf)
            kept = -val > mu.min()
            if not kept:
                point = end
        disc = np.concatenate([np.reshape(shared, (-1, ps)), point[None]])
        rows.append((point, i0, kept, mu.min(), disc, mean(gp, disc).min()))
    cols = list(zip(*rows))
    return pm_optima_ref.Optima(np.array(cols[0]), None, np.array(cols[1]), np.array(cols[2], dtype=int),
                                np.array(cols[3]), np.array(cols[4]), np.array(cols[5]))


def assert_same_bits(a, b, members=None):
    for name in a._fields:
        x, y = getattr(a, name), getattr(b, name)
        if x is None or y is None:
            continue
        if members is not None:
            x, y = x[members], y[members]
        np.testing.assert_array_equal(x, y, err_msg=name)


@gpu
@pytest.mark.parametrize("kernel,g_idx,nf", [(0, (), 0), (1, (), 0), (1, (0, 2), 0), (0, (1,), 1), (1, (), 1)])
def test_against_the_checker(kernel, g_idx, nf):
    prob, ens, hypers = make_ensemble(kernel, g_idx)
    ps = prob["dim"] - nf
    rng = np.random.default_rng(17)
    pts, shared = rng.uniform(size=(200, ps)), rng.uniform(size=(6, ps))
    out = ens.posterior_mean_optima(pts, LONG_GD, unit_bounds(ps), nf, True, shared)
    ref = pm_optima_ref.optima(checker_members(kernel, prob, hypers), prob["X"], pts, LONG_GD, unit_bounds(ps), nf, True,
                               shared)
    np.testing.assert_array_equal(out.start_index, ref.start_index)
    np.testing.assert_array_equal(out.kept_start, ref.kept_start)
    # tolerances as for the single-GP call (tests/test_gpu_mcmc.py::test_posterior_mean_optimization): the descent stops
    # on a 1e-8 step tolerance, so the end point is defined to about 1e-8; the mean is flat there
    np.testing.assert_allclose(out.optima, ref.optima, rtol=1e-7, atol=1e-7)
    np.testing.assert_allclose(out.means, ref.means, rtol=1e-9)
    np.testing.assert_allclose(out.screen_min, ref.screen_min, rtol=1e-9)
    np.testing.assert_allclose(out.best_so_far, ref.best_so_far, rtol=1e-9)
    np.testing.assert_array_equal(out.discrete_pts[:, :6], np.broadcast_to(shared, (len(ens), 6, ps)))
    np.testing.assert_array_equal(out.discrete_pts[:, 6], out.optima)


@gpu
@pytest.mark.parametrize("kernel,g_idx,nf", [(1, (), 0), (0, (0,), 1)])
def test_screen_is_the_ensemble_screen_bit_for_bit(kernel, g_idx, nf):
    prob, ens, _ = make_ensemble(kernel, g_idx)
    ps = prob["dim"] - nf
    rng = np.random.default_rng(5)
    pts = rng.uniform(size=(3000, ps))
    _, member_values = ens.posterior_mean(pts, nf, per_member=True)
    out = ens.posterior_mean_optima(pts, EXAMPLE_INNER_GD, unit_bounds(ps), nf, include_sampled=False)
    np.testing.assert_array_equal(out.start_index, np.argmin(-member_values, axis=1))
    np.testing.assert_array_equal(out.screen_min, (-member_values).min(axis=1))
    # with the sampled points: an index past num_points names a sampled point.  Three given points far from the data
    # cannot win against the data's own minimum.
    far = np.full((3, ps), 0.999)
    everything = np.concatenate([far, prob["X"][:, :ps]])
    _, member_values = ens.posterior_mean(everything, nf, per_member=True)
    out = ens.posterior_mean_optima(far, [1, 6, 0, 3, 0.0, 1.0, 0.1, 1e-10], unit_bounds(ps), nf, include_sampled=True)
    np.testing.assert_array_equal(out.start_index, np.argmin(-member_values, axis=1))
    assert (out.start_index >= 3).any()
    np.testing.assert_array_equal(out.optima, everything[out.start_index])
    np.testing.assert_array_equal(out.screen_min, (-member_values).min(axis=1))
    # ties go to the lowest index
    dup = np.concatenate([pts[:50], pts[:50]])
    out = ens.posterior_mean_optima(dup, EXAMPLE_INNER_GD, unit_bounds(ps), nf, include_sampled=False)
    assert (out.start_index < 50).all()


@gpu
@pytest.mark.parametrize("N,one_slice", [(40, True), (300, False)])
def test_against_the_loop_of_single_calls(N, one_slice):
    prob, ens, _ = make_ensemble(1, (), M=5, N=N, dim=3, seed=8)
    rng = np.random.default_rng(23)
    pts, shared = rng.uniform(size=(500, 3)), rng.uniform(size=(10, 3))
    sampled = [prob["X"]] * len(ens)
    for gd in (EXAMPLE_INNER_GD, LONG_GD):
        out = ens.posterior_mean_optima(pts, gd, unit_bounds(3), 0, True, shared)
        loop = loop_of_single_calls(ens.members, sampled, pts, gd, unit_bounds(3), 0, True, shared)
        np.testing.assert_array_equal(out.start_index, loop.start_index)
        np.testing.assert_array_equal(out.screen_min, loop.screen_min)
        np.testing.assert_array_equal(out.kept_start, loop.kept_start)
        if one_slice:  # N (1 + g) < 128 rows: one warp, the single-GP kernel's row order
            assert_same_bits(out, loop)
        else:
            np.testing.assert_allclose(out.optima, loop.optima, rtol=1e-7, atol=1e-7)
            np.testing.assert_allclose(out.best_so_far, loop.best_so_far, rtol=1e-9)


@gpu
def test_a_member_gives_the_same_bits_alone_shared_or_per_member_chunked_or_not():
    prob, ens, _ = make_ensemble(1, (), M=16, N=20, dim=2, seed=12)
    rng = np.random.default_rng(31)
    # 16 members x 600000 points: 9.6e6 CTAs in the screen's grid.x (more than 65535 x 8), and with 16 + 2 doubles per
    # screen index two chunks of the 64 MiB workspace; the one-member call takes a single chunk
    pts, shared = rng.uniform(size=(600000, 2)), rng.uniform(size=(4, 2))
    assert 8 * (16 + 2) * len(pts) > 64 << 20 > 8 * (1 + 2) * len(pts)
    out = ens.posterior_mean_optima(pts, LONG_GD, unit_bounds(2), 0, True, shared)
    for m in (0, 7, 15):
        alone = capi.GaussianProcessEnsemble.from_members([ens.members[m]]).posterior_mean_optima(
            pts, LONG_GD, unit_bounds(2), 0, True, shared)
        assert_same_bits(alone, pm_optima_ref.Optima(*[v[m:m + 1] for v in out]))
    # the minimum in the second chunk, and the same points given per member
    small = pts[:2000]
    out = ens.posterior_mean_optima(small, LONG_GD, unit_bounds(2), 0, True, shared)
    per = ens.posterior_mean_optima(np.broadcast_to(small, (16,) + small.shape), LONG_GD, unit_bounds(2), 0, True, shared)
    assert_same_bits(out, per)
    moved = np.concatenate([np.full((500000, 2), 0.999), small])
    late = ens.posterior_mean_optima(moved, LONG_GD, unit_bounds(2), 0, False, shared)
    first = ens.posterior_mean_optima(small, LONG_GD, unit_bounds(2), 0, False, shared)
    np.testing.assert_array_equal(late.start_index, first.start_index + 500000)
    np.testing.assert_array_equal(late.optima, first.optima)
    np.testing.assert_array_equal(late.best_so_far, first.best_so_far)


@gpu
def test_members_with_different_numbers_of_points():
    prob, ens, hypers = make_ensemble(1, (), M=4, N=20, dim=2, seed=5)
    rng = np.random.default_rng(7)
    new, new_y = rng.uniform(size=(150, 2)), rng.standard_normal(150) * 0.3
    ens.members[1].add_sampled_points(new, new_y)
    ens.members[3].add_sampled_points(new[:2], new_y[:2])
    mixed = capi.GaussianProcessEnsemble.from_members(ens.members)
    assert [gp.N for gp in mixed.members] == [20, 170, 20, 22]
    extra = {1: 150, 3: 2}
    Xs = [np.vstack([prob["X"], new[:extra.get(m, 0)]]) for m in range(4)]
    ys = [np.concatenate([prob["y"], new_y[:extra.get(m, 0)]]) for m in range(4)]
    pts, shared = rng.uniform(size=(100, 2)), rng.uniform(size=(3, 2))
    out = mixed.posterior_mean_optima(pts, LONG_GD, unit_bounds(2), 0, True, shared)
    ref = pm_optima_ref.optima(checker_members(1, prob, hypers, Xs, ys), Xs, pts, LONG_GD, unit_bounds(2), 0, True, shared)
    np.testing.assert_array_equal(out.start_index, ref.start_index)
    np.testing.assert_array_equal(out.kept_start, ref.kept_start)
    np.testing.assert_allclose(out.optima, ref.optima, rtol=1e-7, atol=1e-7)
    np.testing.assert_allclose(out.best_so_far, ref.best_so_far, rtol=1e-9)
    loop = loop_of_single_calls(mixed.members, Xs, pts, LONG_GD, unit_bounds(2), 0, True, shared)
    assert_same_bits(out, loop, members=[0, 2, 3])  # one row slice each
    np.testing.assert_allclose(out.optima[1], loop.optima[1], rtol=1e-7, atol=1e-7)
    # a sampled point of the larger member only: its index is past the other members' lists
    only = mixed.posterior_mean_optima(np.full((1, 2), 0.999), [1, 6, 0, 3, 0.0, 1.0, 0.1, 1e-10], unit_bounds(2))
    np.testing.assert_array_equal(only.optima[1], np.concatenate([[[0.999, 0.999]], Xs[1]])[only.start_index[1]])


@gpu
def test_outputs_feed_the_ensemble_kg():
    prob, ens, _ = make_ensemble(1, (), M=3, N=18, dim=3, seed=44)
    rng = np.random.default_rng(3)
    pts, shared = rng.uniform(size=(300, 3)), rng.uniform(size=(5, 3))
    out = ens.posterior_mean_optima(pts, EXAMPLE_INNER_GD, unit_bounds(3), 0, True, shared)
    loop = loop_of_single_calls(ens.members, [prob["X"]] * 3, pts, EXAMPLE_INNER_GD, unit_bounds(3), 0, True, shared)
    cands = rng.uniform(size=(4, 2, 3))
    args = (cands, None, 32)
    rest = (EXAMPLE_INNER_GD, unit_bounds(3))
    np.testing.assert_array_equal(ens.kg(*args, out.best_so_far, *rest, out.discrete_pts, seed=9),
                                  ens.kg(*args, loop.best_so_far, *rest, loop.discrete_pts, seed=9))


@gpu
def test_edges():
    prob, ens, _ = make_ensemble(0, (), M=3, N=25, dim=2, seed=2)
    rng = np.random.default_rng(1)
    pts = rng.uniform(size=(64, 2))
    # one point, no shared points, no sampled points: the discretisation set is the optimum alone
    out = ens.posterior_mean_optima(pts[:1], LONG_GD, unit_bounds(2), include_sampled=False)
    assert out.discrete_pts.shape == (3, 1, 2) and (out.start_index == 0).all()
    np.testing.assert_array_equal(out.discrete_pts[:, 0], out.optima)
    full = [gp.posterior(out.optima[m][None, None, :], (), ("mean",))["mean"].ravel()[0]
            for m, gp in enumerate(ens.members)]
    np.testing.assert_array_equal(out.best_so_far, full)
    # no restart: the start is the answer; no step: the descent evaluates the start and does not move
    for gd in ([1, 50, 0, 0, 0.7, 1.0, 0.2, 1e-8], [1, 50, -1, 0, 0.7, 1.0, 0.2, 1e-8]):
        out = ens.posterior_mean_optima(pts, gd, unit_bounds(2), include_sampled=False)
        assert out.kept_start.all()
        np.testing.assert_array_equal(out.optima, pts[out.start_index])
        np.testing.assert_array_equal(out.means, out.screen_min)
    out = ens.posterior_mean_optima(pts, [1, 0, 2, 0, 0.7, 1.0, 0.2, 1e-8], unit_bounds(2), include_sampled=False)
    np.testing.assert_array_equal(out.optima, pts[out.start_index])
    np.testing.assert_allclose(out.means, out.screen_min, rtol=1e-12)
    # a screen point outside the box is allowed
    ens.posterior_mean_optima(pts * 3.0 - 1.0, EXAMPLE_INNER_GD, unit_bounds(2))


@gpu
def test_input_checks_that_need_a_handle():
    prob, ens, _ = make_ensemble(1, (), M=2, N=10, dim=2)
    pts = np.full((4, 2), 0.5)
    for nf in (2, 3):
        buf, info, p = np.zeros(16), ctypes.c_int(), capi.GDParams.from_seq(EXAMPLE_INNER_GD)
        rc = capi.lib().cmoe_posterior_mean_optima_mcmc(ens._handles(), 2, nf, ctypes.byref(p), capi._d(buf),
                                                        capi._d(buf), 1, 0, 1, None, 0, capi._d(buf), None, None, None,
                                                        None, None, None, ctypes.byref(info))
        assert rc == capi.ERR_BOUNDS and "num_fidelity" in capi.lib().cmoe_last_error().decode()
    with pytest.raises(capi.BoundsError, match="EMPTY"):
        ens.posterior_mean_optima(pts, EXAMPLE_INNER_GD, [0.0, 1.0, 1.0, 0.0])
    bad = pts.copy()
    bad[2, 1] = np.nan
    with pytest.raises(capi.InvalidValueError, match="finite"):
        ens.posterior_mean_optima(bad, EXAMPLE_INNER_GD, unit_bounds(2))
    with pytest.raises(capi.InvalidValueError, match="finite"):
        ens.posterior_mean_optima(pts, EXAMPLE_INNER_GD, unit_bounds(2), shared_discrete=[[0.1, np.inf]])
    other = capi.GaussianProcess(capi.MATERN_NU_2P5, 1.0, [0.5] * 3, np.zeros((2, 3)) + [[0.0], [1.0]], [0.0, 1.0],
                                 [0.01])
    with pytest.raises(capi.InvalidValueError):
        capi.GaussianProcessEnsemble.from_members([ens.members[0], other]).posterior_mean_optima(
            pts, EXAMPLE_INNER_GD, unit_bounds(2))


@gpu
def test_gpp_entry_agrees_with_capi():
    import GPP  # noqa: E402

    prob, ens, hypers = make_ensemble(1, (), M=3, N=16, dim=3, seed=6)
    X, y, dim, nf = prob["X"], prob["y"], 3, 1
    ps = dim - nf
    noises = np.full((3, 1), 0.05)
    mcmc = GPP.GaussianProcessMCMC(list(hypers.ravel()), list(noises.ravel()), list(X.ravel()), list(y), [], 3, 0, dim,
                                   X.shape[0])
    wrappers = [type("Wrapper", (), {"_gaussian_process": GPP.GaussianProcess(
        [h[0], list(h[1:])], list(X.ravel()), list(y), [0.05], [], 0, dim, X.shape[0])})() for h in hypers]
    rng = np.random.default_rng(2)
    pts, shared = rng.uniform(size=(50, ps)), rng.uniform(size=(4, ps))
    out = ens.posterior_mean_optima(pts, EXAMPLE_INNER_GD, unit_bounds(ps), nf, True, shared)
    params = GPP.GradientDescentParameters(*EXAMPLE_INNER_GD)
    for gps in (mcmc, wrappers):
        disc, best, optima = GPP.posterior_mean_optima_mcmc(gps, nf, params, list(unit_bounds(ps)), list(pts.ravel()),
                                                            50, list(shared.ravel()), 4)
        np.testing.assert_array_equal(np.reshape(disc, (3, 5, ps)), out.discrete_pts)
        np.testing.assert_array_equal(best, out.best_so_far)
        np.testing.assert_array_equal(np.reshape(optima, (3, ps)), out.optima)
    disc, best, optima = GPP.posterior_mean_optima_mcmc(mcmc, nf, params, list(unit_bounds(ps)), list(pts.ravel()), 50,
                                                        [], 0, include_sampled=False)
    none = ens.posterior_mean_optima(pts, EXAMPLE_INNER_GD, unit_bounds(ps), nf, False)
    np.testing.assert_array_equal(np.reshape(optima, (3, ps)), none.optima)
    np.testing.assert_array_equal(np.reshape(disc, (3, 1, ps)), none.discrete_pts)

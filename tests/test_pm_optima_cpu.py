"""CPU checks of the per-member posterior-mean optima (cmoe_posterior_mean_optima_mcmc): the host restatement
(tests/pm_optima_ref.py) on the CPU checker, the argument errors that are reported before a device is needed, and the
GPP name."""
import ctypes
import os
import sys

import numpy as np

import oracle as orc
import pm_optima_ref
from cornell_moe_b200 import capi
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))


def checker():
    return orc.load_reference() if orc.have_reference() else orc.load_oracle()


def small_ensemble(kernel=1, nf=0, g_idx=(), M=3, N=14, dim=3):
    prob = make_problem(N, dim, g_idx=g_idx, seed=21, noise=0.05)
    rng = np.random.default_rng(4)
    gps = []
    for _ in range(M):
        gp, lm = checker().gp(kernel, rng.uniform(0.8, 1.5), rng.uniform(0.4, 0.9, size=dim), prob["X"], prob["y"],
                              prob["noise"], prob["derivs"])
        assert lm == 0
        gps.append(gp)
    return prob, gps


def test_restatement_on_the_checker():
    nf = 1
    prob, gps = small_ensemble(nf=nf)
    ps = prob["dim"] - nf
    rng = np.random.default_rng(9)
    pts, shared = rng.uniform(size=(40, ps)), rng.uniform(size=(5, ps))
    gd = [1, 50, 3, 0, 0.7, 1.0, 0.2, 1e-8]
    out = pm_optima_ref.optima(gps, prob["X"], pts, gd, unit_bounds(ps), nf, True, shared)
    screen = np.concatenate([pts, prob["X"][:, :ps]])
    assert out.start_index.max() < len(screen) and out.discrete_pts.shape == (3, 6, ps)
    for m, gp in enumerate(gps):
        full = np.ones((len(screen), prob["dim"]))
        full[:, :ps] = screen
        mu = gp.mean_additional(full)
        assert out.start_index[m] == np.argmin(mu) and out.screen_min[m] == mu.min()
        end, f_end = gp.posterior_mean_optimization(screen[out.start_index[m]], gd, unit_bounds(ps), nf)
        assert not out.kept_start[m]  # the line search only accepts steps that lower the mean
        np.testing.assert_array_equal(out.optima[m], end)
        assert out.means[m] == -f_end and out.means[m] <= out.screen_min[m]
        np.testing.assert_array_equal(out.discrete_pts[m, :5], shared)
        np.testing.assert_array_equal(out.discrete_pts[m, 5], out.optima[m])
        assert out.best_so_far[m] <= out.means[m] + 1e-12 * max(1.0, abs(out.means[m]))
    # per-member lists: member m screens its own points
    per = rng.uniform(size=(3, 7, ps))
    out = pm_optima_ref.optima(gps, prob["X"], per, gd, unit_bounds(ps), nf, False, None)
    for m in range(3):
        one = pm_optima_ref.optima(gps[m:m + 1], prob["X"], per[m], gd, unit_bounds(ps), nf, False, None)
        np.testing.assert_array_equal(one.optima[0], out.optima[m])
        assert one.start_index[0] == out.start_index[m] < 7 and out.discrete_pts.shape == (3, 1, ps)


def test_no_restart_keeps_the_start_and_a_worse_end_point_falls_back():
    prob, gps = small_ensemble()
    pts = np.random.default_rng(2).uniform(size=(10, 3))
    out = pm_optima_ref.optima(gps, prob["X"], pts, [1, 50, 0, 0, 0.7, 1.0, 0.2, 1e-8], unit_bounds(3), 0, False)
    assert out.kept_start.all()
    np.testing.assert_array_equal(out.optima, pts[out.start_index])
    np.testing.assert_array_equal(out.means, out.screen_min)

    class EndsHigher:
        """A member whose descent reports a mean above the screened minimum (the two are computed by different sums
        on the device, so a descent that does not move can end an ulp higher): main.py:191-193 keeps the start."""
        dim = 3

        def __init__(self, gp):
            self.gp = gp

        def mean_additional(self, x):
            return self.gp.mean_additional(x)

        def posterior_mean_optimization(self, x0, gd, bounds, num_fidelity=0):
            return np.full(3, 0.5), -(float(self.gp.mean_additional(x0[None])[0]) + 1e-9)

    out = pm_optima_ref.optima([EndsHigher(gps[0])], prob["X"], pts, EXAMPLE_INNER_GD, unit_bounds(3), 0, False)
    assert out.kept_start[0] == 1 and out.means[0] == out.screen_min[0]
    np.testing.assert_array_equal(out.optima[0], pts[out.start_index[0]])
    np.testing.assert_array_equal(out.discrete_pts[0, -1], out.optima[0])


def _call(gps=None, num_gp=1, nf=0, params=True, bounds=True, points=True, optima=True, num_points=1, shared=False,
          num_shared=0, steps=6):
    p = capi.GDParams(1, steps, 1, 3, 0.0, 1.0, 0.1, 1e-10)
    buf = np.zeros(8)
    info = ctypes.c_int()
    return capi.lib().cmoe_posterior_mean_optima_mcmc(
        gps, num_gp, nf, ctypes.byref(p) if params else None, capi._d(buf) if bounds else None,
        capi._d(buf) if points else None, num_points, 0, 1, capi._d(buf) if shared else None, num_shared,
        capi._d(buf) if optima else None, None, None, None, None, None, None, ctypes.byref(info))


def _last_error():
    return capi.lib().cmoe_last_error().decode()


def test_input_checks_need_no_device():
    for missing in ("params", "bounds", "points", "optima"):
        assert _call(**{missing: False}) == capi.ERR_INVALID_VALUE and "NULL" in _last_error()
    assert _call(num_shared=2) == capi.ERR_INVALID_VALUE and "shared_discrete" in _last_error()
    assert _call(num_points=0) == capi.ERR_BOUNDS and "num_points" in _last_error()
    assert _call(shared=True, num_shared=-1) == capi.ERR_BOUNDS and "num_shared" in _last_error()
    assert _call(steps=(1 << 20) + 1) == capi.ERR_BOUNDS and "max_num_steps" in _last_error()
    assert _call(nf=-1) == capi.ERR_BOUNDS and "num_fidelity" in _last_error()
    # NULL or empty ensemble, NULL member (num_fidelity >= dim, an empty box and non-finite points need a GP handle:
    # tests/test_gpu_pm_optima.py)
    one_null = (ctypes.c_void_p * 1)(None)
    assert _call(None, 1) == capi.ERR_BOUNDS and "ensemble" in _last_error()
    assert _call(one_null, 0) == capi.ERR_BOUNDS and "ensemble" in _last_error()
    assert _call(one_null, 1) == capi.ERR_INVALID_VALUE and "NULL GP" in _last_error()


def test_gpp_has_the_name_and_its_keywords():
    import GPP  # noqa: E402

    doc = GPP.posterior_mean_optima_mcmc.__doc__
    for arg in ("gps", "num_fidelity", "optimizer_parameters", "domain_bounds", "points", "num_points",
                "shared_discrete_pts", "num_shared", "include_sampled"):
        assert arg in doc, (arg, doc)
    assert hasattr(capi.GaussianProcessEnsemble, "posterior_mean_optima")
    assert capi.PosteriorMeanOptima._fields == ("optima", "means", "start_index", "kept_start", "screen_min",
                                                "discrete_pts", "best_so_far")

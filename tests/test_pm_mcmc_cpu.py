"""CPU checks of the ensemble posterior-mean path: the host restatement (tests/pm_mcmc_ref.py) against the reference's
answers in tests/golden/reference_pm_mcmc.npz, the new GPP names, and the input checks that need no device."""
import ctypes
import os
import sys

import numpy as np
import pytest

import oracle as orc
import pm_mcmc_ref
from cornell_moe_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "reference_pm_mcmc.npz"))


def golden_case(name):
    return {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(name + "_")}


def restated_objective(backend, g):
    derivs = [int(d) for d in g["derivs"]]
    gps = []
    for h, noise in zip(g["hypers"], g["noises"]):
        gp, lm = backend.gp(int(g["kernel"]), h[0], h[1:], g["X"], g["y"], noise, derivs=derivs)
        assert lm == 0
        gps.append(gp)
    return pm_mcmc_ref.ensemble_objective(
        [(lambda x, gp=gp: float(gp.mean_additional(x)[0])) for gp in gps],
        [(lambda x, gp=gp: gp.posterior(x, want=("grad_mean",))["grad_mean"]) for gp in gps], g["X"].shape[1],
        int(g["num_fidelity"])), gps


def restated_params(g):
    p = g["params"]
    return int(p[1]), int(p[3]), float(p[4]), float(p[5]), float(p[6])


@pytest.mark.parametrize("name", [str(c) for c in GOLDEN["cases"]])
def test_restatement_matches_reference_answers(name):
    """With the reference's compiled means the restatement is the reference's arithmetic (the generator checks it bit
    for bit); with the C restatement of the means the trajectories agree to rounding."""
    g = golden_case(name)
    backend = orc.load_reference() if orc.have_reference() else orc.load_oracle()
    (f, grad_f), _ = restated_objective(backend, g)
    params = restated_params(g)
    pts, vals, best, _, idx = pm_mcmc_ref.multistart(f, grad_f, g["starts"], params, g["bounds"])
    np.testing.assert_allclose(pts, g["points"], rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(vals, g["values"], rtol=1e-9, atol=1e-11)
    assert idx == int(g["best_index"])
    np.testing.assert_allclose(best, g["best_point"], rtol=1e-9, atol=1e-11)
    report, _, screen = pm_mcmc_ref.recommend(f, grad_f, g["eval_pts"], params, g["bounds"])
    np.testing.assert_allclose(screen, g["screen"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(report, g["report_point"], rtol=1e-9, atol=1e-11)


def test_golden_covers_the_edge_cases():
    navs = {int(golden_case(c)["params"][3]) for c in GOLDEN["cases"]}
    assert {0, -1} <= navs and any(n > int(golden_case(c)["params"][1]) for c in GOLDEN["cases"]
                                   for n in [int(golden_case(c)["params"][3])])
    assert any(float(golden_case(c)["params"][6]) == 1.0 for c in GOLDEN["cases"])
    assert any(int(golden_case(c)["num_fidelity"]) == 1 for c in GOLDEN["cases"])
    assert any(golden_case(c)["derivs"].size > 0 for c in GOLDEN["cases"])
    # a start on the boundary does not move along the coordinate it touches when mrc * dist = 0
    g = golden_case("navneg")
    on = g["starts"][2]
    assert np.all(on == g["bounds"][:, 1]) and np.all(g["points"][2] == on)
    # duplicate best starts: the first one is reported
    d = golden_case("dup")
    assert d["values"][1] == d["values"][2] == d["values"][4] and int(d["best_index"]) == 1


def test_averaging_range_matches_the_python_optimiser():
    assert pm_mcmc_ref.averaging_range(-1, 7) == (1, 8)
    assert pm_mcmc_ref.averaging_range(0, 7) == (7, 8)
    assert pm_mcmc_ref.averaging_range(3, 7) == (5, 8)
    assert pm_mcmc_ref.averaging_range(20, 7) == (1, 8)


def test_gpp_has_the_ensemble_names():
    import GPP  # noqa: E402

    for name, args in [("compute_posterior_mean_mcmc_of_points", ("gps", "num_fidelity", "points", "num_points")),
                       ("compute_grad_posterior_mean_mcmc_of_points", ("gps", "num_fidelity", "points", "num_points")),
                       ("posterior_mean_mcmc_optimization", ("gps", "num_fidelity", "optimizer_parameters",
                                                             "domain_bounds", "starting_points", "num_starts"))]:
        doc = getattr(GPP, name).__doc__
        assert all(a in doc for a in args), (name, doc)


def _opt(gps, num_gp, nf, steps=10, starts=1, bounds=(0.0, 1.0)):
    params = capi.GDParams(1, steps, 1, 3, 0.5, 1.0, 0.5, 1e-10)
    db = np.array(bounds * 4, dtype=np.float64)
    st = np.zeros(8)
    out = np.zeros(8)
    bv, info = ctypes.c_double(), ctypes.c_int()
    return capi.lib().cmoe_posterior_mean_mcmc_optimization(
        gps, num_gp, nf, ctypes.byref(params), capi._d(db), capi._d(st), starts, capi._d(out), capi._d(out),
        capi._d(out), ctypes.byref(bv), ctypes.byref(info))


def _screen(gps, num_gp, nf, num_points=1):
    pts, out = np.zeros(8), np.zeros(8)
    info = ctypes.c_int()
    return capi.lib().cmoe_posterior_mean_mcmc(gps, num_gp, nf, capi._d(pts), num_points, capi._d(out), None, None,
                                               ctypes.byref(info))


def _last_error():
    return capi.lib().cmoe_last_error().decode()


def test_input_checks_need_no_device():
    one_null = (ctypes.c_void_p * 1)(None)
    # NULL or empty ensemble
    assert _opt(None, 1, 0) == capi.ERR_BOUNDS and "ensemble" in _last_error()
    assert _opt(one_null, 0, 0) == capi.ERR_BOUNDS and "ensemble" in _last_error()
    assert _screen(None, 1, 0) == capi.ERR_BOUNDS and "ensemble" in _last_error()
    assert _screen(one_null, 0, 0) == capi.ERR_BOUNDS and "ensemble" in _last_error()
    # max_num_steps = 0, where the Python optimiser averages an empty range
    assert _opt(None, 1, 0, steps=0) == capi.ERR_BOUNDS and "max_num_steps" in _last_error()
    assert _opt(None, 1, 0, steps=-3) == capi.ERR_BOUNDS and "max_num_steps" in _last_error()
    # no start, no point
    assert _opt(None, 1, 0, starts=0) == capi.ERR_BOUNDS and "num_starts" in _last_error()
    assert _screen(None, 1, 0, num_points=0) == capi.ERR_BOUNDS and "num_points" in _last_error()
    # negative num_fidelity (num_fidelity >= dim and lo > hi need a GP handle: tests/test_gpu_pm_mcmc.py)
    assert _opt(None, 1, -1) == capi.ERR_BOUNDS and "num_fidelity" in _last_error()
    assert _screen(None, 1, -1) == capi.ERR_BOUNDS and "num_fidelity" in _last_error()

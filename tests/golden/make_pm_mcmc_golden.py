"""Regenerates tests/golden/reference_pm_mcmc.npz: the reference's recommendation step on GP ensembles.

The answers come from the reference's own, unmodified Python classes: PosteriorMeanMCMC
(cpp_wrappers/knowledge_gradient_mcmc.py), RepeatedDomain, python_version TensorProductDomain, GradientDescentOptimizer,
GradientDescentParameters and multistart_optimize, driven through the sequence of examples/main.py:243-260.  Two stubs
stand in for what that code imports and this environment lacks:

* ``future.utils.with_metaclass`` and ``past.utils.old_div`` (the Python 2/3 compatibility packages), if not installed;
* ``moe.build.GPP``, the reference's compiled module.  Its ``compute_posterior_mean`` / ``compute_grad_posterior_mean``
  do what ComputePosteriorMeanWrapper does (gpp_python_knowledge_gradient.cpp:44-75): pad the fidelity coordinates with
  1.0, take the member's mean (or its gradient) from the compiled reference in oracle/_ref, and negate.

The reference checkout is CMOE_REFERENCE_CPP's parent's parent's parent, or `reference` beside this repository, and
oracle/_ref/libmoe_ref.so must have been built by __graft_entry__.build().  The script also checks that the host
restatement (tests/pm_mcmc_ref.py), fed the same means, reproduces every answer bit for bit.
Run from the repository root:  python tests/golden/make_pm_mcmc_golden.py
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import oracle as orc  # noqa: E402
import pm_mcmc_ref  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_pm_mcmc.npz")
REF_CPP = os.environ.get("CMOE_REFERENCE_CPP") or os.path.join(os.path.dirname(ROOT), "reference", "moe",
                                                                "optimal_learning", "cpp")
REF_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(REF_CPP))))


def _install_stubs(ref):
    try:
        import future.utils  # noqa: F401
    except ImportError:
        def with_metaclass(meta, *bases):
            class metaclass(meta):
                def __new__(cls, name, this_bases, d):
                    return meta(name, bases, d)
            return type.__new__(metaclass, "temporary_class", (), {})
        fut, fut_utils = types.ModuleType("future"), types.ModuleType("future.utils")
        fut_utils.with_metaclass = with_metaclass
        fut.utils = fut_utils
        sys.modules.update({"future": fut, "future.utils": fut_utils})
    try:
        import past.utils  # noqa: F401
    except ImportError:
        import numbers

        def old_div(a, b):
            if isinstance(a, numbers.Integral) and isinstance(b, numbers.Integral):
                return a // b
            return a / b
        past, past_utils = types.ModuleType("past"), types.ModuleType("past.utils")
        past_utils.old_div = old_div
        past.utils = past_utils
        sys.modules.update({"past": past, "past.utils": past_utils})

    def _full(gp, num_fidelity, pt):
        x = np.ones(gp.dim)
        x[:gp.dim - num_fidelity] = np.asarray(pt, dtype=np.float64).ravel()
        return x

    def compute_posterior_mean(gp, num_fidelity, pt):
        return -float(gp.mean_additional(_full(gp, num_fidelity, pt))[0])

    def compute_grad_posterior_mean(gp, num_fidelity, pt):
        g = gp.posterior(_full(gp, num_fidelity, pt), want=("grad_mean",))["grad_mean"]
        return list(-g[:gp.dim - num_fidelity])

    class RandomnessSourceContainer:
        def __init__(self, num_threads):
            pass

        def SetRandomizedUniformGeneratorSeed(self, seed):
            pass

        def SetRandomizedNormalRNGSeed(self, seed):
            pass

    gpp = types.ModuleType("moe.build.GPP")
    gpp.compute_posterior_mean = compute_posterior_mean
    gpp.compute_grad_posterior_mean = compute_grad_posterior_mean
    gpp.RandomnessSourceContainer = RandomnessSourceContainer
    build = types.ModuleType("moe.build")
    build.GPP = gpp
    sys.path.insert(0, REF_ROOT)
    import moe
    moe.build = build
    sys.modules.update({"moe.build": build, "moe.build.GPP": gpp})


class Member:
    """What PosteriorMeanMCMC holds per hyper-parameter sample: an object with ``_gaussian_process`` and ``dim``."""

    def __init__(self, gp):
        self._gaussian_process = gp
        self.dim = gp.dim


def branin(x):
    a, b, c, r, s, t = 1.0, 5.1 / (4 * np.pi ** 2), 5 / np.pi, 6.0, 10.0, 1 / (8 * np.pi)
    return a * (x[:, 1] - b * x[:, 0] ** 2 + c * x[:, 0] - r) ** 2 + s * (1 - t) * np.cos(x[:, 0]) + s


def case(ref, name, kernel, box, N, M, params, num_fidelity=0, derivs=(), n_eval=200, starts=None, rng_seed=0):
    from moe.optimal_learning.python.cpp_wrappers.knowledge_gradient_mcmc import PosteriorMeanMCMC
    from moe.optimal_learning.python.geometry_utils import ClosedInterval
    from moe.optimal_learning.python.python_version.domain import TensorProductDomain
    from moe.optimal_learning.python.python_version.optimization import (GradientDescentOptimizer,
                                                                         GradientDescentParameters,
                                                                         multistart_optimize)
    from moe.optimal_learning.python.repeated_domain import RepeatedDomain

    rng = np.random.default_rng(rng_seed)
    box = np.asarray(box, dtype=np.float64)  # [dim, 2] incl. fidelity coordinates
    dim = box.shape[0]
    ps = dim - num_fidelity
    g = len(derivs)
    X = box[:, 0] + (box[:, 1] - box[:, 0]) * rng.uniform(size=(N, dim))
    if dim == 2:
        val = branin(X)
    else:
        val = np.sin(3 * X).sum(axis=1) * (1 + X[:, -1])
    val = (val - val.mean()) / val.std()
    y = val if not g else np.column_stack([val] + [np.cos(X[:, d]) for d in derivs]).ravel()
    width = box[:, 1] - box[:, 0]
    hypers = np.column_stack([rng.uniform(0.5, 2.0, M), width * rng.uniform(0.2, 0.5, (M, dim))])
    noises = np.tile(rng.uniform(1e-3, 1e-2, (M, 1)), (1, 1 + g))
    gps = []
    for m in range(M):
        gp, lm = ref.gp(kernel, hypers[m, 0], hypers[m, 1:], X, y, noises[m], derivs=list(derivs))
        assert lm == 0, (name, m, lm)
        gps.append(gp)
    bounds = box[:ps]
    eval_pts = bounds[:, 0] + (bounds[:, 1] - bounds[:, 0]) * rng.uniform(size=(n_eval, ps))
    eval_pts = np.vstack([eval_pts, X[:, :ps]])  # plus every sampled point, as main.py appends them
    if starts is None:
        starts = bounds[:, 0] + (bounds[:, 1] - bounds[:, 0]) * rng.uniform(size=(6, ps))
    starts = np.asarray(starts, dtype=np.float64)
    steps, nav, gamma, pre_mult, mrc = params
    py_params = GradientDescentParameters(max_num_steps=steps, max_num_restarts=3, num_steps_averaged=nav, gamma=gamma,
                                          pre_mult=pre_mult, max_relative_change=mrc, tolerance=1.0e-10)

    # ---- the reference's classes -------------------------------------------------------------------------------
    ps_obj = PosteriorMeanMCMC([Member(gp) for gp in gps], num_fidelity)
    test = np.zeros(eval_pts.shape[0])
    for i, pt in enumerate(eval_pts):
        ps_obj.set_current_point(pt.reshape((1, ps)))
        test[i] = -ps_obj.compute_objective_function()
    domain = RepeatedDomain(num_repeats=1, domain=TensorProductDomain([ClosedInterval(lo, hi) for lo, hi in bounds]))
    opt = GradientDescentOptimizer(domain, ps_obj, py_params)
    # per start, what MultistartOptimizer.optimize does (optimization.py:595-599), keeping each averaged point
    pts, vals = np.empty((len(starts), ps)), np.empty(len(starts))
    for i, s in enumerate(starts):
        opt.objective_function.current_point = s
        opt.optimize()
        pts[i] = opt.objective_function.current_point.ravel()
        vals[i] = opt.objective_function.compute_objective_function()
    best_point, function_values = multistart_optimize(opt, starts)
    np.testing.assert_array_equal(function_values, vals)
    # examples/main.py:252-260
    initial_point = eval_pts[np.argmin(test)].reshape((1, ps))
    report_point = multistart_optimize(opt, initial_point, num_multistarts=1)[0]
    ps_obj.set_current_point(report_point.reshape((1, ps)))
    if -ps_obj.compute_objective_function() > np.min(test):
        report_point = initial_point
    report_point = np.asarray(report_point, dtype=np.float64).ravel()

    # ---- the host restatement on the same means, bit for bit ----------------------------------------------------
    f, grad_f = pm_mcmc_ref.ensemble_objective(
        [(lambda x, gp=gp: float(gp.mean_additional(x)[0])) for gp in gps],
        [(lambda x, gp=gp: gp.posterior(x, want=("grad_mean",))["grad_mean"]) for gp in gps], dim, num_fidelity)
    r_pts, r_vals, r_best, _, r_idx = pm_mcmc_ref.multistart(f, grad_f, starts, params, bounds)
    np.testing.assert_array_equal(r_pts, pts)
    np.testing.assert_array_equal(r_vals, vals)
    np.testing.assert_array_equal(r_best, np.asarray(best_point).ravel())
    r_report, _, r_screen = pm_mcmc_ref.recommend(f, grad_f, eval_pts, params, bounds)
    np.testing.assert_array_equal(r_screen, -test)
    np.testing.assert_array_equal(r_report, report_point)

    return {f"{name}_kernel": kernel, f"{name}_X": X, f"{name}_y": y, f"{name}_noises": noises,
            f"{name}_hypers": hypers, f"{name}_derivs": np.asarray(derivs, dtype=np.int32),
            f"{name}_num_fidelity": num_fidelity, f"{name}_eval_pts": eval_pts, f"{name}_starts": starts,
            f"{name}_params": np.array([1, steps, 3, nav, gamma, pre_mult, mrc, 1.0e-10]), f"{name}_bounds": bounds,
            f"{name}_screen": -test, f"{name}_points": pts, f"{name}_values": vals,
            f"{name}_best_point": np.asarray(best_point, dtype=np.float64).ravel(), f"{name}_best_index": r_idx,
            f"{name}_report_point": report_point}


def main():
    if not orc.have_reference():
        raise SystemExit("oracle/_ref/libmoe_ref.so is missing: run __graft_entry__.build() with a reference checkout")
    ref = orc.load_reference()
    _install_stubs(ref)
    main_params = (1000, 15, 0.7, 1.0, 0.02)  # examples/main.py:115-121
    data = {}
    data.update(case(ref, "branin", 1, [[-5.0, 10.0], [0.0, 15.0]], 20, 4, main_params, rng_seed=1))
    data.update(case(ref, "fidelity", 1, [[0.0, 1.0], [0.0, 1.0], [0.2, 1.0]], 25, 3, main_params, num_fidelity=1,
                     rng_seed=2))
    data.update(case(ref, "derivs", 0, [[0.0, 1.0], [0.0, 1.0]], 15, 3, (300, 10, 0.6, 0.5, 0.1), derivs=(0,),
                     rng_seed=3))
    edge_starts = np.array([[0.3, 0.6], [0.0, 0.5], [1.0, 1.0], [0.7, 0.2]])  # the 2nd and 3rd lie on the boundary
    data.update(case(ref, "nav0", 1, [[0.0, 1.0], [0.0, 1.0]], 12, 2, (7, 0, 0.5, 2.0, 0.5), starts=edge_starts,
                     rng_seed=4))
    data.update(case(ref, "navneg", 1, [[0.0, 1.0], [0.0, 1.0]], 12, 2, (7, -1, 0.5, 2.0, 1.0), starts=edge_starts,
                     rng_seed=4))
    data.update(case(ref, "navbig", 0, [[0.0, 1.0], [0.0, 1.0]], 12, 2, (7, 20, 0.5, 2.0, 1.0), starts=edge_starts,
                     rng_seed=5))
    dup = case(ref, "dup", 1, [[-5.0, 10.0], [0.0, 15.0]], 20, 4, (200, 15, 0.7, 1.0, 0.02), rng_seed=6)
    # duplicate starts: the best one three times, so that the strict `>` keeps the first of them
    s = dup["dup_starts"]
    best = s[int(np.argmax(dup["dup_values"]))]
    data.update(case(ref, "dup", 1, [[-5.0, 10.0], [0.0, 15.0]], 20, 4, (200, 15, 0.7, 1.0, 0.02), rng_seed=6,
                     starts=np.array([s[0], best, best, s[1], best])))
    assert data["dup_values"][1] == data["dup_values"][2] == data["dup_values"][4]
    data["cases"] = np.array(["branin", "fidelity", "derivs", "nav0", "navneg", "navbig", "dup"])
    np.savez(OUT, **data)
    print("wrote", OUT, {c: int(data[f"{c}_best_index"]) for c in data["cases"]})


if __name__ == "__main__":
    main()

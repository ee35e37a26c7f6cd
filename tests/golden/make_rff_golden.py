"""Regenerates tests/golden/reference_rff.npz: the reference's random-feature sampler of the global minimum.

The answers come from the reference's own, unmodified ``sample_gp_with_random_features`` and
``sample_from_global_optima`` (moe/optimal_learning/python/random_features.py).  ``past.utils.old_div`` is stubbed if
the Python 2/3 compatibility package is not installed, and the GP is a small stub object with the attributes the routine
reads (dim, num_sampled, num_derivatives, noise_variance, derivatives, _points_sampled, _points_sampled_value and
get_covariance_copy().get_hyperparameters()).

``numpy.random.randn`` and ``numpy.random.uniform`` are wrapped to record Omega (F x d), u (as b = 2 pi u) and z (the
``randomness`` draw); theta, W and b are read from the returned closure.  The mean m is recorded by a second run that
replays Omega and b and forces z to zeros.  ``scipy.optimize.fmin_slsqp`` is wrapped to record its end point.

Stored per case: the inputs, Omega, b, z, W, theta, m, the grid values, the grid argmin, the SLSQP end point and the
returned point, for the draw and (suffix _m) for the mean's sample function.  The reference checkout is
CMOE_REFERENCE_PY, or `reference` beside this repository.
Run from the repository root:  python tests/golden/make_rff_golden.py
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "reference_rff.npz")
REF_PY = os.environ.get("CMOE_REFERENCE_PY") or os.path.join(os.path.dirname(ROOT), "reference")

# name, n, d, derivs, noise per type, F
CASES = [
    ("chol_m_eq_f_plus_1", 20, 2, (), (1e-2,), 19),
    ("chol_m_eq_f", 20, 2, (), (1e-2,), 20),
    ("woodbury_m_eq_f_minus_1", 20, 2, (), (1e-2,), 21),
    ("woodbury_g2", 10, 2, (0, 1), (1e-2, 4e-2, 9e-2), 100),
    ("chol_d6_g1", 40, 6, (3,), (2e-2, 5e-2), 50),
    ("woodbury_d6", 30, 6, (), (1e-2,), 200),
    ("chol_noise_free", 15, 2, (), (1e-8,), 10),
    ("woodbury_noise_free", 15, 2, (), (1e-8,), 60),
]
GRID = 200


def _objective(X):
    return np.sin(3.0 * X[:, 0]) + np.cos(2.0 * X.sum(axis=1)) + 0.5 * (X ** 2).sum(axis=1)


def _gradient(X, j):
    s = X.sum(axis=1)
    return (3.0 * np.cos(3.0 * X[:, 0]) if j == 0 else 0.0) - 2.0 * np.sin(2.0 * s) + X[:, j]


class _Cov:
    def __init__(self, h):
        self.h = h

    def get_hyperparameters(self):
        return self.h.copy()


class StubGP:
    def __init__(self, X, Y, noise, derivs, alpha, lengths):
        self.dim = X.shape[1]
        self.num_sampled = X.shape[0]
        self.num_derivatives = len(derivs)
        self.derivatives = list(derivs)
        self.noise_variance = np.array(noise, dtype=float)
        self._points_sampled = X
        self._points_sampled_value = Y
        self._h = np.concatenate([[alpha], lengths])

    def get_covariance_copy(self):
        return _Cov(self._h)


def _load_reference():
    try:
        import past.utils  # noqa: F401
    except ImportError:
        past, past_utils = types.ModuleType("past"), types.ModuleType("past.utils")
        past_utils.old_div = lambda a, b: a / b
        past.utils = past_utils
        sys.modules.update({"past": past, "past.utils": past_utils})
    sys.path.insert(0, REF_PY)
    from moe.optimal_learning.python import random_features as rf
    return rf


def main():
    rf = _load_reference()
    npr = rf.npr
    real_randn, real_uniform, real_slsqp = npr.randn, npr.uniform, rf.spo.fmin_slsqp
    out = {"names": np.array([c[0] for c in CASES])}
    for ci, (name, n, d, derivs, noise, F) in enumerate(CASES):
        rng = np.random.default_rng(1000 + ci)
        X = rng.uniform(0.0, 1.0, size=(n, d))
        Y = np.column_stack([_objective(X)] + [_gradient(X, j) for j in derivs])
        alpha, lengths = 1.3, np.full(d, 0.35) * (1.0 + 0.1 * np.arange(d))
        gp = StubGP(X, Y, noise, derivs, alpha, lengths)
        grid = rng.uniform(0.0, 1.0, size=(GRID, d))
        bounds = [[0.0, 1.0]] * d

        rec = {"randn": [], "uniform": []}
        np.random.seed(2000 + ci)

        def randn(*shape):
            v = real_randn(*shape)
            rec["randn"].append(np.array(v))
            return v

        def uniform(low=0.0, high=1.0, size=None):
            v = real_uniform(low=low, high=high, size=size)
            rec["uniform"].append(np.array(v))
            return v

        slsqp_end = []

        def slsqp(*a, **k):
            x = real_slsqp(*a, **k)
            slsqp_end.append(np.array(x))
            return x

        npr.randn, npr.uniform, rf.spo.fmin_slsqp = randn, uniform, slsqp
        try:
            fun = rf.sample_gp_with_random_features(gp, F)
            omega, b, z = rec["randn"][0], rec["uniform"][0], rec["randn"][1]
            theta = np.array(fun.__closure__[[c for c in fun.__code__.co_freevars].index("theta")].cell_contents)
            W = np.array(fun.__closure__[fun.__code__.co_freevars.index("W")].cell_contents)
            bb = np.array(fun.__closure__[fun.__code__.co_freevars.index("b")].cell_contents).ravel()
            grid_vals = np.asarray(fun(grid, gradient=False)).ravel()
            point = rf.global_optimization_of_GP_approximation(fun, bounds, d, grid)[0]
            # the mean: Omega and b replayed, z forced to zeros
            replay = [omega, np.zeros(F)]
            npr.randn = lambda *shape: replay.pop(0)
            npr.uniform = lambda low=0.0, high=1.0, size=None: b
            fun_m = rf.sample_gp_with_random_features(gp, F)
            m = np.array(fun_m.__closure__[fun.__code__.co_freevars.index("theta")].cell_contents)
            # the mean's sample function on the grid and its local end point (on the M < F branch the draw is not
            # replayed on the device, the mean is)
            grid_vals_m = np.asarray(fun_m(grid, gradient=False)).ravel()
            point_m = rf.global_optimization_of_GP_approximation(fun_m, bounds, d, grid)[0]
            # the whole routine once, from the reference's entry point (its own fresh draws)
            npr.randn, npr.uniform = real_randn, real_uniform
            np.random.seed(3000 + ci)
            pts = rf.sample_from_global_optima(gp, F, bounds, grid, 2)
        finally:
            npr.randn, npr.uniform, rf.spo.fmin_slsqp = real_randn, real_uniform, real_slsqp
        assert np.array_equal(bb, b) and np.allclose(W, omega / lengths, rtol=0, atol=0)
        p = f"{name}/"
        out.update({p + "X": X, p + "Y": Y, p + "noise": np.array(noise), p + "derivs": np.array(derivs, dtype=np.int32),
                    p + "alpha": np.array(alpha), p + "lengths": lengths, p + "F": np.array(F), p + "grid": grid,
                    p + "bounds": np.array(bounds), p + "omega": omega, p + "b": b, p + "z": z, p + "W": W,
                    p + "theta": theta, p + "m": m, p + "grid_vals": grid_vals,
                    p + "grid_argmin": np.array(int(np.argmin(grid_vals))), p + "slsqp_end": slsqp_end[0],
                    p + "point": point, p + "entry_points": pts, p + "grid_vals_m": grid_vals_m,
                    p + "grid_argmin_m": np.array(int(np.argmin(grid_vals_m))), p + "slsqp_end_m": slsqp_end[1],
                    p + "point_m": point_m})
        M = n * (1 + len(derivs))
        print(f"{name}: M = {M}, F = {F}, {'Woodbury' if M < F else 'Cholesky'}, argmin {np.argmin(grid_vals)}, "
              f"point {point}")
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()

"""Regenerates tests/golden/reference_lcb.npz: the reference's LCB batch selection.

The answers come from the reference's own, unmodified ``lower_confidence_bound_optimization``
(cpp_wrappers/lower_confidence_bound.py) called on the reference's own ``cpp_wrappers.gaussian_process.GaussianProcess``.
Two stubs stand in for what that code imports and this environment lacks:

* ``future.utils.with_metaclass`` and ``past.utils.old_div`` (the Python 2/3 compatibility packages), if not installed;
* ``moe.build.GPP``, the reference's compiled module.  Its ``GaussianProcess`` fits through the compiled reference in
  oracle/_ref, answers ``compute_mean_of_points`` (value mean, GetMeanWrapper) and ``compute_cholesky_variance_of_points``
  (the one-point set with the GP's derivative rows, GetCholVarWrapper) from it, and does ``add_sampled_points`` as
  AddPointsToGP does: append and refit from scratch.  A failed factorisation raises ``SingularMatrixException`` with the
  reference's leading-minor index.  Every mean and Cholesky-variance answer is recorded, so the file holds the screen
  and every round's sigma over the satisfied set as the reference computed them.

Stored per case: the inputs, the selected points (and the lowest candidate index with those coordinates), mu, sigma,
each round's sigma, each decision's relative margin, the num_sampled the reference leaves in the caller's GP, or the
exception's info and the failing candidate.  The reference checkout is CMOE_REFERENCE_CPP's parent's parent's parent,
or `reference` beside this repository; oracle/_ref/libmoe_ref.so must have been built by __graft_entry__.build().
Run from the repository root:  python tests/golden/make_lcb_golden.py
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import oracle as orc  # noqa: E402
from synth import make_problem  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_lcb.npz")
REF_CPP = os.environ.get("CMOE_REFERENCE_CPP") or os.path.join(os.path.dirname(ROOT), "reference", "moe",
                                                                "optimal_learning", "cpp")
REF_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(REF_CPP))))

STATE = {"kernel": 1, "means": [], "sigmas": [], "last_point": None}


class SingularMatrixException(RuntimeError):
    def __init__(self, info):
        super().__init__(f"singular, leading minor {info}")
        self.info = info


def _install_stubs(backend):
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
        past, past_utils = types.ModuleType("past"), types.ModuleType("past.utils")
        past_utils.old_div = lambda a, b: a / b
        past.utils = past_utils
        sys.modules.update({"past": past, "past.utils": past_utils})

    class GaussianProcess:
        def __init__(self, hyperparameters, points_sampled, points_sampled_value, noise_variance, derivatives,
                     num_derivatives, dim, num_sampled):
            self.alpha = float(hyperparameters[0])
            self.lengths = np.array(hyperparameters[1], dtype=np.float64)
            self.derivs = np.array(derivatives, dtype=np.int32).reshape(-1)
            self.noise = np.array(noise_variance, dtype=np.float64)
            self.dim = dim
            self.X = np.array(points_sampled, dtype=np.float64).reshape(num_sampled, dim)
            self.y = np.array(points_sampled_value, dtype=np.float64).reshape(-1)
            self._fit()

        def _fit(self):
            gp, lm = backend.gp(STATE["kernel"], self.alpha, self.lengths, self.X, self.y, self.noise, self.derivs)
            if gp is None:
                raise SingularMatrixException(lm)
            self.gp = gp

        @property
        def num_sampled(self):
            return self.X.shape[0]

        def compute_mean_of_points(self, pts, n):
            P = np.array(pts, dtype=np.float64).reshape(n, self.dim)
            # in slices: the checker's binding sizes every output buffer for the whole set
            mu = np.concatenate([self.gp.posterior(P[i:i + 32], None, want=("mean",))["mean"] for i in range(0, n, 32)])
            STATE["means"].append(mu)
            return list(mu)

        def compute_cholesky_variance_of_points(self, pts, n):
            P = np.array(pts, dtype=np.float64).reshape(n, self.dim)
            STATE["last_point"] = P[0].copy()
            r = self.gp.posterior(P, self.derivs, want=("chol_var",))
            if r["rc"] != 0:
                raise SingularMatrixException(r["rc"])
            Q = n * (1 + len(self.derivs))
            L = r["chol_var"].reshape(Q, Q).T  # column-major -> [row, col]
            STATE["sigmas"].append(L[0, 0])
            return list(L.ravel())

        def add_sampled_points(self, pts, vals, num):
            self.X = np.vstack([self.X, np.array(pts, dtype=np.float64).reshape(num, self.dim)])
            self.y = np.concatenate([self.y, np.array(vals, dtype=np.float64).reshape(-1)])
            self._fit()

    gpp = types.ModuleType("moe.build.GPP")
    gpp.GaussianProcess = GaussianProcess
    gpp.SingularMatrixException = SingularMatrixException
    build = types.ModuleType("moe.build")
    build.GPP = gpp
    sys.path.insert(0, REF_ROOT)
    import moe
    moe.build = build
    sys.modules.update({"moe.build": build, "moe.build.GPP": gpp})


def margin(values, best, coords, winner):
    others = np.array([v for v, c in zip(values, coords) if not np.array_equal(c, coords[winner])])
    if others.size == 0:
        return np.inf
    return float(np.min(np.abs(others - best)) / max(abs(best), 1e-300))


# name, kernel (0 SE, 1 Matern-5/2), (N, d, derivs), C, q, seed, noise, alpha, candidates ("uniform", "dup": every
# candidate twice, "train": uniform plus training point 3).  The two g = 2 cases have satisfied sets smaller than q, so
# points repeat; the zero-noise GP fails at a training point in the screen and on the first selection in round 1.
CASES = [
    ("se_20_2_c7_q2", 0, (20, 2, ()), 7, 2, 0, 1e-2, 1.0, "uniform"),
    ("m52_20_2_c500_q5", 1, (20, 2, ()), 500, 5, 1, 1e-2, 1.0, "uniform"),
    ("se_60_3_c500_q12", 0, (60, 3, ()), 500, 12, 2, 1e-2, 1.0, "uniform"),
    ("m52_60_3_c1_q2", 1, (60, 3, ()), 1, 2, 3, 1e-2, 1.0, "uniform"),
    ("m52_200_6_c3000_q5", 1, (200, 6, ()), 3000, 5, 4, 1e-2, 1.0, "uniform"),
    ("se_200_6_c3000_q1", 0, (200, 6, ()), 3000, 1, 5, 1e-2, 1.0, "uniform"),
    ("se_30_3_g2_c500_q5", 0, (30, 3, (0, 2)), 500, 5, 6, 1e-2, 1.0, "uniform"),
    ("m52_30_3_g2_c7_q12", 1, (30, 3, (0, 2)), 7, 12, 7, 1e-2, 1.0, "uniform"),
    ("se_20_2_dup_q8", 0, (20, 2, ()), 80, 8, 8, 1e-2, 1.0, "dup"),
    ("se_zero_noise_screen", 0, (10, 2, ()), 7, 1, 4, 0.0, 1e-3, "train"),
    ("se_zero_noise_round", 0, (10, 2, ()), 8, 3, 4, 0.0, 1e-3, "uniform"),
]


def candidates(kind, C, d, seed, X):
    rng = np.random.default_rng(50 + seed)
    if kind == "dup":
        base = rng.uniform(size=(C // 2, d))
        return np.vstack([base, base])
    if kind == "train":
        return np.vstack([rng.uniform(size=(C - 1, d)), X[3:4]])
    return rng.uniform(size=(C, d))


def main():
    backend = orc.load_reference()
    _install_stubs(backend)
    from moe.optimal_learning.python.cpp_wrappers.covariance import SquareExponential
    from moe.optimal_learning.python.cpp_wrappers.gaussian_process import GaussianProcess
    from moe.optimal_learning.python.cpp_wrappers.lower_confidence_bound import lower_confidence_bound_optimization
    from moe.optimal_learning.python.data_containers import HistoricalData

    out = {"names": np.array([c[0] for c in CASES])}
    for name, kernel, (N, d, derivs), C, q, seed, noise, alpha, kind in CASES:
        pr = make_problem(N, d, derivs, seed=seed, noise=noise, alpha=alpha)
        cand = candidates(kind, C, d, seed, pr["X"])
        g = len(derivs)
        STATE.update(kernel=kernel, means=[], sigmas=[], last_point=None)
        hist = HistoricalData(d, g)
        hist.append_historical_data(pr["X"], pr["y"].reshape(N, 1 + g), np.full(N, noise))
        cov = SquareExponential(np.concatenate([[alpha], pr["lengths"]]))  # only carries the hyper-parameters
        gp = GaussianProcess(cov, pr["noise"], hist, list(derivs))
        rec = {"kernel": kernel, "alpha": alpha, "lengths": pr["lengths"], "X": pr["X"], "y": pr["y"],
               "noise": pr["noise"], "derivs": np.array(derivs, dtype=np.int32), "cand": cand, "q": q}
        try:
            points, zero = lower_confidence_bound_optimization(gp, cand, q)
            assert zero == 0.0
            mu, sig = STATE["means"][0], np.array(STATE["sigmas"])
            sd = sig[:C]
            target, ucb = mu - sd, mu + sd
            first, upper = int(np.argmin(target)), np.min(ucb)
            sat = np.nonzero(target <= upper)[0]
            rounds = sig[C:].reshape(q - 1, len(sat)) if q > 1 else np.zeros((0, len(sat)))
            margins = [margin(target, target[first], cand, first),
                       float(np.min(np.abs(target - upper)) / max(abs(upper), 1e-300))]
            for s in rounds:
                j = int(np.argmax(s))
                margins.append(margin(s, s[j], cand[sat], j))
            index = np.array([int(np.nonzero(np.all(cand == p, axis=1))[0][0]) for p in points])
            rec.update(points=points, index=index, mean=mu, sd=sd, sat=sat, rounds=rounds, margins=np.array(margins),
                       num_sampled_after=gp.num_sampled, info=0, fail_cand=-1)
            print(f"{name}: index {index.tolist()}, C' = {len(sat)}, num_sampled {N} -> {gp.num_sampled}, "
                  f"min margin {min(margins):.2e}")
        except SingularMatrixException as e:
            fail = int(np.nonzero(np.all(cand == STATE["last_point"], axis=1))[0][0])
            rec.update(info=e.info, fail_cand=fail, num_sampled_after=gp.num_sampled)
            print(f"{name}: SingularMatrixException info {e.info} at candidate {fail}, num_sampled {gp.num_sampled}")
        for k, v in rec.items():
            out[f"{name}/{k}"] = np.asarray(v)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()

"""ctypes binding of the C ABI declared in include/cmoe_b200.h.

This is the thinnest possible host layer: numpy arrays in, numpy arrays out, every call goes straight to
libcornell_moe_b200.so (hand-written sm_90a kernels).  If the library is missing or no CUDA device is visible the
calls raise — there is deliberately no fallback.
"""
import collections
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CMOE_B200_LIB", os.path.join(_HERE, "libcornell_moe_b200.so"))

OK, ERR_SINGULAR, ERR_BOUNDS, ERR_INVALID_VALUE, ERR_RUNTIME, ERR_NO_DEVICE = range(6)
SQUARE_EXPONENTIAL, MATERN_NU_2P5 = 0, 1

_dp = ctypes.POINTER(ctypes.c_double)
_ip = ctypes.POINTER(ctypes.c_int)


class CmoeError(RuntimeError):
    """Base error (reference: OptimalLearningException)."""

    def __init__(self, code, msg, info=0):
        super().__init__(msg)
        self.code = code
        self.info = info


class SingularMatrixError(CmoeError):
    """reference: SingularMatrixException; ``info`` = leading minor index."""


class BoundsError(CmoeError):
    """reference: BoundsException."""


class InvalidValueError(CmoeError):
    """reference: InvalidValueException."""


class NoDeviceError(CmoeError):
    """No CUDA device: the product has no CPU path."""


_ERRS = {ERR_SINGULAR: SingularMatrixError, ERR_BOUNDS: BoundsError, ERR_INVALID_VALUE: InvalidValueError,
         ERR_RUNTIME: CmoeError, ERR_NO_DEVICE: NoDeviceError}


class GDParams(ctypes.Structure):
    """GradientDescentParameters (gpp_optimizer_parameters.hpp:81)."""
    _fields_ = [("num_multistarts", ctypes.c_int), ("max_num_steps", ctypes.c_int), ("max_num_restarts", ctypes.c_int),
                ("num_steps_averaged", ctypes.c_int), ("gamma", ctypes.c_double), ("pre_mult", ctypes.c_double),
                ("max_relative_change", ctypes.c_double), ("tolerance", ctypes.c_double)]

    @classmethod
    def from_seq(cls, p):
        if isinstance(p, cls):
            return p
        return cls(int(p[0]), int(p[1]), int(p[2]), int(p[3]), float(p[4]), float(p[5]), float(p[6]), float(p[7]))


class KGStats(ctypes.Structure):
    _fields_ = [("mc_samples", ctypes.c_uint64), ("posterior_evals", ctypes.c_uint64),
                ("line_search_steps", ctypes.c_uint64), ("point_evals", ctypes.c_uint64),
                ("line_batches", ctypes.c_uint64)]


class RffTable(ctypes.Structure):
    """cmoe_rff_table: the numbers that replace Philox in cmoe_gp_sample_rff_optima."""
    _fields_ = [("omega", _dp), ("b", _dp), ("z", _dp), ("eps", _dp)]


RFF_SPECTRAL_REFERENCE, RFF_SPECTRAL_KERNEL = 0, 1


class RffOpts(ctypes.Structure):
    """cmoe_rff_opts: the frequencies' distribution (RFF_SPECTRAL_*) and the chi^2_5 table of the Matern draw."""
    _fields_ = [("spectral", ctypes.c_int), ("chi2", _dp)]


_lib = None


def lib():
    """Loads libcornell_moe_b200.so (raises if it has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: build it with `make -C cornell-moe_b200` (or __graft_entry__.build()); "
                "there is no fallback implementation")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.cmoe_last_error.restype = ctypes.c_char_p
        _lib.cmoe_version.restype = ctypes.c_char_p
    return _lib


def _check(rc, info=0):
    if rc != OK:
        msg = lib().cmoe_last_error().decode()
        raise _ERRS.get(rc, CmoeError)(rc, msg, info)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return np.zeros(0, dtype=np.int32) if a is None else np.ascontiguousarray(a, dtype=np.int32)


def _d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _i(a):
    return None if a is None else a.ctypes.data_as(_ip)


def set_option(name, value):
    """cmoe_set_option: 'legacy_linalg' / 'cov_tma' (0 or 1), 'ensemble_members_in_flight' (k >= 0; 0 = no cap)."""
    _check(lib().cmoe_set_option(name.encode(), int(value)))


def device_count():
    return lib().cmoe_device_count()


def version():
    return lib().cmoe_version().decode()


def cholesky(A, device=0):
    """Lower Cholesky of a symmetric [n, n] array through the device path; returns L as [row, col] array."""
    A = np.array(A, dtype=np.float64)
    n = A.shape[0]
    buf = np.ascontiguousarray(A.T)
    info = ctypes.c_int(0)
    rc = lib().cmoe_cholesky(n, _d(buf), int(device), ctypes.byref(info))
    _check(rc, info.value)
    return buf.T.copy()


def potrs(L, B, device=0):
    Lc = np.ascontiguousarray(np.array(L, dtype=np.float64).T)
    B = np.array(B, dtype=np.float64)
    B2 = B.reshape(B.shape[0], -1)
    buf = np.ascontiguousarray(B2.T)
    _check(lib().cmoe_potrs(Lc.shape[0], B2.shape[1], _d(Lc), _d(buf), int(device)))
    return buf.T.copy().reshape(B.shape)


def philox_normals(seed, first_draw, num_draws, per_draw, device=0):
    out = np.empty(num_draws * per_draw)
    _check(lib().cmoe_philox_normals(ctypes.c_uint64(seed), ctypes.c_uint64(first_draw), int(num_draws),
                                     int(per_draw), _d(out), int(device)))
    return out.reshape(num_draws, per_draw)


def _rff_args(dim, n, F, P, table, spectral):
    """(table struct or None, opts struct or None, keep-alive list) of the random-feature calls on a GP of dimension
    dim with n = num_sampled (1 + g) rows."""
    tab, opts, keep = None, None, []
    if table is not None:
        M = n
        need = {"omega": P * F * dim, "b": P * F, "z": P * F, "eps": P * M if M < F else None}
        tab = RffTable()
        for name in ("omega", "b", "z", "eps"):
            a = table.get(name)
            if a is not None:
                a = _f64(a).ravel()
                keep.append(a)
            if need[name] is not None and (a is None or a.size != need[name]):
                got = "none" if a is None else a.size
                raise BoundsError(ERR_BOUNDS, f"table[{name!r}] needs {need[name]} values, got {got}")
            setattr(tab, name, _d(a))
    chi2 = None if table is None else table.get("chi2")
    if chi2 is not None:
        chi2 = _f64(chi2).ravel()
        if chi2.size != P * F:
            raise BoundsError(ERR_BOUNDS, f"table['chi2'] needs {P * F} values, got {chi2.size}")
        keep.append(chi2)
    if spectral != RFF_SPECTRAL_REFERENCE or chi2 is not None:
        opts = RffOpts(int(spectral), _d(chi2))
    return tab, opts, keep


class GaussianProcess:
    """Device-resident GP (reference: optimal_learning::GaussianProcess, gpp_math.hpp:275)."""

    def __init__(self, kernel, alpha, lengths, X, y, noise, derivs=None, device=0):
        X = _f64(X)
        self.N, self.dim = X.shape
        self.derivs = _i32(derivs)
        self.g = len(self.derivs)
        self.n = self.N * (1 + self.g)
        y = _f64(y).ravel()
        noise = _f64(noise).ravel()
        lengths = _f64(lengths).ravel()
        assert y.size == self.n and noise.size == 1 + self.g and lengths.size == self.dim
        self.kernel = kernel
        self.alpha = float(alpha)
        self.device = device
        h = ctypes.c_void_p()
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_create(int(kernel), ctypes.c_double(alpha), _d(lengths), _d(X), _d(y), _d(noise),
                                  _i(self.derivs), self.g, self.dim, self.N, int(device), ctypes.byref(h),
                                  ctypes.byref(info))
        self.h = None
        _check(rc, info.value)
        self.h = h

    def __del__(self):
        try:
            if self.h:
                lib().cmoe_gp_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def state(self):
        K = np.empty(self.n * self.n)
        kinvy = np.empty(self.n)
        mean = ctypes.c_double()
        _check(lib().cmoe_gp_get_state(self.h, _d(K), _d(kinvy), ctypes.byref(mean)))
        return K.reshape(self.n, self.n).T.copy(), kinvy, mean.value

    def fit_timings_usec(self):
        t = np.zeros(3)
        lib().cmoe_gp_fit_timings(self.h, _d(t))
        return t

    def add_sampled_points(self, pts, vals):
        pts = _f64(pts).reshape(-1, self.dim)
        vals = _f64(vals).ravel()
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_add_sampled_points(self.h, _d(pts), _d(vals), pts.shape[0], ctypes.byref(info))
        _check(rc, info.value)
        self.N += pts.shape[0]
        self.n = self.N * (1 + self.g)

    def bench_cov_build(self, repeats=10):
        t = ctypes.c_double()
        _check(lib().cmoe_bench_cov_build(self.h, int(repeats), ctypes.byref(t)))
        return t.value

    def bench_cholesky(self, repeats=3):
        t = ctypes.c_double()
        _check(lib().cmoe_bench_cholesky(self.h, int(repeats), ctypes.byref(t)))
        return t.value

    def posterior(self, sets, derivs_s=None, want=("mean", "var")):
        """sets: [num_sets, num_pts, dim].  Returns dict of arrays with a leading num_sets axis (reference layouts)."""
        sets = _f64(sets)
        if sets.ndim == 2:
            sets = sets[None]
        ns, num, _ = sets.shape
        ds = _i32(derivs_s)
        Q = num * (1 + len(ds))
        shapes = {"mean": (ns, Q), "grad_mean": (ns, Q * self.dim), "var": (ns, Q * Q), "chol_var": (ns, Q * Q),
                  "grad_var": (ns, num * Q * Q * self.dim), "grad_chol": (ns, num * Q * Q * self.dim)}
        bufs = {k: (np.empty(shapes[k]) if k in want else None) for k in shapes}
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_posterior(self.h, _d(sets), ns, num, _i(ds), len(ds), _d(bufs["mean"]),
                                     _d(bufs["grad_mean"]), _d(bufs["var"]), _d(bufs["chol_var"]),
                                     _d(bufs["grad_var"]), _d(bufs["grad_chol"]), ctypes.byref(info))
        _check(rc, info.value)
        return {k: v for k, v in bufs.items() if v is not None}

    def ei(self, candidates, Xp, num_mc, best_so_far, seed=0, table=None, grad=False):
        cand = _f64(candidates)
        if cand.ndim == 2:
            cand = cand[None]
        nc, q, _ = cand.shape
        Xp = _f64(Xp).reshape(-1, self.dim) if Xp is not None and len(Xp) else np.zeros((0, self.dim))
        table = _f64(table).ravel() if table is not None else None
        if table is not None:
            assert table.size >= num_mc * (q + Xp.shape[0])
        ei = np.empty(nc)
        g = np.empty((nc, q, self.dim)) if grad else None
        info = ctypes.c_int(0)
        rc = lib().cmoe_ei_eval(self.h, _d(cand), nc, q, _d(Xp), Xp.shape[0], int(num_mc),
                                ctypes.c_double(best_so_far), ctypes.c_uint64(seed), _d(table), _d(ei), _d(g),
                                ctypes.byref(info))
        _check(rc, info.value)
        return (ei, g) if grad else ei

    def ei_large(self, candidates, Xp, num_mc, best_so_far, seed=0, table=None, grad=False):
        """cmoe_ei_eval_large: ``ei`` for union sets of up to 8192 rows (q + p), same draws."""
        cand = _f64(candidates)
        if cand.ndim == 2:
            cand = cand[None]
        nc, q, _ = cand.shape
        Xp = _f64(Xp).reshape(-1, self.dim) if Xp is not None and len(Xp) else np.zeros((0, self.dim))
        table = _f64(table).ravel() if table is not None else None
        if table is not None and table.size < num_mc * (q + Xp.shape[0]):
            raise BoundsError(ERR_BOUNDS, f"normals table needs num_mc*(q+p) = {num_mc * (q + Xp.shape[0])} values")
        ei = np.empty(nc)
        g = np.empty((nc, q, self.dim)) if grad else None
        info = ctypes.c_int(0)
        rc = lib().cmoe_ei_eval_large(self.h, _d(cand), nc, q, _d(Xp), Xp.shape[0], int(num_mc),
                                      ctypes.c_double(best_so_far), ctypes.c_uint64(seed), _d(table), _d(ei), _d(g),
                                      ctypes.byref(info))
        _check(rc, info.value)
        return (ei, g) if grad else ei

    def posterior_large(self, sets, derivs_s=None, want=("mean", "var")):
        """cmoe_gp_posterior_large: mean [num_sets, Q], var and chol_var [num_sets, Q*Q] (column-major, as
        ``posterior``) for Q = num_pts (1 + len(derivs_s)) up to 8192."""
        sets = _f64(sets)
        if sets.ndim == 2:
            sets = sets[None]
        ns, num, _ = sets.shape
        ds = _i32(derivs_s)
        Q = num * (1 + len(ds))
        shapes = {"mean": (ns, Q), "var": (ns, Q * Q), "chol_var": (ns, Q * Q)}
        bufs = {k: (np.empty(shapes[k]) if k in want else None) for k in shapes}
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_posterior_large(self.h, _d(sets), ns, num, _i(ds), len(ds), _d(bufs["mean"]),
                                           _d(bufs["var"]), _d(bufs["chol_var"]), ctypes.byref(info))
        _check(rc, info.value)
        return {k: v for k, v in bufs.items() if v is not None}

    def kg(self, candidates, Xp, num_mc, best_so_far, inner, inner_bounds, discrete_pts, num_fidelity=0, seed=0,
           table=None, grad=False, stats=False):
        cand = _f64(candidates)
        if cand.ndim == 2:
            cand = cand[None]
        nc, q, _ = cand.shape
        Xp = _f64(Xp).reshape(-1, self.dim) if Xp is not None and len(Xp) else np.zeros((0, self.dim))
        table = _f64(table).ravel() if table is not None else None
        inner = GDParams.from_seq(inner)
        inner_bounds = _f64(inner_bounds).ravel()
        disc = _f64(discrete_pts).reshape(-1, self.dim - num_fidelity)
        kg = np.empty(nc)
        g = np.empty((nc, q, self.dim)) if grad else None
        st = KGStats()
        info = ctypes.c_int(0)
        rc = lib().cmoe_kg_eval(self.h, int(num_fidelity), ctypes.byref(inner), _d(inner_bounds), _d(disc),
                                disc.shape[0], _d(cand), nc, q, _d(Xp), Xp.shape[0], int(num_mc),
                                ctypes.c_double(best_so_far), ctypes.c_uint64(seed), _d(table), _d(kg), _d(g),
                                ctypes.byref(st), ctypes.byref(info))
        _check(rc, info.value)
        return self._kg_result(kg, g, st, grad, stats)

    def kg_large(self, candidates, Xp, num_mc, best_so_far, inner, inner_bounds, discrete_pts, num_fidelity=0, seed=0,
                 table=None, grad=False, stats=False):
        """cmoe_kg_eval_large: ``kg`` for unions of up to 1024 rows ((q + p)(1 + g)), same arguments and draws."""
        cand = _f64(candidates)
        if cand.ndim == 2:
            cand = cand[None]
        nc, q, _ = cand.shape
        Xp = _f64(Xp).reshape(-1, self.dim) if Xp is not None and len(Xp) else np.zeros((0, self.dim))
        Q = (q + Xp.shape[0]) * (1 + self.g)
        table = _f64(table).ravel() if table is not None else None
        if table is not None and table.size < ((num_mc + 1) // 2) * Q:
            raise BoundsError(ERR_BOUNDS, f"normals table needs ((num_mc+1)/2)*Q = {((num_mc + 1) // 2) * Q} values")
        inner = GDParams.from_seq(inner)
        inner_bounds = _f64(inner_bounds).ravel()
        disc = _f64(discrete_pts).reshape(-1, self.dim - num_fidelity)
        kg = np.empty(nc)
        g = np.empty((nc, q, self.dim)) if grad else None
        st = KGStats()
        info = ctypes.c_int(0)
        rc = lib().cmoe_kg_eval_large(self.h, int(num_fidelity), ctypes.byref(inner), _d(inner_bounds), _d(disc),
                                      disc.shape[0], _d(cand), nc, q, _d(Xp), Xp.shape[0], int(num_mc),
                                      ctypes.c_double(best_so_far), ctypes.c_uint64(seed), _d(table), _d(kg), _d(g),
                                      ctypes.byref(st), ctypes.byref(info))
        _check(rc, info.value)
        return self._kg_result(kg, g, st, grad, stats)

    @staticmethod
    def _kg_result(kg, g, st, grad, stats):
        res = [kg]
        if grad:
            res.append(g)
        if stats:
            res.append({"mc_samples": st.mc_samples, "posterior_evals": st.posterior_evals,
                        "line_search_steps": st.line_search_steps, "point_evals": st.point_evals,
                        "line_batches": st.line_batches})
        return res[0] if len(res) == 1 else tuple(res)


    def sample_joint(self, sets, derivs_s=None, seed=0, first_draw=0, table=None, jitter=0.0,
                     want=("samples", "argmin")):
        """cmoe_gp_sample_joint: one joint posterior draw per point set.  sets: [num_sets, num_pts, dim].  Set b uses
        Philox draw first_draw + b, or row b of ``table`` [num_sets, Q].  Returns a dict with any of samples
        [num_sets, Q], argmin [num_sets], mean [num_sets, Q], chol [num_sets, Q, Q] (lower, as a [row, col] array)."""
        sets = _f64(sets)
        if sets.ndim == 2:
            sets = sets[None]
        ns, num, _ = sets.shape
        ds = _i32(derivs_s)
        Q = num * (1 + len(ds))
        table = _f64(table).ravel() if table is not None else None
        if table is not None and table.size != ns * Q:
            raise BoundsError(ERR_BOUNDS, f"normals table needs num_sets*Q = {ns * Q} values, got {table.size}")
        bufs = {"samples": np.empty((ns, Q)) if "samples" in want else None,
                "argmin": np.empty(ns, dtype=np.int32) if "argmin" in want else None,
                "mean": np.empty((ns, Q)) if "mean" in want else None,
                "chol": np.empty((ns, Q, Q)) if "chol" in want else None}
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_sample_joint(self.h, _d(sets), ns, num, _i(ds), len(ds), ctypes.c_uint64(seed),
                                        ctypes.c_uint64(first_draw), _d(table), ctypes.c_double(jitter),
                                        _d(bufs["samples"]), _i(bufs["argmin"]), _d(bufs["mean"]), _d(bufs["chol"]),
                                        ctypes.byref(info))
        _check(rc, info.value)
        if bufs["chol"] is not None:
            bufs["chol"] = np.ascontiguousarray(bufs["chol"].transpose(0, 2, 1))  # column-major -> [row, col]
        return {k: v for k, v in bufs.items() if v is not None}

    def sample_global_optima(self, num_optima, inner_number, domain_bounds, seed=0, first_draw=0, jitter=0.0):
        """cmoe_gp_sample_global_optima: [num_optima, dim] minimisers of joint draws over Latin hypercubes."""
        bounds = _f64(domain_bounds).ravel()
        if bounds.size != 2 * self.dim:
            raise BoundsError(ERR_BOUNDS, f"domain_bounds needs 2*dim = {2 * self.dim} values, got {bounds.size}")
        out = np.empty((int(num_optima), self.dim))
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_sample_global_optima(self.h, int(num_optima), int(inner_number), _d(bounds),
                                                ctypes.c_uint64(seed), ctypes.c_uint64(first_draw),
                                                ctypes.c_double(jitter), _d(out), ctypes.byref(info))
        _check(rc, info.value)
        return out

    def sample_rff_optima(self, num_features, num_points, domain_bounds, grid, seed=0, first_draw=0, table=None,
                          return_functions=False, spectral=RFF_SPECTRAL_REFERENCE):
        """cmoe_gp_sample_rff_optima_ex: minimisers of num_points random-Fourier-feature draws of the GP, each found on
        ``grid`` [G, dim] and refined inside ``domain_bounds`` ([dim, 2] or flat).  Sample s uses Philox draw
        first_draw + s, or row s of ``table`` (a dict with omega [P, F, dim], b [P, F], z [P, F] and, when
        num_sampled (1 + g) < F, eps [P, num_sampled (1 + g)]; with the Matern draw also chi2 [P, F]).  ``spectral``:
        RFF_SPECTRAL_REFERENCE (SquareExponential frequencies whatever the kernel, as the reference) or
        RFF_SPECTRAL_KERNEL (the GP's own kernel).  Returns (points [P, dim], values [P]); with return_functions, also
        a dict of each sample function f(x) = sqrt(2 alpha / F) theta . cos(omega x + b): omega [P, F, dim] (the
        frequencies), b [P, F], theta [P, F]."""
        F, P = int(num_features), int(num_points)
        bounds = _f64(domain_bounds).ravel()
        if bounds.size != 2 * self.dim:
            raise BoundsError(ERR_BOUNDS, f"domain_bounds needs 2*dim = {2 * self.dim} values, got {bounds.size}")
        grid = _f64(grid).reshape(-1, self.dim)
        tab, opts, keep = _rff_args(self.dim, self.n, F, P, table, spectral)
        pts = np.empty((max(P, 0), self.dim))
        vals = np.empty(max(P, 0))
        fun = ({"omega": np.empty((P, F, self.dim)), "b": np.empty((P, F)), "theta": np.empty((P, F))}
               if return_functions and P >= 1 and F >= 1 else None)
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_sample_rff_optima_ex(self.h, F, P, _d(bounds), _d(grid), grid.shape[0],
                                                ctypes.c_uint64(seed), ctypes.c_uint64(first_draw),
                                                None if tab is None else ctypes.byref(tab),
                                                None if opts is None else ctypes.byref(opts), _d(pts), _d(vals),
                                                _d(fun and fun["omega"]), _d(fun and fun["b"]),
                                                _d(fun and fun["theta"]), ctypes.byref(info))
        del keep
        _check(rc, info.value)
        return (pts, vals, fun) if return_functions else (pts, vals)

    def sample_rff_functions(self, num_features, num_points, seed=0, first_draw=0, table=None,
                             spectral=RFF_SPECTRAL_REFERENCE):
        """cmoe_gp_sample_rff_functions (sample_gp_with_random_features): the sample functions of num_points draws,
        without the grid and the optimiser; arguments as sample_rff_optima.  Returns an RffFunctions whose omega, b and
        theta are those sample_rff_optima returns for the same arguments, bit for bit."""
        F, P = int(num_features), int(num_points)
        tab, opts, keep = _rff_args(self.dim, self.n, F, P, table, spectral)
        omega, b, theta = np.empty((max(P, 0), max(F, 0), self.dim)), np.empty((max(P, 0), max(F, 0))), \
            np.empty((max(P, 0), max(F, 0)))
        info = ctypes.c_int(0)
        rc = lib().cmoe_gp_sample_rff_functions(self.h, F, P, ctypes.c_uint64(seed), ctypes.c_uint64(first_draw),
                                                None if tab is None else ctypes.byref(tab),
                                                None if opts is None else ctypes.byref(opts), _d(omega), _d(b),
                                                _d(theta), ctypes.byref(info))
        del keep
        _check(rc, info.value)
        return RffFunctions(omega, b, theta, float(np.sqrt(2.0 * self.alpha / F)), self.device)

    def lower_confidence_bound(self, candidates, num_to_sample):
        """cmoe_lcb_select: the reference's LCB batch selection over ``candidates`` [C, dim].  Returns (indices [q] into
        candidates, mean [C], sd [C]); mean and sd are the round-0 screen.  The GP is not modified."""
        cand = _f64(candidates).reshape(-1, self.dim)
        idx = np.empty(max(int(num_to_sample), 0), dtype=np.int32)
        mean = np.empty(cand.shape[0])
        sd = np.empty(cand.shape[0])
        info = ctypes.c_int(0)
        rc = lib().cmoe_lcb_select(self.h, _d(cand), cand.shape[0], int(num_to_sample), _i(idx), _d(mean), _d(sd),
                                   None, ctypes.byref(info))
        _check(rc, info.value)
        return idx, mean, sd


class RffFunctions:
    """P random-Fourier-feature sample functions f_p(x) = c sum_f theta[p, f] cos(omega[p, f] . x + b[p, f]):
    omega [P, F, dim], b [P, F], theta [P, F], c = sqrt(2 alpha / F).  Calling it evaluates them on the device
    (cmoe_rff_evaluate)."""

    def __init__(self, omega, b, theta, c, device=0):
        self.omega, self.b, self.theta, self.c, self.device = omega, b, theta, float(c), device

    def __len__(self):
        return self.theta.shape[0]

    def __call__(self, x, gradient=False):
        """x: [dim] or [X, dim] (shared by the functions) or [P, X, dim] (per function).  Returns values [P, X]; with
        gradient, (values [P, X], grads [P, X, dim])."""
        return rff_evaluate(self.omega, self.b, self.theta, self.c, x, grads=gradient, device=self.device)


def rff_evaluate(omega, b, theta, c, points, values=True, grads=False, device=0):
    """cmoe_rff_evaluate: values [P, X] and/or grads [P, X, dim] of the sample functions (omega [P, F, dim], b [P, F],
    theta [P, F], c) at points [X, dim] (shared; [dim] is one point) or [P, X, dim] (per function).  Returns values,
    grads or (values, grads)."""
    omega = _f64(omega)
    P, F, dim = omega.shape
    b, theta = _f64(b).reshape(P, F), _f64(theta).reshape(P, F)
    pts = _f64(points)
    per_function = pts.ndim == 3
    pts = pts.reshape((P, -1, dim) if per_function else (-1, dim))
    X = pts.shape[-2]
    v = np.empty((P, X)) if values else None
    g = np.empty((P, X, dim)) if grads else None
    info = ctypes.c_int(0)
    _check(lib().cmoe_rff_evaluate(int(dim), int(F), int(P), _d(omega), _d(b), _d(theta), ctypes.c_double(c), _d(pts),
                                   int(X), int(per_function), _d(v), _d(g), int(device), ctypes.byref(info)),
           info.value)
    if values and grads:
        return v, g
    return v if values else g


def rff_chi2_draws(seed, first_draw, num_draws, num_features, device=0):
    """cmoe_rff_chi2_draws: the chi^2_5 numbers g [num_draws, num_features] of the Matern random-feature draw."""
    out = np.empty((int(num_draws), int(num_features)))
    _check(lib().cmoe_rff_chi2_draws(ctypes.c_uint64(seed), ctypes.c_uint64(first_draw), int(num_draws),
                                     int(num_features), _d(out), int(device)))
    return out


def latin_hypercube(num_sets, num_pts, domain_bounds, seed=0, first_draw=0, device=0):
    """cmoe_latin_hypercube: [num_sets, num_pts, dim] points; set b is a pure function of (seed, first_draw + b).
    domain_bounds: [dim, 2] (min, max) or the flat list."""
    bounds = _f64(domain_bounds).ravel()
    if bounds.size % 2:
        raise BoundsError(ERR_BOUNDS, "domain_bounds needs (min, max) per dimension")
    dim = bounds.size // 2
    out = np.empty((int(num_sets), int(num_pts), max(dim, 0)))
    _check(lib().cmoe_latin_hypercube(ctypes.c_uint64(seed), ctypes.c_uint64(first_draw), int(num_sets), int(num_pts),
                                      int(dim), _d(bounds), _d(out), int(device)))
    return out


def bench_cholesky_batched(mats, repeats=3, device=0):
    """cmoe_bench_cholesky_batched: (usec per batched call, usec per loop of the single-matrix Cholesky) for the
    [num_mats, Q, Q] symmetric positive definite matrices ``mats``."""
    mats = np.ascontiguousarray(np.asarray(mats, dtype=np.float64).transpose(0, 2, 1))
    nm, Q, _ = mats.shape
    tb, tl = ctypes.c_double(), ctypes.c_double()
    info = ctypes.c_int(0)
    rc = lib().cmoe_bench_cholesky_batched(_d(mats), nm, Q, int(repeats), int(device), ctypes.byref(tb),
                                           ctypes.byref(tl), ctypes.byref(info))
    _check(rc, info.value)
    return tb.value, tl.value


def log_marginal_likelihood(kernel, alpha, lengths, X, y, noise, derivs=None, device=0):
    """cmoe_log_marginal_likelihood (gpp_model_selection.cpp:540-612): one device fit + two host reductions."""
    X = _f64(X)
    N, dim = X.shape
    derivs = _i32(derivs)
    val = ctypes.c_double()
    info = ctypes.c_int()
    rc = lib().cmoe_log_marginal_likelihood(int(kernel), ctypes.c_double(alpha), _d(_f64(lengths).ravel()), _d(X),
                                            _d(_f64(y).ravel()), _d(_f64(noise).ravel()), _i(derivs), len(derivs), dim, N,
                                            int(device), ctypes.byref(val), ctypes.byref(info))
    _check(rc, info.value)
    return val.value


def _lml_list(entry, grads, kernel, hypers, X, y, derivs, device):
    """One of the cmoe_*log_marginal_likelihood_list calls: values [num_sets], and with ``grads`` also the gradients
    [num_sets, 2 + dim + g]."""
    X = _f64(X)
    N, dim = X.shape
    derivs = _i32(derivs)
    H = _f64(hypers).reshape(-1, 2 + dim + derivs.size)
    out = (np.empty(H.shape[0]), np.empty(H.shape)) if grads else (np.empty(H.shape[0]),)
    info = ctypes.c_int()
    rc = getattr(lib(), entry)(int(kernel), _d(H), H.shape[0], _d(X), _d(_f64(y).ravel()), _i(derivs), derivs.size,
                               dim, N, int(device), *(_d(o) for o in out), ctypes.byref(info))
    _check(rc, info.value)
    return out if grads else out[0]


def log_marginal_likelihood_list(kernel, hypers, X, y, derivs=None, device=0):
    """cmoe_log_marginal_likelihood_list (EvaluateLogLikelihoodAtPointList, gpp_model_selection.hpp:1274-1308): the
    log marginal likelihood at every row of ``hypers`` [num_sets, 2 + dim + g] = (alpha, lengths..., noise by
    observation type) in one device call.  Returns a [num_sets] array; a set whose Cholesky fails is -inf."""
    return _lml_list("cmoe_log_marginal_likelihood_list", False, kernel, hypers, X, y, derivs, device)


def grad_log_marginal_likelihood_list(kernel, hypers, X, y, derivs=None, device=0):
    """cmoe_grad_log_marginal_likelihood_list: (values [num_sets], grads [num_sets, 2 + dim + g]) at every row of
    ``hypers`` (the layout of log_marginal_likelihood_list) in one device call.  The values equal
    log_marginal_likelihood_list's bit for bit; a set whose Cholesky fails gets -inf and a zero gradient."""
    return _lml_list("cmoe_grad_log_marginal_likelihood_list", True, kernel, hypers, X, y, derivs, device)


def hyperparameter_gradient_descent(kernel, gd, bounds, starts, X, y, derivs=None, device=0):
    """cmoe_hyperparameter_gradient_descent: restarted gradient ascent of the log marginal likelihood from every row of
    ``starts`` [num_starts, 2 + dim + g] on the linear-space box ``bounds`` [2 + dim + g, 2].  Returns
    (best_point, best_value, found, end_points, end_values)."""
    X = _f64(X)
    N, dim = X.shape
    derivs = _i32(derivs)
    nh = 2 + dim + derivs.size
    S = _f64(starts).reshape(-1, nh)
    B = _f64(bounds).reshape(-1)
    if B.size < 2 * nh:
        raise BoundsError(ERR_BOUNDS, f"bounds needs 2 * (2 + dim + g) = {2 * nh} values, got {B.size}")
    gd = GDParams.from_seq(gd)
    best, ends, end_v = np.empty(nh), np.empty(S.shape), np.empty(S.shape[0])
    best_v, found, info = ctypes.c_double(), ctypes.c_int(), ctypes.c_int()
    rc = lib().cmoe_hyperparameter_gradient_descent(int(kernel), ctypes.byref(gd), _d(B), _d(S), S.shape[0], _d(X),
                                                    _d(_f64(y).ravel()), _i(derivs), derivs.size, dim, N, int(device),
                                                    _d(best), ctypes.byref(best_v), ctypes.byref(found), _d(ends),
                                                    _d(end_v), ctypes.byref(info))
    _check(rc, info.value)
    return best, best_v.value, bool(found.value), ends, end_v


def grad_log_marginal_likelihood_list_exact(kernel, hypers, X, y, derivs=None, device=0):
    """cmoe_grad_log_marginal_likelihood_list_exact: grad_log_marginal_likelihood_list with the exact gradient (every
    entry of a Matern-5/2 derivative block contributes).  Equal to it bit for bit with g = 0 and for SE."""
    return _lml_list("cmoe_grad_log_marginal_likelihood_list_exact", True, kernel, hypers, X, y, derivs, device)


class MapOpts(ctypes.Structure):
    """cmoe_map_opts: gtol and max_iterations (0 = 200 nh) of hyperparameter_map."""
    _fields_ = [("gtol", ctypes.c_double), ("max_iterations", ctypes.c_int)]


def hyperparameter_map(kernel, starts, X, y, derivs=None, noisy=True, default_prior=True, gtol=1e-5,
                       max_iterations=None, device=0):
    """cmoe_hyperparameter_map (DESIGN.md K19): GaussianProcessLogLikelihoodMCMC.optimize's BFGS on
    -compute_log_likelihood from every row of ``starts`` [num_starts, 2 + dim + g] (log scale), with the analytic
    gradient.  Returns a dict of positions, values (nll), gradients, iterations, evaluations and status
    (0 converged, 1 max_iterations, 2 line search failed or objective not finite, 3 NaN)."""
    X = _f64(X)
    N, dim = X.shape
    derivs = _i32(derivs)
    nh = 2 + dim + derivs.size
    S = _f64(starts).reshape(-1, nh)
    M = S.shape[0]
    opts = MapOpts(float(gtol), 0 if max_iterations is None else int(max_iterations))
    pos, grads, vals = np.empty(S.shape), np.empty(S.shape), np.empty(M)
    iters, evals, status = (np.empty(M, dtype=np.int32) for _ in range(3))
    info = ctypes.c_int()
    rc = lib().cmoe_hyperparameter_map(int(kernel), int(bool(default_prior)), int(bool(noisy)), _d(S), M,
                                       ctypes.byref(opts), _d(X), _d(_f64(y).ravel()), _i(derivs), derivs.size, dim, N,
                                       int(device), _d(pos), _d(vals), _d(grads), _i(iters), _i(evals), _i(status),
                                       ctypes.byref(info))
    _check(rc, info.value)
    return dict(positions=pos, values=vals, gradients=grads, iterations=iters, evaluations=evals, status=status)


class MCMCTable(ctypes.Structure):
    """cmoe_mcmc_table: host-supplied random numbers of hyperparameter_mcmc, each [num_steps, num_walkers]."""
    _fields_ = [("z_uniform", _dp), ("partner", _ip), ("accept_uniform", _dp)]


def hyperparameter_mcmc(kernel, p0, X, y, num_steps, derivs=None, noisy=True, default_prior=True, seed=0, first_step=0,
                        table=None, device=0):
    """cmoe_hyperparameter_mcmc (DESIGN.md K12): num_steps steps of emcee 2.2.1's stretch-move ensemble sampler on the
    log-probability of GaussianProcessLogLikelihoodMCMC.compute_log_likelihood, from the walkers ``p0`` [num_walkers,
    2 + dim + g] (log scale), in one device call.  ``table`` = (z_uniform, partner, accept_uniform), each [num_steps,
    num_walkers], replaces the Philox draws.  Returns (positions [num_walkers, 2 + dim + g], lnprob [num_walkers])."""
    X = _f64(X)
    N, dim = X.shape
    derivs = _i32(derivs)
    nh = 2 + dim + derivs.size
    P = _f64(p0).reshape(-1, nh)
    W = P.shape[0]
    pos, lnp = np.empty(P.shape), np.empty(W)
    tab, keep = None, None
    if table is not None:
        keep = (_f64(table[0]).ravel(), _i32(table[1]).ravel(), _f64(table[2]).ravel())
        need = int(num_steps) * W
        if any(t.size < need for t in keep):
            raise BoundsError(ERR_BOUNDS, f"each table needs num_steps * num_walkers = {need} entries")
        tab = ctypes.byref(MCMCTable(_d(keep[0]), _i(keep[1]), _d(keep[2])))
    info = ctypes.c_int()
    rc = lib().cmoe_hyperparameter_mcmc(int(kernel), int(bool(default_prior)), int(bool(noisy)), _d(P), W,
                                        int(num_steps), ctypes.c_uint64(seed), ctypes.c_uint64(first_step), tab, _d(X),
                                        _d(_f64(y).ravel()), _i(derivs), derivs.size, dim, N, int(device), _d(pos),
                                        _d(lnp), ctypes.byref(info))
    _check(rc, info.value)
    return pos, lnp


def grad_log_marginal_likelihood(kernel, alpha, lengths, X, y, noise, derivs=None, device=0):
    """cmoe_grad_log_marginal_likelihood: d log p / d (alpha, lengths..., noise by observation type)."""
    X = _f64(X)
    N, dim = X.shape
    derivs = _i32(derivs if derivs is not None else [])
    grad = np.zeros(dim + 2 + derivs.size)
    info = ctypes.c_int(0)
    rc = lib().cmoe_grad_log_marginal_likelihood(int(kernel), ctypes.c_double(alpha), _d(_f64(lengths).ravel()), _d(X),
                                                 _d(_f64(y).ravel()), _d(_f64(noise).ravel()), _i(derivs), derivs.size,
                                                 dim, N, int(device), _d(grad), ctypes.byref(info))
    _check(rc, info.value)
    return grad


def fp64_peaks(device=0):
    """Measured FP64 peaks (TFLOP/s): (DFMA vector pipe, DMMA tensor pipe)."""
    t = np.zeros(2)
    _check(lib().cmoe_bench_fp64_peaks(int(device), _d(t)))
    return float(t[0]), float(t[1])


def fp64_mixed(device=0):
    """cmoe_bench_fp64_mixed: total TFLOP/s with DFMA and DMMA interleaved in every warp."""
    out = np.zeros(1)
    _check(lib().cmoe_bench_fp64_mixed(int(device), _d(out)))
    return float(out[0])


class KGPlan:
    """Device-resident q-KG evaluation plan (cmoe_kg_plan_*): create -> upload -> run -> sync -> download."""

    def __init__(self, gp, num_mc, best_so_far, inner, inner_bounds, discrete_pts, max_candidates, q, Xp=None,
                 num_fidelity=0, seed=0, want_grad=True, table=None):
        self.gp = gp
        self.q = q
        self.dim = gp.dim
        self.want_grad = want_grad
        Xp = _f64(Xp).reshape(-1, gp.dim) if Xp is not None and len(Xp) else np.zeros((0, gp.dim))
        inner = GDParams.from_seq(inner)
        inner_bounds = _f64(inner_bounds).ravel()
        disc = _f64(discrete_pts).reshape(-1, gp.dim - num_fidelity)
        h = ctypes.c_void_p()
        rc = lib().cmoe_kg_plan_create(gp.h, int(num_fidelity), ctypes.byref(inner), _d(inner_bounds), _d(disc),
                                       disc.shape[0], int(max_candidates), int(q), _d(Xp), Xp.shape[0], int(num_mc),
                                       ctypes.c_double(best_so_far), ctypes.c_uint64(seed), int(bool(want_grad)),
                                       ctypes.byref(h))
        self.h = None
        _check(rc)
        self.h = h
        self.nc = 0
        if table is not None:
            table = _f64(table).ravel()
            _check(lib().cmoe_kg_plan_set_table(self.h, _d(table), table.size))

    def __del__(self):
        try:
            if self.h:
                lib().cmoe_kg_plan_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set_stale_union(self, points):
        """Reference-driver compatibility (cmoe_kg_plan_set_stale_union): the discretisation set keeps these q points."""
        pts = _f64(points).reshape(self.q, self.dim) if points is not None else None
        _check(lib().cmoe_kg_plan_set_stale_union(self.h, _d(pts)))

    def upload(self, candidates):
        cand = _f64(candidates).reshape(-1, self.q, self.dim)
        self.nc = cand.shape[0]
        _check(lib().cmoe_kg_plan_upload(self.h, _d(cand), self.nc))

    def run(self):
        _check(lib().cmoe_kg_plan_run(self.h))

    def sync(self):
        info = ctypes.c_int(0)
        _check(lib().cmoe_kg_plan_sync(self.h, ctypes.byref(info)), info.value)

    def download(self):
        kg = np.empty(self.nc)
        g = np.empty((self.nc, self.q, self.dim)) if self.want_grad else None
        st = KGStats()
        _check(lib().cmoe_kg_plan_download(self.h, _d(kg), _d(g), ctypes.byref(st)))
        return kg, g, {"mc_samples": st.mc_samples, "posterior_evals": st.posterior_evals,
                       "line_search_steps": st.line_search_steps, "point_evals": st.point_evals,
                       "line_batches": st.line_batches}

    def timings(self):
        total, mc = ctypes.c_double(), ctypes.c_double()
        launches = ctypes.c_int()
        _check(lib().cmoe_kg_plan_timings(self.h, ctypes.byref(total), ctypes.byref(mc), ctypes.byref(launches)))
        return total.value, mc.value, launches.value


def _gd_args(gp, outer, inner, domain_bounds, inner_bounds, discrete_pts, num_fidelity):
    return (GDParams.from_seq(outer), GDParams.from_seq(inner) if inner is not None else None,
            _f64(domain_bounds).ravel(), _f64(inner_bounds).ravel() if inner_bounds is not None else None,
            _f64(discrete_pts).reshape(-1, gp.dim - num_fidelity) if discrete_pts is not None else None)


class MultistartOpts(ctypes.Structure):
    _fields_ = [("normals_table", ctypes.POINTER(ctypes.c_double)), ("table_len", ctypes.c_size_t),
                ("devices", ctypes.POINTER(ctypes.c_int)), ("num_devices", ctypes.c_int),
                ("domain_type", ctypes.c_int), ("fresh_discretisation", ctypes.c_int),
                ("stale_union", ctypes.POINTER(ctypes.c_double))]


TENSOR_PRODUCT, SIMPLEX = 0, 1


def limit_update(domain_type, bounds, mrc, x, upd):
    """cmoe_limit_update: one LimitUpdate of the outer optimiser's domain (host arithmetic)."""
    x = _f64(x).ravel()
    upd = _f64(upd).ravel().copy()
    _check(lib().cmoe_limit_update(int(domain_type), _d(_f64(bounds).ravel()), x.size, ctypes.c_double(mrc), _d(x),
                                   _d(upd)))
    return upd


def _multistart_opts(table, devices, domain_type=0, fresh=False, stale=None):
    """(opts struct or None, keep-alive tuple) for cmoe_multistart_{kg,ei}_ex."""
    if table is None and not devices and not domain_type and not fresh and stale is None:
        return None, ()
    t = _f64(table).ravel() if table is not None else None
    dv = _i32(devices) if devices else None
    o = MultistartOpts(_d(t) if t is not None else None, t.size if t is not None else 0,
                       _i(dv) if dv is not None else None, dv.size if dv is not None else 0, int(domain_type),
                       int(bool(fresh)), None)
    st = None
    if stale is not None:
        st = _f64(stale).ravel()
        o.stale_union = _d(st)
    return o, (t, dv, st)


def multistart_kg(gp, starts, Xp, num_mc, best_so_far, outer, inner, domain_bounds, inner_bounds, discrete_pts,
                  num_fidelity=0, seed=0, table=None, devices=None, fresh_discretisation=False, stale_union=None):
    """cmoe_multistart_kg(_ex): returns (best_point [q, dim], best_value, found_flag, start_values).
    table: normals replayed by every evaluation (NormalRNGSimulator semantics); devices: GPUs to shard the starts over."""
    starts = _f64(starts)
    ns, q, dim = starts.shape
    Xp = _f64(Xp).reshape(-1, dim) if Xp is not None and len(Xp) else np.zeros((0, dim))
    outer, inner, db, ib, disc = _gd_args(gp, outer, inner, domain_bounds, inner_bounds, discrete_pts, num_fidelity)
    vals = np.empty(ns)
    best = np.empty((q, dim))
    bv = ctypes.c_double()
    found = ctypes.c_int()
    info = ctypes.c_int()
    opts, keep = _multistart_opts(table, devices, 0, fresh_discretisation, stale_union)
    rc = lib().cmoe_multistart_kg_ex(gp.h, int(num_fidelity), ctypes.byref(outer), ctypes.byref(inner), _d(db), _d(ib),
                                     _d(disc), disc.shape[0], _d(starts), ns, q, _d(Xp), Xp.shape[0], int(num_mc),
                                     ctypes.c_double(best_so_far), ctypes.c_uint64(seed),
                                     ctypes.byref(opts) if opts is not None else None, _d(vals), _d(best),
                                     ctypes.byref(bv), ctypes.byref(found), ctypes.byref(info))
    del keep
    _check(rc, info.value)
    return best, bv.value, bool(found.value), vals


def multistart_ei(gp, starts, Xp, num_mc, best_so_far, outer, domain_bounds, seed=0, table=None, devices=None,
                  domain_type=0):
    starts = _f64(starts)
    ns, q, dim = starts.shape
    Xp = _f64(Xp).reshape(-1, dim) if Xp is not None and len(Xp) else np.zeros((0, dim))
    outer = GDParams.from_seq(outer)
    db = _f64(domain_bounds).ravel()
    vals = np.empty(ns)
    best = np.empty((q, dim))
    bv = ctypes.c_double()
    found = ctypes.c_int()
    info = ctypes.c_int()
    opts, keep = _multistart_opts(table, devices, domain_type)
    rc = lib().cmoe_multistart_ei_ex(gp.h, ctypes.byref(outer), _d(db), _d(starts), ns, q, _d(Xp), Xp.shape[0],
                                     int(num_mc), ctypes.c_double(best_so_far), ctypes.c_uint64(seed),
                                     ctypes.byref(opts) if opts is not None else None, _d(vals), _d(best),
                                     ctypes.byref(bv), ctypes.byref(found), ctypes.byref(info))
    del keep
    _check(rc, info.value)
    return best, bv.value, bool(found.value), vals


def kg_gradient_descent(gp, starts, Xp, num_mc, best_so_far, outer, inner, domain_bounds, inner_bounds, discrete_pts,
                        num_fidelity=0, seed=0, stale_union=None):
    starts = _f64(starts)
    ns, q, dim = starts.shape
    Xp = _f64(Xp).reshape(-1, dim) if Xp is not None and len(Xp) else np.zeros((0, dim))
    outer, inner, db, ib, disc = _gd_args(gp, outer, inner, domain_bounds, inner_bounds, discrete_pts, num_fidelity)
    vals = np.empty(ns)
    pts = np.empty((ns, q, dim))
    info = ctypes.c_int()
    st = _f64(stale_union).ravel() if stale_union is not None else None
    rc = lib().cmoe_kg_gradient_descent_ex(gp.h, int(num_fidelity), ctypes.byref(outer), ctypes.byref(inner), _d(db),
                                           _d(ib), _d(disc), disc.shape[0], _d(starts), ns, q, _d(Xp), Xp.shape[0],
                                           int(num_mc), ctypes.c_double(best_so_far), ctypes.c_uint64(seed), _d(st),
                                           _d(vals), _d(pts), ctypes.byref(info))
    _check(rc, info.value)
    return vals, pts


def ei_gradient_descent(gp, starts, Xp, num_mc, best_so_far, outer, domain_bounds, seed=0):
    starts = _f64(starts)
    ns, q, dim = starts.shape
    Xp = _f64(Xp).reshape(-1, dim) if Xp is not None and len(Xp) else np.zeros((0, dim))
    outer = GDParams.from_seq(outer)
    db = _f64(domain_bounds).ravel()
    vals = np.empty(ns)
    pts = np.empty((ns, q, dim))
    info = ctypes.c_int()
    rc = lib().cmoe_ei_gradient_descent(gp.h, ctypes.byref(outer), _d(db), _d(starts), ns, q, _d(Xp), Xp.shape[0],
                                        int(num_mc), ctypes.c_double(best_so_far), ctypes.c_uint64(seed), _d(vals),
                                        _d(pts), ctypes.byref(info))
    _check(rc, info.value)
    return vals, pts


CONSTANT_LIAR, KRIGING_BELIEVER = 0, 1


class EstimationPolicy(ctypes.Structure):
    """cmoe_estimation_policy: CONSTANT_LIAR (value = the lie) or KRIGING_BELIEVER (value = std_deviation_coef)."""
    _fields_ = [("policy", ctypes.c_int), ("value", ctypes.c_double), ("noise_variance", ctypes.c_double)]


def heuristic_ei(gp, starts, best_so_far, policy, value, noise_variance, outer=None, domain_bounds=None):
    """cmoe_heuristic_ei: q points by Constant Liar or Kriging Believer.  ``starts`` [q, num_starts, dim] (round r uses
    block r); ``outer`` gradient-descent parameters, or None for the random search of the screen alone.  Returns
    (points [q, dim], fantasy_values [q], ei_values [q], found [q]).  The GP is not modified."""
    starts = _f64(starts)
    q, ns, dim = starts.shape
    gd = None if outer is None else GDParams.from_seq(outer)
    db = _f64(domain_bounds).ravel()
    pol = EstimationPolicy(int(policy), float(value), float(noise_variance))
    pts = np.empty((q, dim))
    fv = np.empty(q)
    ev = np.empty(q)
    found = np.empty(q, dtype=np.int32)
    info = ctypes.c_int()
    rc = lib().cmoe_heuristic_ei(gp.h, ctypes.byref(pol), None if gd is None else ctypes.byref(gd), _d(db),
                                 _d(starts), ns, q, ctypes.c_double(best_so_far), _d(pts), _d(fv), _d(ev), _i(found),
                                 ctypes.byref(info))
    _check(rc, info.value)
    return pts, fv, ev, found.astype(bool)


def posterior_mean_optimization(gp, initial_guess, params, domain_bounds, num_fidelity=0):
    """cmoe_posterior_mean_optimization: returns (best_point [dim - num_fidelity], -min mu, found)."""
    ps = gp.dim - num_fidelity
    x0 = _f64(initial_guess).ravel()
    assert x0.size == ps
    params = GDParams.from_seq(params)
    db = _f64(domain_bounds).ravel()
    best = np.zeros(ps)
    val = ctypes.c_double()
    found = ctypes.c_int()
    _check(lib().cmoe_posterior_mean_optimization(gp.h, int(num_fidelity), ctypes.byref(params), _d(db), _d(x0),
                                                  _d(best), ctypes.byref(val), ctypes.byref(found)))
    return best, val.value, bool(found.value)


def ei_analytic(gp, points, best_so_far, grad=False):
    """cmoe_ei_analytic: closed-form 1-EI (and gradient) at points [n, dim]."""
    pts = _f64(points).reshape(-1, gp.dim)
    vals = np.empty(pts.shape[0])
    g = np.empty_like(pts) if grad else None
    info = ctypes.c_int()
    _check(lib().cmoe_ei_analytic(gp.h, _d(pts), pts.shape[0], ctypes.c_double(best_so_far), _d(vals), _d(g),
                                  ctypes.byref(info)), info.value)
    return (vals, g) if grad else vals


class GaussianProcessEnsemble:
    """An array of GP handles over the same data, one per hyper-parameter sample — the reference's GaussianProcessMCMC
    (gpp_knowledge_gradient_mcmc_optimization.cpp:24-48).  hypers[M][1+dim] = (alpha, lengths); noises[M][1+g]."""

    def __init__(self, hypers, noises, X, y, derivs=None, kernel=MATERN_NU_2P5, device=0):
        hypers, noises = _f64(hypers), _f64(noises)
        self.members = [GaussianProcess(kernel, hypers[m, 0], hypers[m, 1:], X, y, noises[m], derivs, device)
                        for m in range(hypers.shape[0])]
        self.dim = self.members[0].dim

    def __len__(self):
        return len(self.members)

    def _handles(self):
        return (ctypes.c_void_p * len(self.members))(*[gp.h for gp in self.members])

    def _cands(self, candidates, Xp):
        cand = _f64(candidates)
        if cand.ndim == 2:
            cand = cand[None]
        Xp = _f64(Xp).reshape(-1, self.dim) if Xp is not None and len(Xp) else np.zeros((0, self.dim))
        return cand, Xp

    def kg(self, candidates, Xp, num_mc, best_so_far, inner, inner_bounds, discrete_pts, num_fidelity=0, seed=0,
           table=None, grad=False):
        """cmoe_kg_eval_mcmc.  discrete_pts [M, num_pts, dim - nf]; best_so_far [M]."""
        cand, Xp = self._cands(candidates, Xp)
        nc, q, _ = cand.shape
        M = len(self.members)
        disc = _f64(discrete_pts).reshape(M, -1, self.dim - num_fidelity)
        best = _f64(best_so_far).ravel()
        assert best.size == M
        table = _f64(table).ravel() if table is not None else None
        inner = GDParams.from_seq(inner)
        ib = _f64(inner_bounds).ravel()
        vals = np.empty(nc)
        g = np.empty((nc, q, self.dim)) if grad else None
        info = ctypes.c_int()
        rc = lib().cmoe_kg_eval_mcmc(self._handles(), M, int(num_fidelity), ctypes.byref(inner), _d(ib), _d(disc),
                                     disc.shape[1], _d(cand), nc, q, _d(Xp), Xp.shape[0], int(num_mc), _d(best),
                                     ctypes.c_uint64(seed), _d(table), _d(vals), _d(g), ctypes.byref(info))
        _check(rc, info.value)
        return (vals, g) if grad else vals

    def ei(self, candidates, Xp, num_mc, best_so_far, seed=0, table=None, grad=False, analytic_single=False):
        """cmoe_ei_eval_mcmc."""
        cand, Xp = self._cands(candidates, Xp)
        nc, q, _ = cand.shape
        M = len(self.members)
        best = _f64(best_so_far).ravel()
        assert best.size == M
        table = _f64(table).ravel() if table is not None else None
        vals = np.empty(nc)
        g = np.empty((nc, q, self.dim)) if grad else None
        info = ctypes.c_int()
        rc = lib().cmoe_ei_eval_mcmc(self._handles(), M, _d(cand), nc, q, _d(Xp), Xp.shape[0], int(num_mc), _d(best),
                                     ctypes.c_uint64(seed), _d(table), int(bool(analytic_single)), _d(vals), _d(g),
                                     ctypes.byref(info))
        _check(rc, info.value)
        return (vals, g) if grad else vals

    def multistart_kg(self, starts, Xp, num_mc, best_so_far, outer, inner, domain_bounds, inner_bounds, discrete_pts,
                      num_fidelity=0, seed=0):
        """cmoe_multistart_kg_mcmc: returns (best_point [q, dim], best_value, found_flag, start_values)."""
        starts = _f64(starts)
        ns, q, dim = starts.shape
        _, Xp = self._cands(starts, Xp)
        M = len(self.members)
        disc = _f64(discrete_pts).reshape(M, -1, self.dim - num_fidelity)
        best_in = _f64(best_so_far).ravel()
        outer, inner = GDParams.from_seq(outer), GDParams.from_seq(inner)
        db, ib = _f64(domain_bounds).ravel(), _f64(inner_bounds).ravel()
        vals, best = np.empty(ns), np.empty((q, dim))
        bv, found, info = ctypes.c_double(), ctypes.c_int(), ctypes.c_int()
        rc = lib().cmoe_multistart_kg_mcmc(self._handles(), M, int(num_fidelity), ctypes.byref(outer),
                                           ctypes.byref(inner), _d(db), _d(ib), _d(disc), disc.shape[1], _d(starts), ns,
                                           q, _d(Xp), Xp.shape[0], int(num_mc), _d(best_in), ctypes.c_uint64(seed),
                                           _d(vals), _d(best), ctypes.byref(bv), ctypes.byref(found),
                                           ctypes.byref(info))
        _check(rc, info.value)
        return best, bv.value, bool(found.value), vals

    def multistart_ei(self, starts, Xp, num_mc, best_so_far, outer, domain_bounds, seed=0):
        """cmoe_multistart_ei_mcmc: returns (best_point [q, dim], best_value, found_flag, start_values)."""
        starts = _f64(starts)
        ns, q, dim = starts.shape
        _, Xp = self._cands(starts, Xp)
        M = len(self.members)
        best_in = _f64(best_so_far).ravel()
        outer = GDParams.from_seq(outer)
        db = _f64(domain_bounds).ravel()
        vals, best = np.empty(ns), np.empty((q, dim))
        bv, found, info = ctypes.c_double(), ctypes.c_int(), ctypes.c_int()
        rc = lib().cmoe_multistart_ei_mcmc(self._handles(), M, ctypes.byref(outer), _d(db), _d(starts), ns, q, _d(Xp),
                                           Xp.shape[0], int(num_mc), _d(best_in), ctypes.c_uint64(seed), _d(vals),
                                           _d(best), ctypes.byref(bv), ctypes.byref(found), ctypes.byref(info))
        _check(rc, info.value)
        return best, bv.value, bool(found.value), vals

    def kg_gradient_descent(self, starts, Xp, num_mc, best_so_far, outer, inner, domain_bounds, inner_bounds,
                            discrete_pts, num_fidelity=0, seed=0):
        """cmoe_kg_gradient_descent_mcmc: returns (values [ns], points [ns, q, dim])."""
        starts = _f64(starts)
        ns, q, dim = starts.shape
        _, Xp = self._cands(starts, Xp)
        M = len(self.members)
        disc = _f64(discrete_pts).reshape(M, -1, self.dim - num_fidelity)
        best_in = _f64(best_so_far).ravel()
        outer, inner = GDParams.from_seq(outer), GDParams.from_seq(inner)
        db, ib = _f64(domain_bounds).ravel(), _f64(inner_bounds).ravel()
        vals, pts = np.empty(ns), np.empty((ns, q, dim))
        info = ctypes.c_int()
        rc = lib().cmoe_kg_gradient_descent_mcmc(self._handles(), M, int(num_fidelity), ctypes.byref(outer),
                                                 ctypes.byref(inner), _d(db), _d(ib), _d(disc), disc.shape[1],
                                                 _d(starts), ns, q, _d(Xp), Xp.shape[0], int(num_mc), _d(best_in),
                                                 ctypes.c_uint64(seed), _d(vals), _d(pts), ctypes.byref(info))
        _check(rc, info.value)
        return vals, pts

    def ei_gradient_descent(self, starts, Xp, num_mc, best_so_far, outer, domain_bounds, seed=0):
        """cmoe_ei_gradient_descent_mcmc: returns (values [ns], points [ns, q, dim])."""
        starts = _f64(starts)
        ns, q, dim = starts.shape
        _, Xp = self._cands(starts, Xp)
        M = len(self.members)
        best_in = _f64(best_so_far).ravel()
        outer = GDParams.from_seq(outer)
        db = _f64(domain_bounds).ravel()
        vals, pts = np.empty(ns), np.empty((ns, q, dim))
        info = ctypes.c_int()
        rc = lib().cmoe_ei_gradient_descent_mcmc(self._handles(), M, ctypes.byref(outer), _d(db), _d(starts), ns, q,
                                                 _d(Xp), Xp.shape[0], int(num_mc), _d(best_in), ctypes.c_uint64(seed),
                                                 _d(vals), _d(pts), ctypes.byref(info))
        _check(rc, info.value)
        return vals, pts

    @classmethod
    def from_members(cls, members):
        """An ensemble over existing GaussianProcess handles (same dim, derivative observations and device; the number
        of sampled points may differ, e.g. after add_sampled_points on some of them)."""
        self = cls.__new__(cls)
        self.members = list(members)
        self.dim = self.members[0].dim
        return self

    def posterior_mean(self, points, num_fidelity=0, grad=False, per_member=False):
        """cmoe_posterior_mean_mcmc: f = -(1/M) sum_m mu_m at points [P, dim - num_fidelity] (PosteriorMeanMCMC's sign;
        fidelity coordinates pinned to 1.0).  Returns values [P], followed by grads [P, dim - num_fidelity] if grad and
        by member values -mu_m [M, P] if per_member."""
        ps = self.dim - num_fidelity
        pts = _f64(points).reshape(-1, ps)
        P, M = pts.shape[0], len(self.members)
        vals = np.empty(P)
        g = np.empty((P, ps)) if grad else None
        mv = np.empty((M, P)) if per_member else None
        info = ctypes.c_int()
        _check(lib().cmoe_posterior_mean_mcmc(self._handles(), M, int(num_fidelity), _d(pts), P, _d(vals), _d(g), _d(mv),
                                              ctypes.byref(info)), info.value)
        out = (vals,) + ((g,) if grad else ()) + ((mv,) if per_member else ())
        return out[0] if len(out) == 1 else out

    def posterior_mean_optimization(self, starts, params, domain_bounds, num_fidelity=0):
        """cmoe_posterior_mean_mcmc_optimization: the Python fixed-step gradient descent with Polyak-Ruppert averaging
        on the ensemble mean from every start [S, dim - num_fidelity].  `params` is a GDParams, an 8-sequence in its
        field order, or any object with its attributes (e.g. the reference's python_version GradientDescentParameters).
        Returns (best_point [dim - nf], best_value, points [S, dim - nf], values [S])."""
        ps = self.dim - num_fidelity
        starts = _f64(starts).reshape(-1, ps)
        ns, M = starts.shape[0], len(self.members)
        params = _gd_params_any(params)
        db = _f64(domain_bounds).ravel()
        pts, vals, best = np.empty((ns, ps)), np.empty(ns), np.empty(ps)
        bv, info = ctypes.c_double(), ctypes.c_int()
        _check(lib().cmoe_posterior_mean_mcmc_optimization(self._handles(), M, int(num_fidelity), ctypes.byref(params),
                                                           _d(db), _d(starts), ns, _d(pts), _d(vals), _d(best),
                                                           ctypes.byref(bv), ctypes.byref(info)), info.value)
        return best, bv.value, pts, vals

    def recommend_point(self, eval_pts, params, domain_bounds, num_fidelity=0):
        """The recommendation step of the reference's examples/main.py:243-260 in two device calls: screen eval_pts,
        descend from the point of least ensemble mean, and keep the screened point if the descended one is strictly
        worse.  Returns the point [dim - num_fidelity]."""
        ps = self.dim - num_fidelity
        pts = _f64(eval_pts).reshape(-1, ps)
        test = -self.posterior_mean(pts, num_fidelity)  # the ensemble's mean posterior mean, as main.py's `test`
        initial = pts[int(np.argmin(test))]
        point, value, _, _ = self.posterior_mean_optimization(initial[None], params, domain_bounds, num_fidelity)
        return initial.copy() if -value > np.min(test) else point

    def posterior_mean_optima(self, points, params, domain_bounds, num_fidelity=0, include_sampled=True,
                              shared_discrete=None):
        """cmoe_posterior_mean_optima_mcmc: per member, screen `points` (and the member's own sampled points if
        include_sampled) by posterior mean, descend from the argmin with the reference's line search, keep the start if
        the descent ended higher, and take the least mean over [shared_discrete ; optimum].  points is [P, ps] (shared by
        the members) or [M, P, ps] (one list per member), ps = dim - num_fidelity; `params` as in
        posterior_mean_optimization.  Returns a PosteriorMeanOptima; its discrete_pts [M, num_shared + 1, ps] and
        best_so_far [M] are what kg / multistart_kg take."""
        ps, M = self.dim - num_fidelity, len(self.members)
        pts = _f64(points)
        per_member = pts.ndim == 3
        pts = pts.reshape((M, -1, ps) if per_member else (-1, ps))
        P = pts.shape[-2]
        shared = _f64(shared_discrete).reshape(-1, ps) if shared_discrete is not None else np.zeros((0, ps))
        ns = shared.shape[0]
        params = _gd_params_any(params)
        db = _f64(domain_bounds).ravel()
        out = PosteriorMeanOptima(np.empty((M, ps)), np.empty(M), np.empty(M, dtype=np.int32),
                                  np.empty(M, dtype=np.int32), np.empty(M), np.empty((M, ns + 1, ps)), np.empty(M))
        _ip = ctypes.POINTER(ctypes.c_int)
        info = ctypes.c_int()
        _check(lib().cmoe_posterior_mean_optima_mcmc(
            self._handles(), M, int(num_fidelity), ctypes.byref(params), _d(db), _d(pts), P, int(per_member),
            int(bool(include_sampled)), _d(shared) if ns else None, ns, _d(out.optima), _d(out.means),
            out.start_index.ctypes.data_as(_ip), out.kept_start.ctypes.data_as(_ip), _d(out.screen_min),
            _d(out.discrete_pts), _d(out.best_so_far), ctypes.byref(info)), info.value)
        return out


PosteriorMeanOptima = collections.namedtuple(
    "PosteriorMeanOptima", "optima means start_index kept_start screen_min discrete_pts best_so_far")


def _gd_params_any(p):
    if isinstance(p, GDParams):
        return p
    if all(hasattr(p, f) for f in ("max_num_steps", "num_steps_averaged", "gamma", "pre_mult", "max_relative_change")):
        return GDParams(int(getattr(p, "num_multistarts", 0)), int(p.max_num_steps), int(getattr(p, "max_num_restarts", 0)),
                        int(p.num_steps_averaged), float(p.gamma), float(p.pre_mult), float(p.max_relative_change),
                        float(getattr(p, "tolerance", 0.0)))
    return GDParams.from_seq(p)

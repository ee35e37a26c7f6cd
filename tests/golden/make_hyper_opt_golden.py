"""Regenerates tests/golden/reference_hyper_opt.npz: the reference side of the GPP-entry tests in
tests/test_gpu_hyper_opt.py.

Everything comes from the reference itself: MultistartGradientDescentHyperparameterOptimization,
LatinHypercubeSearchHyperparameterOptimization and RestartedGradientDescentHyperparameterOptimizationTensor
(gpp_model_selection.hpp), unmodified, called through tests/golden/hyper_opt_ref_driver.cpp, which this script compiles
against the reference headers and links to oracle/_ref/libmoe_ref.so (built by __graft_entry__.build() from a
Cornell-MOE checkout).  For every case it stores, per call of NUM_CALLS consecutive calls on one seeded generator, the
best point, the found flag and the linear-space starts the call drew; for the gradient-descent cases also the end point
of the restarted driver from each start of the first call.  Before writing it checks that the best end value beats the
runner-up by a relative margin of at least 1e-6, so that device rounding cannot flip the choice, and that the
multistart answer is the restarted driver's end point of the best start.  Run from the repository root:

    python tests/golden/make_hyper_opt_golden.py
"""
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import oracle as orc  # noqa: E402
import test_gpu_hyper_opt as t  # noqa: E402

DRIVER = os.path.join(ROOT, "tests", "golden", "hyper_opt_ref_driver.cpp")
REF_CPP = os.environ.get("CMOE_REFERENCE_CPP") or os.path.join(os.path.dirname(ROOT), "reference", "moe",
                                                                "optimal_learning", "cpp")


def load_driver(tmp):
    """Compiles hyper_opt_ref_driver.cpp with the flags oracle/Makefile uses for the reference, linked to
    libmoe_ref.so."""
    so = os.path.join(tmp, "libhyper_opt_ref.so")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.run(["g++", "-std=c++14", "-O2", "-fopenmp", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "oracle", "compat"), "-I" + REF_CPP, DRIVER, "-o", so,
                    "-L" + ref_dir, "-lmoe_ref", "-Wl,-rpath," + ref_dir], check=True)
    return ctypes.CDLL(so)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def reference_answers(lib):
    ref = orc.load_reference()
    out = {}
    for name in sorted(t.REF_CASES):
        prob, log_domain, optimizer, gd, seed = t.ref_case(name)
        X, y = _f(prob["X"]), _f(prob["y"])
        derivs = np.ascontiguousarray(prob["derivs"], dtype=np.int32)
        N, dim = X.shape
        g = derivs.size
        nh = 2 + dim + g
        n = gd[0]
        common = (_dp(X), _dp(y), derivs.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), g, dim, N)
        dom, gdv = _f(log_domain), _f(gd)
        best = np.zeros((t.NUM_CALLS, nh))
        found = np.zeros(t.NUM_CALLS, dtype=np.int32)
        starts = np.zeros((t.NUM_CALLS, n, nh))
        lib.href_multistart(optimizer, ctypes.c_double(prob["alpha"]), _dp(_f(prob["lengths"])), _dp(_f(prob["noise"])),
                            *common, _dp(dom), _dp(gdv), ctypes.c_uint(seed), t.NUM_CALLS, _dp(best),
                            found.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), _dp(starts))

        def lml(h):
            return ref.log_marginal_likelihood(1, h[0], h[1:1 + dim], X, y, h[1 + dim:], derivs)

        if optimizer == 0:
            for c in range(t.NUM_CALLS):
                vals = np.array([lml(h) for h in starts[c]])
                assert np.array_equal(best[c], starts[c][int(np.argmax(vals))])
                top = np.sort(vals)[-2:]
                assert top[1] - top[0] >= 1e-6 * abs(top[1]), (name, c, top)
        else:
            ends = np.zeros((n, nh))
            for s in range(n):
                h = _f(starts[0, s])
                lib.href_restarted(ctypes.c_double(h[0]), _dp(_f(h[1:1 + dim])), _dp(_f(h[1 + dim:])), *common,
                                   _dp(dom), _dp(gdv), _dp(ends[s]))
            end_v = np.array([lml(h) for h in ends])
            top = np.sort(end_v)[-2:]
            assert top[1] - top[0] >= 1e-6 * abs(top[1]), (name, top)
            if found[0]:
                assert np.array_equal(best[0], ends[int(np.argmax(end_v))])
            out[f"{name}_restarted"] = ends
        out[f"{name}_best"] = best
        out[f"{name}_found"] = found.astype(bool)
        out[f"{name}_starts"] = starts
    return out


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        arrays = reference_answers(load_driver(tmp))
    np.savez_compressed(t.GOLDEN, **arrays)
    print(t.GOLDEN, os.path.getsize(t.GOLDEN), "bytes,", len(arrays), "arrays")

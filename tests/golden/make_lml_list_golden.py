"""Regenerates tests/golden/reference_lml_list.npz: the reference side of test_gpp_entry_matches_reference in
tests/test_gpu_lml_list.py.

The values and found flag come from the reference itself: EvaluateLogLikelihoodAtPointList
(gpp_model_selection.hpp:1274-1308), unmodified, called through tests/golden/lml_list_ref_driver.cpp, which this script
compiles against the reference headers and links to oracle/_ref/libmoe_ref.so (built by __graft_entry__.build() from a
Cornell-MOE checkout).  The script also checks each value against the reference's single-set ComputeLogLikelihood
(through oracle/_ref) before it writes the file.  Run from the repository root:

    python tests/golden/make_lml_list_golden.py
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
import test_gpu_lml_list as t  # noqa: E402

DRIVER = os.path.join(ROOT, "tests", "golden", "lml_list_ref_driver.cpp")
REF_CPP = os.environ.get("CMOE_REFERENCE_CPP") or os.path.join(os.path.dirname(ROOT), "reference", "moe",
                                                                "optimal_learning", "cpp")


def load_driver(tmp):
    """Compiles lml_list_ref_driver.cpp with the flags oracle/Makefile uses for the reference, linked to libmoe_ref.so."""
    so = os.path.join(tmp, "liblml_list_ref.so")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.run(["g++", "-std=c++14", "-O2", "-fopenmp", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "oracle", "compat"), "-I" + REF_CPP, DRIVER, "-o", so,
                    "-L" + ref_dir, "-lmoe_ref", "-Wl,-rpath," + ref_dir], check=True)
    lib = ctypes.CDLL(so)
    lib.lref_log_likelihood_at_hyperparameter_list.restype = ctypes.c_int
    return lib


def _dp(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def reference_values(lib):
    ref = orc.load_reference()
    out = {}
    for name in t.REF_CASES:
        prob, H = t._ref_case(name)
        X, y, derivs = prob["X"], prob["y"], np.ascontiguousarray(prob["derivs"], dtype=np.int32)
        N, dim = X.shape
        vals = np.empty(H.shape[0])
        found = lib.lref_log_likelihood_at_hyperparameter_list(
            ctypes.c_double(prob["alpha"]), _dp(prob["lengths"]), _dp(prob["noise"]), _dp(H), H.shape[0], _dp(X),
            _dp(y), derivs.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), derivs.size, dim, N, _dp(vals))
        single = [ref.log_marginal_likelihood(1, h[0], h[1:1 + dim], X, y, h[1 + dim:], derivs) for h in H]
        np.testing.assert_allclose(vals, single, rtol=1e-12)
        out[f"{name}_values"] = vals
        out[f"{name}_found"] = np.asarray(bool(found))
    return out


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        vals = reference_values(load_driver(tmp))
    np.savez_compressed(t.GOLDEN, **vals)
    print(t.GOLDEN, os.path.getsize(t.GOLDEN), "bytes,", len(vals), "arrays")

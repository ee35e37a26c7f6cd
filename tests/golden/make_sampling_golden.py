"""Regenerates tests/golden/reference_sampling.npz: answers of the reference's joint posterior sampling.

The samples and the argmin come from the reference itself: GaussianProcess::SamplePointsFromGP / SamplePointFromGP
(gpp_math.cpp:1761-1848) after SetExplicitSeed(seed), called through tests/golden/sampling_ref_driver.cpp, which this
script compiles against the reference headers and links to oracle/_ref/libmoe_ref.so (built by __graft_entry__.build()
from a Cornell-MOE checkout).  Alongside, the fixture keeps what those calls consume, for the device tests: the first Q
draws of NormalRNG(seed) (its constructor calls SetExplicitSeed, gpp_random.cpp:91-121), the reference's posterior mean
and Cholesky factor.  The script checks the host restatement (tests/sampling_ref.py) against the reference's answers
and that the reference returns -1 for the case whose minimum is at point 0.
Run from the repository root:  python tests/golden/make_sampling_golden.py
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
from sampling_ref import sample_from_posterior  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_sampling.npz")
DRIVER = os.path.join(ROOT, "tests", "golden", "sampling_ref_driver.cpp")
REF_CPP = os.environ.get("CMOE_REFERENCE_CPP") or os.path.join(os.path.dirname(ROOT), "reference", "moe",
                                                                "optimal_learning", "cpp")


def load_sampling_driver(tmp):
    """Compiles sampling_ref_driver.cpp with the flags oracle/Makefile uses for the reference, linked to libmoe_ref.so."""
    so = os.path.join(tmp, "libsampling_ref.so")
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    subprocess.run(["g++", "-std=c++14", "-O2", "-fopenmp", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "oracle", "compat"), "-I" + REF_CPP, DRIVER, "-o", so,
                    "-L" + ref_dir, "-lmoe_ref", "-Wl,-rpath," + ref_dir], check=True)
    lib = ctypes.CDLL(so)
    lib.sref_sample_points.restype = ctypes.c_int
    return lib


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def case(ref, drv, name, kernel, dim, N, num, seed, derivs=(), lengths=0.4, rng_seed=0, want_first_min=False):
    rng = np.random.default_rng(rng_seed)
    X = rng.uniform(size=(N, dim))
    g = len(derivs)
    y = np.sin(3 * X).sum(axis=1)
    if g:
        y = np.column_stack([y] + [3 * np.cos(3 * X[:, d]) for d in derivs]).ravel()
    noise = np.full(1 + g, 1e-2)
    lens = np.full(dim, lengths)
    gp, lm = ref.gp(kernel, 1.0, lens, X, y, noise, derivs=list(derivs))
    assert lm == 0
    Q = num * (1 + g)
    for attempt in range(1000):
        pts = rng.uniform(size=(num, dim))
        out = np.empty(Q)
        if g:  # the one-point case with the GP's derivative rows
            assert num == 1
            drv.sref_sample_point(gp.h, ctypes.c_uint(seed), _dp(np.ascontiguousarray(pts[0])), _dp(out))
            amin_ref = None
        else:
            amin_ref = drv.sref_sample_points(gp.h, ctypes.c_uint(seed), _dp(np.ascontiguousarray(pts)), num, _dp(out))
        if not want_first_min or amin_ref == -1:
            break
    else:
        raise RuntimeError("no set with the minimum at point 0 found")
    post = gp.posterior(pts, derivs_s=list(derivs), want=("mean", "chol_var"))
    assert post["rc"] == 0
    L = post["chol_var"].reshape(Q, Q).T  # column-major -> [row, col]
    w = orc.normal_draws(seed, Q)
    s, amin_restated, _ = sample_from_posterior(post["mean"], L, w, 1 + g)
    np.testing.assert_allclose(s, out, rtol=1e-12, atol=1e-14)  # the host restatement reproduces the reference
    if amin_ref is not None:
        assert amin_restated == amin_ref
    return {f"{name}_kernel": kernel, f"{name}_X": X, f"{name}_y": y, f"{name}_noise": noise, f"{name}_lengths": lens,
            f"{name}_derivs": np.asarray(derivs, dtype=np.int32), f"{name}_pts": pts, f"{name}_seed": seed,
            f"{name}_normals": w, f"{name}_mean": post["mean"], f"{name}_chol": L, f"{name}_samples": out,
            f"{name}_has_argmin": amin_ref is not None,
            f"{name}_argmin_ref": -2 if amin_ref is None else amin_ref}


def main():
    if not orc.have_reference():
        raise SystemExit("oracle/_ref/libmoe_ref.so is missing: run __graft_entry__.build() with a reference checkout")
    ref = orc.load_reference()
    with tempfile.TemporaryDirectory() as tmp:
        drv = load_sampling_driver(tmp)
        data = {}
        data.update(case(ref, drv, "se", 0, 3, 30, 40, seed=11, rng_seed=1))
        data.update(case(ref, drv, "matern", 1, 4, 25, 60, seed=12, rng_seed=2))
        data.update(case(ref, drv, "first", 0, 2, 20, 12, seed=13, rng_seed=3, want_first_min=True))
        data.update(case(ref, drv, "point", 1, 3, 15, 1, seed=14, derivs=(0, 2), rng_seed=4))
    assert data["first_argmin_ref"] == -1  # returned by the reference's SamplePointsFromGP
    data["cases"] = np.array(["se", "matern", "first", "point"])
    np.savez(OUT, **data)
    print("wrote", OUT, {c: int(data[f"{c}_argmin_ref"]) for c in data["cases"]})


if __name__ == "__main__":
    main()

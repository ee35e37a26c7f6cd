"""Generates tests/golden/reference_dkg_wide.npz: the reference side of the multistart-driver test in
tests/test_gpu_dkg_wide.py, computed by the UNMODIFIED reference (oracle/_ref/libmoe_ref.so, `make -C oracle ref
REF=...`).  Run from the repository root:

    python tests/golden/make_dkg_wide_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import oracle as orc  # noqa: E402
import test_gpu_dkg_wide as t  # noqa: E402

if __name__ == "__main__":
    vals = t.reference_values(orc.load_reference())
    np.savez_compressed(t.GOLDEN, **vals)
    print(t.GOLDEN, os.path.getsize(t.GOLDEN), "bytes,", len(vals), "arrays")

"""Build-time checks of the kernel-matched random features and the sample-function evaluator (no GPU needed, DESIGN.md
K14 addendum): `-Xptxas -v` reports no stack frame and no spills in the new kernels (both instantiations of the
evaluator, the chi^2 kernel) and in the grid kernel, whose loop is now the shared rff_accumulate.  rff_features_kernel,
which gained the chi^2_5 draw, keeps exactly the 40-byte frame of philox_normal_pair's sincos (the chi^2 draw's cosine
is rff_sincos, which has none) and no spills."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "cornell-moe_b200", "build", "rff.ptxas.log")
NO_LOCAL = ("rff_eval_kernelILb0E", "rff_eval_kernelILb1E", "rff_chi2_kernel", "rff_grid_kernel")


def _stats(name):
    blocks = open(LOG).read().split("Compiling entry function")
    block = next((b for b in blocks if name in b.split("\n")[0]), None)
    assert block is not None, name
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
    assert m, (name, block)
    return m.groups()


@pytest.mark.parametrize("name", NO_LOCAL)
def test_new_and_changed_kernels_use_no_local_memory(name):
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    assert _stats(name) == ("0", "0", "0"), name


def test_features_kernel_keeps_only_the_box_muller_frame():
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    assert _stats("rff_features_kernel") == ("40", "0", "0")

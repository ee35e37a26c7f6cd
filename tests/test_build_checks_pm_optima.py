"""Build-time check of the per-member posterior-mean optima kernels (no GPU needed): `-Xptxas -v` reports them compiled
for sm_90a without register spills; the screen and the argmin use no local memory at all, the descent keeps the
optimiser's per-thread vectors (CMOE_MAX_DIM doubles each) in its stack frame as pm_opt_kernel does (DESIGN.md K15)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "cornell-moe_b200", "build", "posterior_mean_opt.ptxas.log")
NO_LOCAL_MEMORY = ("pm_members_screen_kernel", "pm_members_argmin_kernel")
NO_SPILLS = NO_LOCAL_MEMORY + ("pm_members_opt_kernel",)


def test_pm_optima_kernels_do_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(LOG).read().split("Compiling entry function")
    for name in NO_SPILLS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None and "for 'sm_90a'" in block.split("\n")[0], name
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups()[1:] == ("0", "0"), (name, block)
        if name in NO_LOCAL_MEMORY:
            assert m.group(1) == "0", (name, block)

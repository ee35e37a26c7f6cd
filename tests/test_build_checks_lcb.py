"""Build-time check of the LCB selection kernels (no GPU needed): `-Xptxas -v` reports no stack frame and no spills,
so none of them uses local memory (DESIGN.md K13)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "cornell-moe_b200", "build", "lcb.ptxas.log")
NEW_KERNELS = ("lcb_screen_kernel", "lcb_select_kernel", "lcb_gather_kernel", "lcb_cross_kernel", "lcb_border_kernel",
               "lcb_round_kernel", "lcb_argmax_kernel")


def test_lcb_kernels_use_no_local_memory():
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(LOG).read().split("Compiling entry function")
    for name in NEW_KERNELS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None, name
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0", "0"), (name, block)

"""Build-time check of the heuristic-EI kernels (no GPU needed): `-Xptxas -v` reports them compiled for sm_90a with no
register spills and no local memory (DESIGN.md K20)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "cornell-moe_b200", "build", "heuristic_ei.ptxas.log")
KERNELS = ("hei_descent_kernel", "hei_select_kernel")


def test_heuristic_ei_kernels_do_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(LOG).read().split("Compiling entry function")
    for name in KERNELS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None and "for 'sm_90a'" in block.split("\n")[0], name
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0", "0"), (name, block)

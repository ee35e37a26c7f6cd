"""Build-time check of the hyper-parameter MAP kernels (no GPU needed): `-Xptxas -v` reports no spills for the
per-start kernels and for the exact-gradient contraction (DESIGN.md K19)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "cornell-moe_b200", "build", "model_selection.ptxas.log")
KERNELS = ("map_prep_kernel", "map_step_kernel", "map_init_kernel", "lml_grad_contract_kernelILb1E",
           "lml_grad_contract_kernelILb0E")


@pytest.mark.parametrize("name", KERNELS)
def test_map_kernels_do_not_spill(name):
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(LOG).read().split("Compiling entry function")
    block = next((b for b in blocks if name in b.split("\n")[0]), None)
    assert block is not None, name
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
    assert m and m.groups() == ("0", "0"), (name, block)

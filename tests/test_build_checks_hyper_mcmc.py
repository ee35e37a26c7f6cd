"""Build-time check of the hyper-parameter MCMC kernels (no GPU needed): `-Xptxas -v` reports no spills for the
proposal and acceptance kernels (DESIGN.md K12)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "cornell-moe_b200", "build", "model_selection.ptxas.log")
NEW_KERNELS = ("hmc_propose_kernel", "hmc_accept_kernel")


def test_mcmc_kernels_do_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(LOG).read().split("Compiling entry function")
    for name in NEW_KERNELS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None, name
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0"), (name, block)

"""Build-time check (no GPU needed): the LINE rounds of both tile builds of `kg_mc_kernel<SE,8,8>` try 6 step sizes per
batch (`kg_line_batch`, kg_mc.cuh), so a LINE half-block (8 rows of 16 samples, 3 DMMAs) runs 4 squarings and 4
accumulating FMAs per lane fewer than a batch of 8: at most 104 FP64 vector instructions in the BIG (`exp2k_shifted`)
build (120 with 8 trials) and 132 in the 64-entry-table build (148).  Neither build may trade the saved registers for
a stack frame or local-memory traffic."""
import os
import re
import shutil

import pytest

from test_build_checks_kg_tile_exp2k import OBJ, _loop_bodies

# kernel -> FP64 vector instructions of its LINE half-block, at most
LINE_HALF_BLOCK = {"kg_mc_kernelILi0ELi8ELi8ELb1E": 104, "kg_mc_kernelILi0ELi8ELi8ELb0E": 132}


@pytest.mark.parametrize("name", sorted(LINE_HALF_BLOCK))
def test_tile_line_half_block_runs_six_trials(name):
    if not os.path.exists(OBJ) or shutil.which("cuobjdump") is None:
        pytest.skip("object file or cuobjdump not available (run __graft_entry__.build() first)")
    inner = [b for b in _loop_bodies(OBJ, name) if b[0] == 3]
    assert inner, f"{name}: no 3-DMMA loop (LINE half-block)"
    _, fp64, _ = min(inner, key=lambda b: b[2])
    assert fp64 <= LINE_HALF_BLOCK[name], f"{name}: {fp64} FP64 vector instructions per LINE half-block"


@pytest.mark.parametrize("name", sorted(LINE_HALF_BLOCK))
def test_tile_builds_have_no_stack_or_local_memory(name):
    log = OBJ.replace(".o", ".ptxas.log")
    if not os.path.exists(log):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    block = next(b for b in open(log).read().split("Compiling entry function") if name in b.split("\n")[0])
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
    assert m and m.groups() == ("0", "0", "0"), block

"""Build-time check of the q-KG tile accumulation kernel (no GPU needed): `kg_acc_tile_kernel<8, 8>` runs its training
rows on FP64 DMMA and keeps its row operands and accumulators in registers; local-memory traffic in it (LDL / STL in the
SASS) would mean they no longer fit (DESIGN.md K6)."""
import os
import re
import shutil

import pytest

from test_build_checks_kg_tile import BUILD, _function_sass

ACC_TILE = "kg_acc_tile_kernelILi8ELi8E"  # kg_acc_tile_kernel<8, 8>


def test_tile_accumulation_kernel_runs_on_dmma_and_does_not_spill():
    obj = os.path.join(BUILD, "kg_mc_inst_8.o")
    if not os.path.exists(obj) or shutil.which("cuobjdump") is None:
        pytest.skip("object file or cuobjdump not available (run __graft_entry__.build() first)")
    insns = _function_sass(obj, ACC_TILE)
    assert insns, "kg_acc_tile_kernel<8, 8> is missing from kg_mc_inst_8.o"
    assert any("DMMA" in t for t in insns), "the tile accumulation kernel no longer runs its rows on DMMA"
    local = [t for t in insns if re.search(r"\b(LDL|STL)\b", t)]
    assert not local, f"{len(local)} local-memory instructions in kg_acc_tile_kernel<8,8>: {local[:8]}"
    log = os.path.join(BUILD, "kg_mc_inst_8.ptxas.log")
    if os.path.exists(log):
        blocks = open(log).read().split("Compiling entry function")
        block = next(b for b in blocks if ACC_TILE in b.split("\n")[0])
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0"), block

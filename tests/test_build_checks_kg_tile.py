"""Build-time check of the q-KG tile instantiation (no GPU needed): `kg_mc_kernel<SE, 8, 8>` runs at 2 CTAs per SM so
that its tile rounds fit in registers; local-memory traffic in it (spill stores and loads, LDL / STL in the SASS) would
mean the register budget was lost again (DESIGN.md K6)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "cornell-moe_b200", "build")
TILE = "kg_mc_kernelILi0ELi8ELi8E"  # kg_mc_kernel<CMOE_KERNEL_SQUARE_EXPONENTIAL, 8, 8>


def _function_sass(obj, name):
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, take = [], False
    for line in sass.split("\n"):
        if "Function :" in line:
            take = name in line
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and take:
            out.append(m.group(1).strip())
    return out


def test_tile_instantiation_of_the_kg_mc_kernel_does_not_spill():
    obj = os.path.join(BUILD, "kg_mc_inst_8.o")
    if not os.path.exists(obj) or shutil.which("cuobjdump") is None:
        pytest.skip("object file or cuobjdump not available (run __graft_entry__.build() first)")
    insns = _function_sass(obj, TILE)
    assert any("DMMA" in t for t in insns), "the tile instantiation no longer runs its rows on DMMA"
    local = [t for t in insns if re.search(r"\b(LDL|STL)\b", t)]
    assert not local, f"{len(local)} local-memory instructions in kg_mc_kernel<SE,8,8>: {local[:8]}"
    # the compiler's own account, where the build kept it (cornell-moe_b200/Makefile writes it next to the object)
    log = os.path.join(BUILD, "kg_mc_inst_8.ptxas.log")
    if os.path.exists(log):
        blocks = open(log).read().split("Compiling entry function")
        block = next(b for b in blocks if TILE in b.split("\n")[0])
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0"), block

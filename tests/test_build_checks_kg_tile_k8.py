"""Build-time check (no GPU needed): the q-KG tile kernels issue their K = 8 products as one DMMA.16x8x8 instead of two
chained DMMA.16x8x4.  Interleaved with the element-wise FP64 work of the row loops a DMMA costs more than its 16 cycles
alone, per instruction, so half the instructions is most of the gain of DESIGN.md K6 "K = 8 products as one DMMA"; the
two forms give the same bits."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "cornell-moe_b200", "build", "kg_mc_inst_8.o")
KERNELS = {
    # <SE,8,8>, both builds: a LINE half-block has 3 products, a POINT block 6; the row loop and the tail block each
    "kg_mc_kernelILi0ELi8ELi8ELb1E": 18,
    "kg_mc_kernelILi0ELi8ELi8ELb0E": 18,
    "kg_acc_tile_kernelILi8ELi8E": 8,  # exponents and R products of its 4 row tiles
}


def _dmma_shapes(obj, name):
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    shapes, take = [], False
    for line in sass.split("\n"):
        if "Function :" in line:
            take = name in line
            continue
        m = re.search(r"\bDMMA\.(\d+x\d+x\d+)", line)
        if m and take:
            shapes.append(m.group(1))
    return shapes


@pytest.mark.parametrize("name", sorted(KERNELS))
def test_tile_products_use_k8_dmma(name):
    if not os.path.exists(OBJ) or shutil.which("cuobjdump") is None:
        pytest.skip("object file or cuobjdump not available (run __graft_entry__.build() first)")
    shapes = _dmma_shapes(OBJ, name)
    assert shapes, f"{name}: no DMMA"
    assert "16x8x4" not in shapes, f"{name}: {shapes.count('16x8x4')} DMMA.16x8x4 left"
    assert shapes.count("16x8x8") >= KERNELS[name], (name, shapes)

"""Build-time checks of the hyper-parameter gradient list kernels (no GPU needed): `-Xptxas -v` reports no spills for
any of them, and the two kernels that carry the O(n^3) work of K^-1 (the off-diagonal blocks of L^-1 and L^-T L^-1)
run it on the FP64 tensor pipe (DESIGN.md K11)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "cornell-moe_b200", "build")
OBJ = os.path.join(BUILD, "model_selection.o")
LOG = os.path.join(BUILD, "model_selection.ptxas.log")
NEW_KERNELS = ("tri_inv_diag_kernel", "tri_inv_offdiag_kernel", "inv_syrk_kernel", "lml_grad_contract_kernel",
               "lml_grad_reduce_kernel", "lml_solve_kernel")
DMMA_KERNELS = ("tri_inv_offdiag_kernel", "inv_syrk_kernel")


def test_gradient_list_kernels_do_not_spill():
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(LOG).read().split("Compiling entry function")
    for name in NEW_KERNELS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None, name
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0"), (name, block)


def test_inverse_kernels_run_on_dmma():
    if not os.path.exists(OBJ) or shutil.which("cuobjdump") is None:
        pytest.skip("object file or cuobjdump not available (run __graft_entry__.build() first)")
    sass = subprocess.run(["cuobjdump", "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in sass.split("\n"):
        if "Function :" in line:
            cur = line.split("Function :")[1].strip()
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    for name in DMMA_KERNELS:
        body = [ln for f, lines in funcs.items() if name in f for ln in lines]
        assert body, name
        assert any("DMMA" in ln for ln in body), f"{name} has no DMMA instruction"

"""Build-time check of the large-set q-EI kernels (no GPU needed): `-Xptxas -v` reports no stack frame and no spills for
any of them, and the forward tiles and the adjoint products issue FP64 tensor-core instructions (DESIGN.md K16)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "cornell-moe_b200", "build")
KERNELS = ("ei_mc_tile_kernel", "ei_winner_kernel", "ei_value_kernel", "ei_bucket_kernel", "ei_cbar_kernel",
           "ei_ctc_kernel", "transpose_kernel", "gemm_nn_kernel", "ei_grad_kernel")
DMMA_KERNELS = ("ei_mc_tile_kernel", "ei_ctc_kernel", "gemm_nn_kernel")


def test_ei_large_kernels_use_no_local_memory():
    log = os.path.join(BUILD, "ei_large.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(log).read().split("Compiling entry function")
    for name in KERNELS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None, name
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0", "0"), (name, block)


def test_ei_large_products_use_dmma():
    obj = os.path.join(BUILD, "ei_large.o")
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(cuobjdump):
        pytest.skip("object or cuobjdump not available (run __graft_entry__.build() first)")
    sass = subprocess.run([cuobjdump, "-sass", obj], check=True, capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    for name in DMMA_KERNELS:
        body = next((f for f in funcs if name in f.split("\n")[0]), None)
        assert body is not None, name
        assert "DMMA" in body, name

"""Build-time check of the large-union q-KG kernels (no GPU needed, DESIGN.md K17): `-Xptxas -v` reports no more local
memory for the stage kernels of kg_large.cu than K17 records and none for the DMMA products and the transpose it shares
with ei_large.cu,
those products issue FP64 tensor-core instructions, and the inner-optimiser builds (kg_mc_large_kernel) spill no more
than K17 records."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "cornell-moe_b200", "build")
STAGE_KERNELS = ("kgl_normals_kernel", "kgl_pack_kernel", "kgl_noise_kernel", "kgl_best_kernel",
                 "kgl_disc_cov_kernel", "kgl_argmin_kernel", "kgl_weights_kernel",
                 "kgl_kx_kernel", "kgl_lbar_kernel", "kgl_grad_kernel")
# local memory the stage kernels are allowed, (stack frame, spill stores, spill loads) in bytes, as DESIGN.md K17 records:
# the Box-Muller sine and cosine's slow-path reduction, the raw minimiser kept as an indexable array, and the gradient
# contraction's spill
STAGE_LOCAL = {"kgl_normals_kernel": (40, 0, 0), "kgl_kx_kernel": (256, 0, 0), "kgl_grad_kernel": (8, 4, 12)}
# the scan (W^T Z), the weights (B C), R (Kx C^T), R2 (B 2 Sigmabar) and the adjoint's C^T Cbar
SHARED_DMMA_KERNELS = ("gemm_nn_kernel", "ei_ctc_kernel")
# every kernel of ei_large.cu that the stages launch: the DMMA products and the batched transpose (B^T, W^T, C^T)
SHARED_KERNELS = SHARED_DMMA_KERNELS + ("transpose_kernel",)
# spill stores (bytes) of every kg_mc_large_kernel build, (kernel, padded dim, wide) -> bytes, as DESIGN.md K17 records
MAX_SPILL_STORES = {
    (0, 2, 0): 0, (1, 2, 0): 0, (0, 4, 0): 0, (1, 4, 0): 0, (0, 6, 0): 0, (1, 6, 0): 0, (0, 8, 0): 0, (1, 8, 0): 0,
    (0, 12, 0): 4, (1, 12, 0): 0, (0, 16, 0): 228, (1, 16, 0): 220, (0, 32, 0): 1928, (1, 32, 0): 1828,
    (0, 12, 1): 0, (1, 12, 1): 0, (0, 16, 1): 160, (1, 16, 1): 0, (0, 32, 1): 1700, (1, 32, 1): 1404,
}


def _blocks(log):
    path = os.path.join(BUILD, log)
    if not os.path.exists(path):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    return open(path).read().split("Compiling entry function")


def _usage(block):
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
    assert m, block
    return tuple(int(x) for x in m.groups())


def test_kg_large_stage_and_shared_kernels_use_no_local_memory():
    blocks = _blocks("kg_large.ptxas.log")
    for name in STAGE_KERNELS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None, name
        assert all(u <= a for u, a in zip(_usage(block), STAGE_LOCAL.get(name, (0, 0, 0)))), (name, block)
    blocks = _blocks("ei_large.ptxas.log")
    for name in SHARED_KERNELS:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None, name
        assert _usage(block) == (0, 0, 0), (name, block)


def test_kg_large_products_use_dmma():
    obj = os.path.join(BUILD, "ei_large.o")
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(cuobjdump):
        pytest.skip("object or cuobjdump not available (run __graft_entry__.build() first)")
    sass = subprocess.run([cuobjdump, "-sass", obj], check=True, capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    for name in SHARED_DMMA_KERNELS:
        body = next((f for f in funcs if name in f.split("\n")[0]), None)
        assert body is not None, name
        assert "DMMA" in body, name


@pytest.mark.parametrize("unit", ["kg_mc_inst_2", "kg_mc_inst_4", "kg_mc_inst_6", "kg_mc_inst_8", "kg_mc_inst_12",
                                  "kg_mc_inst_16", "kg_mc_inst_32", "kg_mc_wide_12", "kg_mc_wide_16", "kg_mc_wide_32"])
def test_inner_optimiser_builds_do_not_spill(unit):
    blocks = [b for b in _blocks(unit + ".ptxas.log") if "kg_mc_large_kernel" in b.split("\n")[0]]
    assert len(blocks) == 2, unit  # SquareExponential and Matern-5/2
    for block in blocks:
        m = re.search(r"kg_mc_large_kernelILi(\d)ELi(\d+)ELb(\d)E", block.split("\n")[0])
        key = tuple(int(x) for x in m.groups())
        assert _usage(block)[1] <= MAX_SPILL_STORES[key], (unit, key, block)

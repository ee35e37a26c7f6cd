"""Build-time checks of the random-feature sampler's kernels (no GPU needed, DESIGN.md K14): `-Xptxas -v` reports no
stack frame and no spills, and rff_gram_kernel runs on the FP64 tensor pipe (DMMA).  rff_features_kernel is left out of
the stack check: its 40-byte frame is the slow-path argument reduction inside philox_normal_pair's sincos (the Box-Muller
step shared with every Philox consumer, sample_rows_kernel included), which its arguments in [0, 2 pi) never take."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "cornell-moe_b200", "build")
LOG = os.path.join(BUILD, "rff.ptxas.log")
NO_LOCAL = ("rff_design_kernel", "rff_gram_kernel", "rff_theta_kernel", "rff_grid_kernel", "best_of_parts_kernel",
            "rff_opt_kernel")


def test_rff_kernels_use_no_local_memory():
    if not os.path.exists(LOG):
        pytest.skip("ptxas log not available (run __graft_entry__.build() first)")
    blocks = open(LOG).read().split("Compiling entry function")
    for name in NO_LOCAL:
        block = next((b for b in blocks if name in b.split("\n")[0]), None)
        assert block is not None, name
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", block)
        assert m and m.groups() == ("0", "0", "0"), (name, block)


def test_rff_gram_kernel_uses_dmma():
    obj = os.path.join(BUILD, "rff.o")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(obj) or not os.path.exists(tool):
        pytest.skip("rff.o or cuobjdump not available")
    sass = subprocess.run([tool, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    gram = next((f for f in funcs if "rff_gram_kernel" in f.split("\n")[0]), None)
    assert gram is not None
    assert re.search(r"\bDMMA\.", gram), "rff_gram_kernel has no DMMA instruction"

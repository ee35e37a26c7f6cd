"""Build-time check (no GPU needed): the row loops of the BIG tile build of `kg_mc_kernel<SE,8,8>` and the sample loop of
`kg_acc_tile_kernel<8,8>` run their exps as exp2k_shifted, with the operands in kKappa units and each sample's exponent
term folded into the rounding constant (kg_mc.cuh).  The FP64 pipe bounds these loops (DESIGN.md K6), so their FP64
vector instruction counts (DFMA + DMUL + DADD) are pinned: 72 per POINT block (9 per row; 88 with exp_tab2k), 120 per
LINE half-block (30 per row; 132 with exp_tab2k) and 112 per accumulation group of 8 samples (144 with exp_tab2k)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "cornell-moe_b200", "build", "kg_mc_inst_8.o")
# kernel -> {DMMA per loop body: max FP64 vector instructions in it}
LOOPS = {
    "kg_mc_kernelILi0ELi8ELi8ELb1E": {6: 72, 3: 120},  # POINT block, LINE half-block
    "kg_acc_tile_kernelILi8ELi8E": {8: 112},          # 8-sample group of 4 row tiles
}


def _loop_bodies(obj, name):
    """(DMMA, FP64 vector, instructions) of every loop body of the kernel: the span from a backward branch's target to
    the branch."""
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    ins, take = [], False
    for line in sass.split("\n"):
        if "Function :" in line:
            take = name in line
            continue
        m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and take:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    index = {a: i for i, (a, _) in enumerate(ins)}
    bodies = []
    for i, (a, text) in enumerate(ins):
        m = re.search(r"\bBRA\b.*?(0x[0-9a-f]+)", text)
        if m and int(m.group(1), 16) <= a and int(m.group(1), 16) in index:
            ops = [re.sub(r"^@!?U?P\w+\s+", "", t).split()[0] for _, t in ins[index[int(m.group(1), 16)]:i + 1]]
            dmma = sum(o.startswith("DMMA") for o in ops)
            fp64 = sum(bool(re.match(r"D(FMA|MUL|ADD)\b", o)) for o in ops)
            bodies.append((dmma, fp64, len(ops)))
    return bodies


@pytest.mark.parametrize("name", sorted(LOOPS))
def test_tile_row_loops_fp64_vector_count(name):
    if not os.path.exists(OBJ) or shutil.which("cuobjdump") is None:
        pytest.skip("object file or cuobjdump not available (run __graft_entry__.build() first)")
    bodies = _loop_bodies(OBJ, name)
    assert bodies, f"{name}: no loops"
    for dmma, limit in LOOPS[name].items():
        # the innermost loop with this many DMMAs: the row (sample) loop, not a loop around it
        inner = [b for b in bodies if b[0] == dmma]
        assert inner, (name, dmma, bodies)
        _, fp64, n = min(inner, key=lambda b: b[2])
        assert fp64 <= limit, f"{name}: {fp64} FP64 vector instructions in the {dmma}-DMMA loop (at most {limit})"

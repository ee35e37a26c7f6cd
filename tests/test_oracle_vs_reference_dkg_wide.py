"""Pins the plain-C oracle (oracle/moe_oracle.c) against the UNMODIFIED reference for d-KG with full gradient
observations past eight partials (g = 10 and g = 16): without a compiled reference the oracle is the checker of
tests/test_gpu_dkg_wide.py.

The reference's answers are stored in tests/golden/reference_calls_dkg_wide.npz (see ref_replay.py).  To regenerate them
from the reference compiled into oracle/_ref/libmoe_ref.so, which also runs every comparison live:

    CMOE_RECORD_REFERENCE=1 python -m pytest tests/test_oracle_vs_reference_dkg_wide.py
"""
import os

import numpy as np
import pytest

import oracle as orc
from ref_replay import RECORD, TapeFile
from synth import DISCRETE_ONLY_GD, EXAMPLE_INNER_GD, make_problem, unit_bounds

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_calls_dkg_wide.npz")


@pytest.fixture(scope="module")
def tapes():
    f = TapeFile(GOLDEN)
    yield f
    if RECORD:
        f.save()


@pytest.fixture
def tape(tapes, request):
    return tapes.tape(request.node.name)


@pytest.mark.parametrize("kernel", [0, 1])
@pytest.mark.parametrize("gd", [DISCRETE_ONLY_GD, EXAMPLE_INNER_GD], ids=["discrete", "inner"])
@pytest.mark.parametrize("d,q", [(10, 2), (16, 1)])
def test_kg_full_gradients(tape, d, q, gd, kernel):
    o, r = orc.load_oracle(), tape.backend()
    prob = make_problem(9, d, g_idx=tuple(range(d)), seed=9 + d, noise=0.1)
    gps = []
    for b in (o, r):
        gp, lm = b.gp(kernel, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
        assert lm == 0
        gps.append(gp)
    go, gr = gps
    rng = np.random.default_rng(27 + d)
    Xq = rng.uniform(size=(q, d))
    disc = rng.uniform(size=(5, d))
    mc = 16
    table = rng.standard_normal((mc // 2) * q * (1 + d))
    best = float(go.mean_additional(disc).min())
    vo, grad_o = go.kg(Xq, None, mc, best, table, gd, unit_bounds(d), disc, grad=True)
    vr, grad_r = gr.kg(Xq, None, mc, best, table, gd, unit_bounds(d), disc, grad=True)
    np.testing.assert_allclose(vo, vr, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(grad_o, grad_r, rtol=1e-6, atol=1e-9)

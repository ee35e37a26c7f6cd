"""GPU tests of the q-KG start-point table (kg_start_kernel): without derivative observations, a sample's inner descent
starts from a value and gradient combined from a per-(candidate, discretisation point) table instead of a POINT round.

- Values and gradients match the CPU checker with table-fed normals at the bench shape and with pending points, one
  fidelity coordinate, Matern-5/2, the global-memory body, max_num_steps = 0 and max_num_restarts = 2.
- The counters match the ones the library recorded before the table existed (tests/golden/kg_start_parent_counters.json,
  written by tests/golden/make_kg_start_counters.py): posterior evaluations, accepted steps and LINE batches are equal,
  and each sample runs exactly one POINT round fewer (a restart run starts from the previous run's end point, whose value
  and gradient are known, so only a sample's first run ever had a start round).
- A candidate's results do not depend on the batch it is evaluated in.
"""
import json
import os

import numpy as np
import pytest

from gpu_util import checker
from synth import EXAMPLE_INNER_GD, make_problem, unit_bounds

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kg_start_parent_counters.json")
COUNTERS = ("posterior_evals", "line_search_steps", "point_evals", "line_batches", "mc_samples")

# name: (kernel, N, d, q, p, num_fidelity, inner optimiser, num_mc)
CASES = {
    "bench_shape": (0, 500, 8, 8, 0, 0, EXAMPLE_INNER_GD, 64),
    "pending_points": (0, 120, 6, 3, 2, 0, EXAMPLE_INNER_GD, 64),
    "one_fidelity": (0, 80, 4, 2, 0, 1, EXAMPLE_INNER_GD, 64),
    "matern52": (1, 200, 8, 4, 0, 0, EXAMPLE_INNER_GD, 64),
    "global_memory_body": (0, 1500, 8, 8, 0, 0, EXAMPLE_INNER_GD, 32),  # N (DIMP + QP + 2) doubles past 200 KiB
    "max_steps_0": (0, 100, 5, 3, 0, 0, [1, 0, 1, 3, 0.0, 1.0, 0.1, 1e-10], 64),
    "max_restarts_2": (0, 100, 8, 8, 0, 0, [1, 6, 2, 3, 0.0, 1.0, 0.1, 1e-10], 64),
}


def case_inputs(name):
    kernel, N, d, q, p, nf, gd, mc = CASES[name]
    prob = make_problem(N, d, seed=N + 7 * d + q, noise=0.05)
    rng = np.random.default_rng(len(name) * 101 + N)
    cands = rng.uniform(size=(2, q, d))
    Xp = rng.uniform(size=(p, d)) if p else None
    disc = rng.uniform(size=(8, d - nf))
    table = rng.standard_normal((mc // 2) * (q + p))
    return prob, dict(kernel=kernel, nf=nf, gd=gd, mc=mc, cands=cands, Xp=Xp, disc=disc, table=table)


def run_case(capi, name, ref=None):
    """(kg, grad, counters) of the case on the device; with a checker `ref`, also (values, gradients) of the checker."""
    prob, c = case_inputs(name)
    gp = capi.GaussianProcess(c["kernel"], prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"],
                              prob["derivs"])
    d, nf = prob["dim"], c["nf"]
    best = 0.1
    kg, grad, st = gp.kg(c["cands"], c["Xp"], c["mc"], best, c["gd"], unit_bounds(d - nf), c["disc"], num_fidelity=nf,
                         table=c["table"], grad=True, stats=True)
    out = {"kg": kg, "grad": grad, "stats": {k: int(st[k]) for k in COUNTERS}}
    if ref is not None:
        r, lm = ref.gp(c["kernel"], prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
        assert lm == 0
        out["ref"] = [r.kg(c["cands"][i], c["Xp"], c["mc"], best, c["table"], c["gd"], unit_bounds(d - nf), c["disc"],
                           num_fidelity=nf, grad=True) for i in range(len(c["cands"]))]
    return out


@pytest.fixture(scope="module")
def capi():
    from cornell_moe_b200 import capi as c
    assert c.device_count() > 0
    return c


@pytest.fixture(scope="module")
def parent_counters():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(CASES))
def test_start_table_matches_checker(capi, name):
    out = run_case(capi, name, ref=checker())
    for i, (v, g) in enumerate(out["ref"]):
        np.testing.assert_allclose(out["kg"][i], v, rtol=1e-7, atol=1e-10)
        np.testing.assert_allclose(out["grad"][i], g, rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("name", sorted(CASES))
def test_start_table_drops_one_point_round_per_sample(capi, parent_counters, name):
    st = run_case(capi, name)["stats"]
    old = parent_counters[name]
    print(name, "parent", old, "now", st)
    for k in ("posterior_evals", "line_search_steps", "line_batches", "mc_samples"):
        assert st[k] == old[k], k
    assert st["point_evals"] == old["point_evals"] - st["mc_samples"]


def test_start_table_results_do_not_depend_on_batch(capi):
    """16 candidates at N = 500, d = 8, q = 6 with 2 pending points, in one call and in subsets of 1 and 5:
    bit-identical values and gradients (the table of a candidate is computed by its own CTAs, in a fixed order)."""
    prob = make_problem(500, 8, seed=77, noise=1e-2)
    gp = capi.GaussianProcess(0, prob["alpha"], prob["lengths"], prob["X"], prob["y"], prob["noise"], prob["derivs"])
    rng = np.random.default_rng(5)
    cands = rng.uniform(size=(16, 6, 8))
    Xp = rng.uniform(size=(2, 8))
    disc = rng.uniform(size=(10, 8))
    mc = 8192
    kg, grad = gp.kg(cands, Xp, mc, 0.1, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xC0FFEE, grad=True)
    assert np.all(np.isfinite(kg)) and np.all(np.isfinite(grad))
    for size in (1, 5):
        for s in range(0, 16, size):
            k, g = gp.kg(cands[s:s + size], Xp, mc, 0.1, EXAMPLE_INNER_GD, unit_bounds(8), disc, seed=0xC0FFEE,
                         grad=True)
            np.testing.assert_array_equal(k, kg[s:s + size])
            np.testing.assert_array_equal(g, grad[s:s + size])

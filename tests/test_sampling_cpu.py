"""CPU checks of joint posterior sampling: the host restatement against the reference's golden answers, the Latin
hypercube's stratification, and the input checks of the C ABI and the GPP surface that need no device."""
import os
import sys

import numpy as np
import pytest

import oracle as orc
from cornell_moe_b200 import capi
from sampling_ref import latin_hypercube, sample_from_posterior

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "cornell-moe_b200"))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "reference_sampling.npz"))


@pytest.mark.parametrize("name", [str(c) for c in GOLDEN["cases"]])
def test_restatement_matches_reference_answers(name):
    g = {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files if k.startswith(name + "_")}
    derivs = list(g["derivs"])
    gp, lm = orc.load_oracle().gp(int(g["kernel"]), 1.0, g["lengths"], g["X"], g["y"], g["noise"], derivs=derivs)
    assert lm == 0
    Q = g["pts"].shape[0] * (1 + len(derivs))
    post = gp.posterior(g["pts"], derivs_s=derivs, want=("mean", "chol_var"))
    assert post["rc"] == 0
    s, amin_ref, amin = sample_from_posterior(post["mean"], post["chol_var"].reshape(Q, Q).T, g["normals"],
                                              1 + len(derivs))
    np.testing.assert_allclose(s, g["samples"], rtol=1e-10, atol=1e-12)
    if g["has_argmin"]:  # SamplePointsFromGP's return value; SamplePointFromGP has none
        assert amin_ref == int(g["argmin_ref"])
        assert amin == max(0, int(g["argmin_ref"]))


def test_golden_covers_a_minimum_at_point_zero():
    assert any(bool(GOLDEN[f"{c}_has_argmin"]) and int(GOLDEN[f"{c}_argmin_ref"]) == -1 for c in GOLDEN["cases"])


@pytest.mark.parametrize("num_pts,seed,draw", [(1, 0, 0), (7, 3, 5), (256, 0xC0FFEE, 2**40 + 3), (1000, 9, 1)])
def test_latin_hypercube_uses_every_stratum_once(num_pts, seed, draw):
    bounds = np.array([[0.0, 1.0], [-2.0, 3.0], [5.0, 5.5], [1.0, 1.0]])
    x = latin_hypercube(seed, draw, num_pts, bounds)
    assert x.shape == (num_pts, 4)
    assert np.all(x >= bounds[:, 0]) and np.all(x <= bounds[:, 1])
    for i in range(3):
        lo, hi = bounds[i]
        strata = np.floor((x[:, i] - lo) / (hi - lo) * num_pts).astype(int)
        assert sorted(np.minimum(strata, num_pts - 1)) == list(range(num_pts))
    assert np.all(x[:, 3] == 1.0)
    # a pure function of (seed, draw); another draw gives other points
    np.testing.assert_array_equal(x, latin_hypercube(seed, draw, num_pts, bounds))
    if num_pts > 1:
        assert not np.array_equal(x, latin_hypercube(seed, draw + 1, num_pts, bounds))


def test_latin_hypercube_checks_its_inputs():
    with pytest.raises(capi.InvalidValueError):
        capi.latin_hypercube(1, 4, [[1.0, 0.0]])
    with pytest.raises(capi.InvalidValueError):
        capi.latin_hypercube(1, 4, [[0.0, np.inf]])
    with pytest.raises(capi.BoundsError):
        capi.latin_hypercube(1, 0, [[0.0, 1.0]])
    with pytest.raises(capi.BoundsError):
        capi.latin_hypercube(1, 8193, [[0.0, 1.0]])
    with pytest.raises(capi.BoundsError):
        capi.latin_hypercube(0, 4, [[0.0, 1.0]])
    with pytest.raises(capi.BoundsError):
        capi.latin_hypercube(1, 4, np.tile([0.0, 1.0], 33))


@pytest.mark.skipif(capi.device_count() > 0, reason="checks the behaviour without a device")
def test_latin_hypercube_without_device():
    with pytest.raises(capi.NoDeviceError):
        capi.latin_hypercube(2, 4, [[0.0, 1.0]])


def test_gpp_sampling_methods_have_the_reference_signatures():
    import GPP  # noqa: E402

    doc = GPP.GaussianProcess.sample_point_from_gp.__doc__
    assert "point_to_sample" in doc
    doc = GPP.GaussianProcess.sample_global_optima.__doc__
    assert "num_optima" in doc and "inner_number" in doc and "domain_bounds" in doc
    assert "seed" in GPP.GaussianProcess.set_explicit_seed.__doc__
    assert "seed" in GPP.GaussianProcess.set_randomized_seed.__doc__

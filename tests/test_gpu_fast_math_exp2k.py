"""exp2k_shifted (kg_mc.cuh), the exp of the BIG tile build of the q-KG kernels, run on the device one argument per
thread through libcmoe_probe.so: 2^((t + H) / 2048) for an argument t in 2048ths of a binary exponent and an integer H
passed as the rounding constant 1.5 2^52 + H.  Held to exp_tab2k's documented bound over the same range (scaled by
kKappa = 2048 log2 e), with H out to kKappa x 1.8e7, the largest |hq| of the range contract (kFastPathRadius); exactly 1
at t = H = 0; and its exponent n = round(t + H) and k = n >> 11 are exp_tab2k's on shared arguments."""
import ctypes
import os
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "cornell-moe_b200", "libcmoe_probe.so")
LD = np.longdouble
EXP2K, EXP_TAB2K_NK = 7, 8  # probe routine ids (fast_math_probe.cu)
BOUND = 4.0e-16             # documented max relative error (kg_mc.cuh, exp2k_shifted)
KAPPA = 2048.0 * 1.4426950408889634  # kKappa, the double the kernels use
LN2 = float(mp.log(2))
ACC_LO, ACC_HI = KAPPA * -1000.0 * LN2, KAPPA * 700.0  # accurate range of t + H (exp_tab2k's, in kKappa units)
H_MAX = float(np.rint(KAPPA * 1.8e7))  # the largest |H|: hq = -(6000)^2 / 2 at the range contract's edge
NS = 1_000_000


@pytest.fixture(scope="module")
def probe():
    lib = ctypes.CDLL(PROBE)
    lib.cmoe_probe_eval.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int]
    lib.cmoe_probe_eval.restype = ctypes.c_int

    def run(routine, x, n_in, n_out):
        x = np.ascontiguousarray(x, dtype=np.float64)
        n = x.size // n_in
        out = np.empty(n * n_out)
        err = lib.cmoe_probe_eval(routine, x.ctypes.data, n, out.ctypes.data, 0)
        assert err == 0, f"cmoe_probe_eval({routine}) returned {err}"
        return out.reshape(n, n_out)
    return run


def _exp2k(probe, t, H):
    return probe(EXP2K, np.stack([t, H], axis=1).ravel(), 2, 3)


def _arguments(rng):
    """(t, H) with t + H uniform over the accurate range and H: 0, small, and out to +-H_MAX.  t is rounded to a double,
    so the exact sum is formed again from the rounded t (the long double holds it exactly: |t|, |H| < 2^36, so t is a
    multiple of 2^-17)."""
    total = np.concatenate([rng.uniform(ACC_LO, ACC_HI, NS), rng.uniform(-2048.0, 2048.0, NS // 5)])
    H = np.concatenate([np.zeros(total.size // 4), np.rint(rng.uniform(-4096, 4096, total.size // 4)),
                        np.rint(rng.uniform(-H_MAX, H_MAX, total.size - 2 * (total.size // 4)))])
    rng.shuffle(H)
    t = total - H
    return t, H


def test_exp2k_bulk_accuracy(probe):
    t, H = _arguments(np.random.default_rng(2048))
    got = _exp2k(probe, t, H)[:, 0]
    x = t.astype(LD) + H.astype(LD)
    ref = np.exp2(x / LD(2048))
    rel = np.abs((got.astype(LD) - ref) / ref)
    worst = float(rel.max())
    print(f"\nexp2k_shifted: max relative error {worst:.3e} ({worst / 2.0 ** -53:.2f} u) over {t.size} arguments "
          f"(documented {BOUND:.1e})")
    assert worst <= BOUND, (worst, float(t[np.argmax(rel)]), float(H[np.argmax(rel)]))


def test_exp2k_edges(probe):
    assert _exp2k(probe, np.array([0.0, -0.0]), np.zeros(2))[:, 0].tolist() == [1.0, 1.0]
    mp.mp.prec = 200
    ts, Hs = [], []
    for H in (0.0, 1.0, -1.0, 2047.0, -2048.0, H_MAX, -H_MAX):
        for tot in (0.0, 0.5, -0.5, 1.5, 2047.5, -2048.5, 1024.0, ACC_HI, ACC_LO, np.rint(ACC_LO) + 0.5):
            for v in (tot, np.nextafter(tot, -np.inf), np.nextafter(tot, np.inf)):
                t = v - H
                if Fraction(t) + Fraction(H) == Fraction(v):  # keep the exactly shifted ones
                    ts.append(t)
                    Hs.append(H)
    ts, Hs = np.array(ts), np.array(Hs)
    got = _exp2k(probe, ts, Hs)[:, 0]
    worst = 0.0
    for t, H, g in zip(ts, Hs, got):
        x = mp.mpf(float(t)) + mp.mpf(float(H))
        ref = mp.power(2, x / 2048)
        rel = float(abs((mp.mpf(float(g)) - ref) / ref))
        worst = max(worst, rel)
        assert rel <= BOUND, (float(t), float(H), float(g), rel)
    print(f"\nexp2k_shifted: max relative error {worst:.3e} at {ts.size} edge arguments (200-bit reference)")
    # below the accurate range: finite, in [0, 2^-999] (a zero contribution to every kernel sum), for every H
    low = np.array([ACC_LO - 1.0, ACC_LO * 2, KAPPA * -2.3e7 / 2])
    for H in (0.0, H_MAX, -H_MAX):
        r = _exp2k(probe, low - H, np.full(low.size, H))[:, 0]
        assert np.all(np.isfinite(r)) and np.all(r >= 0.0) and np.all(r <= 2.0 ** -999), (H, r)


def test_exp2k_exponent_matches_exp_tab2k(probe):
    """On t natural and t' = fl(kKappa t) split as t' - H + H, exp2k_shifted rounds t' where exp_tab2k rounds kKappa t
    with one FMA: the same n and k wherever both round to the same integer (all but arguments within an ulp of a
    half-integer, which are left out)."""
    rng = np.random.default_rng(11)
    tn = np.concatenate([rng.uniform(-1000.0 * LN2, 700.0, NS // 2), rng.uniform(-1.8e7, -1000.0 * LN2, NS // 10),
                         rng.uniform(-8.0, 8.0, NS // 10)])
    tp = KAPPA * tn
    H = np.rint(rng.uniform(0.0, 1.0, tn.size) * tp)  # same sign as t', |H| <= |t'|: t' - H is exact
    t = tp - H
    assert np.all(t.astype(LD) + H.astype(LD) == tp.astype(LD))
    frac = np.abs(tp - np.rint(tp))
    keep = np.abs(frac - 0.5) > 1e-3  # fl(kKappa t) and kKappa t round to the same integer
    assert keep.mean() > 0.99
    t, H, tn = t[keep], H[keep], tn[keep]
    new = _exp2k(probe, t, H)
    old = probe(EXP_TAB2K_NK, tn, 1, 2)
    np.testing.assert_array_equal(new[:, 1], old[:, 0])  # n (the low word: exact for |n| < 2^31)
    np.testing.assert_array_equal(new[:, 2], old[:, 1])  # k = n >> 11, clamped at -1000
    n = np.rint(tp[keep])
    np.testing.assert_array_equal(new[:, 2], np.maximum(np.floor(n / 2048), -1000))

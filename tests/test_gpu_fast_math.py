"""The hand-written math routines of the kernels, run on the device one argument per thread, against correctly rounded
references: 80-bit np.longdouble for the bulk samples and mpmath at 200 bits for the edges.

The device code is the product's own: libcmoe_probe.so (cornell-moe_b200/probe/fast_math_probe.cu) includes the
headers and calls exp_fast, exp_tab, exp_tab2k, exp_tab_cov, rff_sincos, sqrt_rsqrt and chol_pivot_fast after staging
their tables as the kernels do.  Each routine is tested over the argument contract written in its comment, with at least
10^6 arguments, and held to the error bound written there.  Worst measured errors are printed (pytest -s)."""
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
U = 2.0 ** -53  # unit roundoff
LN2 = float(mp.log(2))
NS = 1_000_000  # bulk samples per routine

EXP_FAST, EXP_TAB, EXP_TAB2K, EXP_TAB_COV, SINCOS, SQRT_RSQRT, PIVOT = range(7)
N_IN = {PIVOT: 2}
N_OUT = {SINCOS: 2, SQRT_RSQRT: 2, PIVOT: 3}
# documented max relative error over the accurate range (device_math.cuh, kg_mc.cuh)
EXPS = {"exp_fast": (EXP_FAST, 1.6e-16, True), "exp_tab": (EXP_TAB, 4.0e-16, False),
        "exp_tab2k": (EXP_TAB2K, 4.0e-16, False), "exp_tab_cov": (EXP_TAB_COV, 4.0e-16, True)}  # (id, bound, guarded)
FAST_PATH_RADIUS = 2000.0  # kFastPathRadius (kg_mc.cuh)
TAB_MIN = -2.3e7           # exp_tab / exp_tab2k: n = round(64 t / ln2) must fit 32 bits


@pytest.fixture(scope="module")
def probe():
    lib = ctypes.CDLL(PROBE)
    lib.cmoe_probe_eval.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int]
    lib.cmoe_probe_eval.restype = ctypes.c_int

    def run(routine, x):
        x = np.ascontiguousarray(x, dtype=np.float64)
        n = x.size // N_IN.get(routine, 1)
        out = np.empty(n * N_OUT.get(routine, 1))
        err = lib.cmoe_probe_eval(routine, x.ctypes.data, n, out.ctypes.data, 0)
        assert err == 0, f"cmoe_probe_eval({routine}) returned {err}"
        return out.reshape(n, -1) if routine in N_OUT else out
    return run


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)))


# ---------------------------------------------------------------------------------------------------------------------
# exps
# ---------------------------------------------------------------------------------------------------------------------
# Accurate range: every t whose exponent n >> (0, 6, 11) is not clamped, i.e. t >= -1000 ln2 for all four, up to 700
# (the SE q-KG arguments reach ln(alpha); exp(709.8) overflows).  Below -1000 ln2 the result is e^r 2^j 2^-1000 with
# |r| <= ln2/2: finite and in [0, 2^-999] (a zero contribution to every kernel sum).
ACC_LO, ACC_HI = -1000.0 * LN2, 700.0


def _exp_edges(guarded):
    ln2 = mp.log(2)
    e = [0.0, -0.0, 1.0, -1.0, 700.0, 699.999, 5e-324, -5e-324, 1e-300, -1e-300, 2.0 ** -30, -(2.0 ** -30),
         float(mp.log(2.0 ** 14)), float(-mp.log(2.0 ** 14))]
    for j in range(-1001, -998):  # both sides of the n = -1000 clamp (j ln2 is the boundary of exp_fast's n +- 1/2)
        for frac in (-0.5, 0.5, -1 / 128, 1 / 128, -1 / 4096, 1 / 4096):
            b = float((j + frac) * ln2)
            e += [b, np.nextafter(b, -np.inf), np.nextafter(b, np.inf)]
    for n in (1, 2, 63, 64, 65, 2047, 2048, 2049):  # table-index wrap points of the reduced exps
        for s in (-1, 1):
            b = float(s * (n + 0.5) * ln2 / 64)
            e += [b, np.nextafter(b, -np.inf), np.nextafter(b, np.inf)]
    if guarded:  # the -1024 input guard, down to -inf
        e += [-1024.0, np.nextafter(-1024.0, 0), np.nextafter(-1024.0, -np.inf), -1e4, -1e300, -np.finfo(float).max,
              -np.inf]
    else:  # the radius contract's -(2 kFastPathRadius)^2 / 2 and the 32-bit exponent limit
        b = -(2 * FAST_PATH_RADIUS) ** 2 / 2
        e += [b, np.nextafter(b, 0), np.nextafter(b, -np.inf), -7.3e5, -7.2e5, TAB_MIN, -1.8e7, -1024.0]
    return np.array(e, dtype=np.float64)


def _exp_samples(guarded, rng):
    acc = np.concatenate([rng.uniform(ACC_LO, ACC_HI, NS), rng.uniform(-1.0, 1.0, NS // 5),
                          rng.uniform(-1e-3, 1e-3, NS // 10), -np.exp(rng.uniform(np.log(1e-300), 0, NS // 10))])
    lo = -1e300 if guarded else TAB_MIN
    clamp = -np.exp(rng.uniform(np.log(-ACC_LO), np.log(-lo), NS // 5))
    if not guarded:  # the whole radius contract and beyond, uniformly
        clamp = np.concatenate([clamp, rng.uniform(-(2 * FAST_PATH_RADIUS) ** 2 / 2, ACC_LO, NS // 10),
                                rng.uniform(TAB_MIN, -(2 * FAST_PATH_RADIUS) ** 2 / 2, NS // 10)])
    return acc, clamp


@pytest.mark.parametrize("name", list(EXPS))
def test_exp_bulk_accuracy_and_clamp(probe, name):
    routine, bound, guarded = EXPS[name]
    acc, clamp = _exp_samples(guarded, np.random.default_rng(11 + routine))
    got = probe(routine, acc)
    ref = np.exp(acc.astype(LD))
    rel = np.abs((got.astype(LD) - ref) / ref)
    worst = float(rel.max())
    print(f"\n{name}: max relative error {worst:.3e} ({worst / U:.2f} u) over {acc.size} arguments in "
          f"[{ACC_LO:.3f}, {ACC_HI}] (documented {bound:.1e})")
    assert worst <= bound, (name, worst, float(acc[np.argmax(rel)]))
    low = probe(routine, clamp)
    assert np.all(np.isfinite(low)) and np.all(low >= 0.0) and np.all(low <= 2.0 ** -999), name


@pytest.mark.parametrize("name", list(EXPS))
def test_exp_edges(probe, name):
    routine, bound, guarded = EXPS[name]
    t = _exp_edges(guarded)
    got = probe(routine, t)
    assert probe(routine, np.array([0.0, -0.0])).tolist() == [1.0, 1.0], name
    mp.mp.prec = 200
    worst = 0.0
    for ti, gi in zip(t, got):
        if ti >= ACC_LO:
            ref = mp.exp(mp.mpf(float(ti)))
            rel = float(abs((mp.mpf(float(gi)) - ref) / ref))
            worst = max(worst, rel)
            assert rel <= bound, (name, float(ti), float(gi), rel)
        else:
            assert np.isfinite(gi) and 0.0 <= gi <= 2.0 ** -999, (name, float(ti), float(gi))
    print(f"\n{name}: max relative error {worst:.3e} at {t.size} edge arguments (200-bit reference)")


# ---------------------------------------------------------------------------------------------------------------------
# rff_sincos
# ---------------------------------------------------------------------------------------------------------------------
SINCOS_ULPS = 2.0  # device_math.cuh: error of sin and cos, in ulps of the correctly rounded result, for |a| < 2^30


def _near_multiples_of_half_pi(rng):
    """Doubles nearest k pi/2 in every binade of [1, 2^30): the closest approaches (denominators of the continued
    fraction convergents of (pi/2) 2^(52-e) and their multiples in the binade's k range) plus random k."""
    mp.mp.prec = 200
    half_pi = mp.pi / 2
    out = []
    for e in range(0, 30):
        beta = half_pi * mp.mpf(2) ** (52 - e)  # a = m 2^(e-52), m in [2^52, 2^53): m ~ k beta
        klo = int(mp.ceil(mp.mpf(2) ** e / half_pi))
        khi = int(mp.floor(mp.mpf(2) ** (e + 1) / half_pi))
        ks = set(int(k) for k in rng.integers(max(klo, 1), khi + 1, 8))
        x, p0, q0, p1, q1 = beta, 0, 1, 1, 0
        for _ in range(60):  # convergents p/q of beta
            a_i = int(mp.floor(x))
            p0, q0, p1, q1 = p1, q1, a_i * p1 + p0, a_i * q1 + q0
            if q1 > khi:
                break
            if q1 > 0:
                j0 = max(1, -(-klo // q1))
                for j in range(j0, j0 + 12):
                    if j * q1 <= khi:
                        ks.add(j * q1)
            frac = x - a_i
            if frac == 0:
                break
            x = 1 / frac
        for k in ks:
            if k < 1:
                continue
            m = int(mp.nint(k * beta))
            for mm in (m - 1, m, m + 1):
                a = float(Fraction(mm) * Fraction(2) ** (e - 52))
                if abs(a) < 2.0 ** 30:
                    out += [a, -a]
    return np.array(out)


def _sincos_ulps(a, got, ref_s, ref_c):
    es = np.abs(got[:, 0].astype(LD) - ref_s) / ulp(ref_s.astype(np.float64))
    ec = np.abs(got[:, 1].astype(LD) - ref_c) / ulp(ref_c.astype(np.float64))
    return es, ec


def test_rff_sincos_bulk(probe):
    rng = np.random.default_rng(5)
    a = np.concatenate([rng.uniform(-2.0 ** 30, 2.0 ** 30, NS // 2),
                        rng.choice([-1, 1], NS // 2) * np.exp(rng.uniform(np.log(1e-8), np.log(2.0 ** 30), NS // 2)),
                        rng.uniform(-8.0, 8.0, NS // 5), [0.0, -0.0, np.nextafter(2.0 ** 30, 0)]])
    got = probe(SINCOS, a)
    al = a.astype(LD)
    es, ec = _sincos_ulps(a, got, np.sin(al), np.cos(al))
    print(f"\nrff_sincos: max error sin {float(es.max()):.3f} ulp, cos {float(ec.max()):.3f} ulp over {a.size} "
          f"arguments, |a| < 2^30 (documented {SINCOS_ULPS})")
    assert float(es.max()) <= SINCOS_ULPS, float(a[np.argmax(es)])
    assert float(ec.max()) <= SINCOS_ULPS, float(a[np.argmax(ec)])
    assert got[-3, 0] == 0.0 and got[-2, 0] == 0.0 and got[-3, 1] == 1.0 and got[-2, 1] == 1.0


def test_rff_sincos_near_multiples_of_half_pi(probe):
    a = _near_multiples_of_half_pi(np.random.default_rng(6))
    got = probe(SINCOS, a)
    mp.mp.prec = 200
    worst = 0.0
    for ai, (s, c) in zip(a, got):
        x = mp.mpf(float(ai))
        for g, r in ((s, mp.sin(x)), (c, mp.cos(x))):
            err = float(abs(mp.mpf(float(g)) - r)) / float(np.spacing(abs(float(r))))
            worst = max(worst, err)
            assert err <= SINCOS_ULPS, (float(ai), float(g), float(r), err)
    print(f"\nrff_sincos: max error {worst:.3f} ulp at {a.size} doubles nearest k pi/2 (200-bit reference)")


# ---------------------------------------------------------------------------------------------------------------------
# square roots
# ---------------------------------------------------------------------------------------------------------------------
SQRT_ULPS, RSQRT_ULPS = 2.0, 2.5  # device_math.cuh: sqrt_rsqrt's l and y, in ulps of the exact sqrt(p), 1/sqrt(p)


def test_sqrt_rsqrt(probe):
    rng = np.random.default_rng(7)
    m = rng.integers(1, 2 ** 26, 20000).astype(np.float64) * 2.0 ** rng.integers(-60, 60, 20000)
    p = np.concatenate([np.exp(rng.uniform(np.log(1e-16), np.log(1e16), NS)),       # Cholesky pivots
                        np.exp(rng.uniform(np.log(1e-280), np.log(1e300), NS // 2)),  # Matern r^2
                        rng.uniform(1.0, 4.0, NS // 5), m * m, [1e-280, 1e-16, 1.0, 4.0, 2.0]])
    got = probe(SQRT_RSQRT, p)
    sl = np.sqrt(p.astype(LD))
    el = np.abs(got[:, 0].astype(LD) - sl) / ulp(sl.astype(np.float64))
    ey = np.abs(got[:, 1].astype(LD) - 1 / sl) / ulp((1 / sl).astype(np.float64))
    print(f"\nsqrt_rsqrt: max error l {float(el.max()):.3f} ulp, y {float(ey.max()):.3f} ulp over {p.size} arguments in "
          f"[1e-280, 1e300]; l != sqrt_rn(p) for {np.mean(got[:, 0] != np.sqrt(p)):.2e} of them")
    assert float(el.max()) <= SQRT_ULPS, float(p[np.argmax(el)])
    assert float(ey.max()) <= RSQRT_ULPS, float(p[np.argmax(ey)])


# ---------------------------------------------------------------------------------------------------------------------
# FAST pivot of chol32_warp<true>
# ---------------------------------------------------------------------------------------------------------------------
# Error of the correction steps (u = 2^-53; library rsqrt y = (1 + e_y)/sqrt(p), |e_y| <= 2u (1 ulp)):
#   l0 = rn(p y) = sqrt(p)(1 + e0), |e0| <= 3u;  l0 + (y/2) rn(p - l0^2) = sqrt(p)(1 - e0^2/2 - (e_y + e2) e0 + ...)
#     -> the value rounded into l is sqrt(p)(1 + eta), |eta| <= 4.5u^2 + 9u^2 = 13.5u^2;
#   q0 = rn(a y) = (a/l)(1 + e3), |e3| <= 4u (y, the product, and l's own rounding against sqrt(p));
#   q0 + y rn(a - q0 l) = (a/l)(1 - (e_l + e_y + e4) e3 + ...) -> |eta| <= 16u^2.
# So l (q) can differ from sqrt_rn(p) (rn(a/l)) only when the exact value lies within DELTA relative of a rounding
# midpoint; DELTA keeps a factor 2 over both bounds for the second-order terms.
DELTA = 32 * U * U
RECIP_ULPS = 0.55  # linalg_dev.cuh: chol_pivot_recip, in ulps of the exact 1/l of the returned l


def _near_midpoint(exact, got, ref):
    """exact (mpf) lies within DELTA relative of the midpoint between the two doubles got and ref (adjacent)."""
    mid = (mp.mpf(float(got)) + mp.mpf(float(ref))) / 2
    return np.nextafter(got, ref) == ref and abs(exact - mid) <= DELTA * abs(exact)


def test_pivot_fast_exact_cases(probe):
    rng = np.random.default_rng(8)
    m = rng.integers(1, 2 ** 26, NS // 4).astype(np.float64) * 2.0 ** rng.integers(-26, 26, NS // 4)
    k = rng.integers(-2 ** 26, 2 ** 26, NS // 4).astype(np.float64) * 2.0 ** rng.integers(-20, 20, NS // 4)
    p = m * m  # exact: m has <= 26 significant bits
    a = k * m  # exact: both have <= 26 significant bits
    got = probe(PIVOT, np.stack([p, a], axis=1))
    assert np.array_equal(got[:, 0], m), "l != sqrt(p) for p = m^2"
    assert np.array_equal(got[:, 1], k), "q != a / l for a = k l"


def test_pivot_fast_bulk(probe):
    rng = np.random.default_rng(9)
    p = np.exp(rng.uniform(np.log(2e-16), np.log(1e8), NS))  # pivots > kPivotTol
    a = np.sqrt(p) * rng.choice([-1, 1], NS) * np.exp(rng.uniform(np.log(1e-12), np.log(1e4), NS))
    a[: NS // 10] = 0.0
    got = probe(PIVOT, np.stack([p, a], axis=1))
    l, q, r = got[:, 0], got[:, 1], got[:, 2]
    l_rn, q_rn = np.sqrt(p), a / l  # numpy's sqrt and divide are correctly rounded
    mp.mp.prec = 200
    bad_l, bad_q = np.flatnonzero(l != l_rn), np.flatnonzero(q != q_rn)
    for i in bad_l:
        assert _near_midpoint(mp.sqrt(mp.mpf(float(p[i]))), l[i], l_rn[i]), (float(p[i]), l[i], l_rn[i])
    for i in bad_q:
        assert _near_midpoint(mp.mpf(float(a[i])) / mp.mpf(float(l[i])), q[i], q_rn[i]), (float(a[i]), q[i], q_rn[i])
    er = np.abs(r.astype(LD) - 1 / l.astype(LD)) / ulp(1 / l)
    print(f"\nchol_pivot_fast: {bad_l.size} of {NS} l and {bad_q.size} q differ from the IEEE results (all near a "
          f"midpoint); 1/l max error {float(er.max()):.3f} ulp")
    assert float(er.max()) <= RECIP_ULPS, float(p[np.argmax(er)])

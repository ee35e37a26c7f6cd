"""Host restatement of the kernel-matched random features (cmoe_rff_opts, DESIGN.md K14 addendum) and of the sample
functions' evaluation (cmoe_rff_evaluate), for the CPU and GPU tests of tests/test_rff_paths_cpu.py and
tests/test_gpu_rff_paths.py.

* ``chi2_draws``: g ~ chi^2_5 of the Matern-5/2 draw from the Philox stream with counter word 3 = 3, operation for
  operation as rff_chi2_at (the logarithm and cosine are NumPy's, so it agrees with the device to a few ulps).
* ``matern_frequencies``: W = (Omega / l) sqrt(5 / g).
* ``correlation_z``: the z-scores of the empirical E[cos(W . delta)] against a kernel's correlation at given offsets.
"""
import numpy as np

from sampling_ref import philox4x32_10

_MASK = np.uint64(0xFFFFFFFF)


def _u53(hi, lo):
    w = (hi << np.uint64(32)) | lo
    return ((w >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0 ** -53


def chi2_draws(seed, draw, F):
    """g[F] of Philox draw `draw`: -2 ln u0 - 2 ln u1 + (-2 ln u2) cos^2(2 pi v2), (u0, u1) from the call (draw, 2f) and
    (u2, v2) from (draw, 2f + 1), counter word 3 = 3."""
    seed, draw = int(seed), int(draw)
    f = np.arange(F, dtype=np.uint64)
    lo, hi = np.full(F, draw & 0xFFFFFFFF, dtype=np.uint64), np.full(F, draw >> 32, dtype=np.uint64)
    three = np.full(F, 3, dtype=np.uint64)
    a = philox4x32_10(lo, hi, 2 * f, three, seed & 0xFFFFFFFF, seed >> 32)
    e = philox4x32_10(lo, hi, 2 * f + np.uint64(1), three, seed & 0xFFFFFFFF, seed >> 32)
    u0, u1 = _u53(a[0], a[1]), _u53(a[2], a[3])
    u2, v2 = _u53(e[0], e[1]), _u53(e[2], e[3])
    cs = np.cos(2.0 * np.pi * v2)
    t = -2.0 * np.log(u2)
    return (-2.0 * np.log(u0) + -2.0 * np.log(u1)) + (t * cs) * cs


def matern_frequencies(omega, lengths, g):
    """omega [..., F, d] standard normals, g [..., F]: the Matern-5/2 frequencies, rounded as the device rounds them."""
    return (omega / lengths) * np.sqrt(5.0 / g)[..., None]


def matern52_corr(delta, lengths):
    r = np.sqrt(np.sum((np.asarray(delta) / lengths) ** 2, axis=-1))
    s = np.sqrt(5.0) * r
    return (1.0 + s + s * s / 3.0) * np.exp(-s)


def se_corr(delta, lengths):
    r2 = np.sum((np.asarray(delta) / lengths) ** 2, axis=-1)
    return np.exp(-0.5 * r2)


def correlation_z(W, deltas, target):
    """z-scores of mean_f cos(W_f . delta) against target(delta) at every row of deltas; W [n, d]."""
    W = np.asarray(W).reshape(-1, np.asarray(deltas).shape[1])
    z = []
    for delta in deltas:
        c = np.cos(W @ delta)
        se = c.std() / np.sqrt(c.size)
        z.append((c.mean() - target(delta)) / se)
    return np.array(z)


# offsets in units of the length scales: r from 0.25 to 2.5, along different directions
def offsets(lengths, rng=None):
    rng = np.random.default_rng(0) if rng is None else rng
    d = len(lengths)
    out = []
    for r in (0.25, 0.5, 0.8, 1.2, 1.7, 2.5):
        u = rng.normal(size=d)
        out.append(r * u / np.linalg.norm(u) * np.asarray(lengths))
    return np.array(out)


def f_values(x, W, b, th, c):
    """f at points x [X, d] of one sample function (the reference wrapper's gradient=False branch)."""
    return c * np.cos(np.atleast_2d(x) @ W.T + b) @ th


def f_grads(x, W, b, th, c):
    """grad f at points x [X, d]: -c sum_f theta_f sin(W_f x + b_f) W_f."""
    S = np.sin(np.atleast_2d(x) @ W.T + b) * th
    return -c * S @ W

"""Host restatement of the joint-sampling path (cmoe_gp_sample_joint, cmoe_latin_hypercube) for the parity tests.

* ``philox_uniform_keys`` / ``latin_hypercube``: the device's Latin hypercube, operation for operation (Philox4x32-10
  with the fourth counter word 1, strata ranked by key with ties broken by index, x = min + edge rank + edge u clamped
  to max; no fused multiply-adds), so the device output must match it bit for bit.
* ``sample_from_posterior``: SamplePointsFromGP / SamplePointFromGP (gpp_math.cpp:1761-1848) given the posterior mean,
  the Cholesky factor of the posterior covariance and the normals: y = mean + L w, and the reference's argmin, which
  starts at -1 with a strict `<` (so a minimum at point 0 gives -1).
"""
import numpy as np

_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised Philox4x32-10 on uint64 arrays holding 32-bit words (the round function of device_math.cuh)."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _MASK for c in (c0, c1, c2, c3))
    k0, k1 = np.uint64(k0) & _MASK, np.uint64(k1) & _MASK
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & _MASK, p1 & _MASK, \
            ((p0 >> np.uint64(32)) ^ c3 ^ k1) & _MASK, p0 & _MASK
        k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK
        k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK
    return c0, c1, c2, c3


def philox_uniform_keys(seed, draw, ks):
    """(53-bit integer key, uniform offset in (0, 1)) of Philox calls ks of `draw`, counter word 3 = 1."""
    ks = np.asarray(ks, dtype=np.uint64)
    seed, draw = int(seed), int(draw)
    c0, c1, c2, c3 = philox4x32_10(np.full(ks.shape, draw & 0xFFFFFFFF, dtype=np.uint64),
                                   np.full(ks.shape, draw >> 32, dtype=np.uint64), ks,
                                   np.ones(ks.shape, dtype=np.uint64), seed & 0xFFFFFFFF, seed >> 32)
    key = ((c0 << np.uint64(32)) | c1) >> np.uint64(11)
    b = ((c2 << np.uint64(32)) | c3) >> np.uint64(11)
    u = (b.astype(np.float64) + 0.5) * 2.0 ** -53
    return key, u


def latin_hypercube(seed, draw, num_pts, bounds):
    """One set: [num_pts, dim] points of the Latin hypercube of (seed, draw) in bounds [dim, 2]."""
    bounds = np.asarray(bounds, dtype=np.float64).reshape(-1, 2)
    dim = bounds.shape[0]
    out = np.empty((num_pts, dim))
    j = np.arange(num_pts)
    for i in range(dim):
        key, u = philox_uniform_keys(seed, draw, i * num_pts + j)
        rank = np.empty(num_pts, dtype=np.int64)
        rank[np.lexsort((j, key))] = j
        lo, hi = bounds[i]
        edge = (hi - lo) / float(num_pts)
        x = lo + edge * rank.astype(np.float64)
        out[:, i] = np.minimum(x + edge * u, hi)
    return out


def sample_from_posterior(mean, chol, normals, rows_per_point=1):
    """(samples, reference argmin (-1 when point 0 is the minimum), true argmin) for one set."""
    L = np.tril(np.asarray(chol, dtype=np.float64))
    y = np.asarray(mean, dtype=np.float64) + L @ np.asarray(normals, dtype=np.float64)
    values = y[::rows_per_point]
    best_point, best = -1, values[0]
    for i, v in enumerate(values):
        if v < best:
            best_point, best = i, v
    return y, best_point, int(np.argmin(values))

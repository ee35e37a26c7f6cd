"""Host restatement of cmoe_posterior_mean_optima_mcmc for the parity tests, on top of a CPU checker's per-member GPs
(``mean_additional`` and ``posterior_mean_optimization`` of oracle.CpuGP).

For every member on its own (examples/main.py:172-197 of the reference, then KnowledgeGradientMCMC's best_so_far,
cpp_wrappers/knowledge_gradient_mcmc.py:386-393):
  1. screen: mu_m at the given points (shared [P, ps] or per member [M, P, ps]) and, if include_sampled, at the first
     ps coordinates of the member's sampled points, which follow the given points; fidelity coordinates are 1.0
  2. argmin, first occurrence
  3. ComputeOptimalPosteriorMean from that start (nothing moves with max_num_restarts <= 0)
  4. the start is kept if mu_m at the end point is greater than the screened minimum
  5. discrete_pts[m] = [shared ; optimum_m], best_so_far[m] = least mu_m over it
"""
import collections

import numpy as np

Optima = collections.namedtuple("Optima", "optima means start_index kept_start screen_min discrete_pts best_so_far")


def _full(pts, dim):
    out = np.ones((pts.shape[0], dim))
    out[:, :pts.shape[1]] = pts
    return out


def member_optimum(gp, sampled, pts, gd, bounds, num_fidelity, include_sampled, shared):
    """One member: (optimum, mu there, start index, kept, screened minimum, discrete points, best_so_far).
    gd is the 8-sequence of GDParams; sampled [N, dim] are the member's sampled points."""
    ps = gp.dim - num_fidelity
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, ps)
    if include_sampled:
        pts = np.concatenate([pts, np.asarray(sampled, dtype=np.float64)[:, :ps]])
    mu = gp.mean_additional(_full(pts, gp.dim))
    i0 = int(np.argmin(mu))
    x0 = pts[i0].copy()
    kept, point, value = True, x0, mu[i0]
    if gd[2] > 0:
        end, f_end = gp.posterior_mean_optimization(x0, gd, bounds, num_fidelity)
        kept = bool(-f_end > mu[i0])
        if not kept:
            point, value = end, -f_end
    disc = np.concatenate([np.asarray(shared, dtype=np.float64).reshape(-1, ps), point[None]])
    best = float(gp.mean_additional(_full(disc, gp.dim)).min())
    return point, float(value), i0, kept, float(mu[i0]), disc, best


def optima(gps, sampled, points, gd, bounds, num_fidelity=0, include_sampled=True, shared=None):
    """gps: the members' CpuGPs; sampled: one [N_m, dim] array per member (or one array for all)."""
    M = len(gps)
    ps = gps[0].dim - num_fidelity
    points = np.asarray(points, dtype=np.float64)
    shared = np.zeros((0, ps)) if shared is None else shared
    if isinstance(sampled, np.ndarray):
        sampled = [sampled] * M
    rows = [member_optimum(gp, sampled[m], points[m] if points.ndim == 3 else points, gd, bounds, num_fidelity,
                           include_sampled, shared) for m, gp in enumerate(gps)]
    cols = list(zip(*rows))
    return Optima(np.array(cols[0]), np.array(cols[1]), np.array(cols[2]), np.array(cols[3], dtype=int),
                  np.array(cols[4]), np.array(cols[5]), np.array(cols[6]))

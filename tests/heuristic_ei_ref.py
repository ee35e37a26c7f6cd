"""NumPy restatement of the GP that heuristic EI (cmoe_heuristic_ei, DESIGN.md K20) builds round by round: the training
rows with the GP's noise, then each chosen point with the policy's own noise on its diagonal, refitted from scratch
(Cholesky of K + diag(noise), prior mean = average of the values, K^-1 (y - mean)).  At each round's chosen point it
gives the posterior mean, the f-variance and the closed-form 1-EI of the GP extended by the earlier rounds."""
import math

import numpy as np

SQUARE_EXPONENTIAL, MATERN_NU_2P5 = 0, 1


def covariance(kernel, alpha, lengths, A, B):
    A = np.atleast_2d(A) / lengths
    B = np.atleast_2d(B) / lengths
    r2 = np.maximum(((A[:, None, :] - B[None, :, :]) ** 2).sum(axis=2), 0.0)
    if kernel == SQUARE_EXPONENTIAL:
        return alpha * np.exp(-0.5 * r2)
    r = np.sqrt(5.0 * r2)
    return alpha * (1.0 + r + 5.0 / 3.0 * r2) * np.exp(-r)


def posterior(kernel, alpha, lengths, X, y, row_noise, x):
    """mu(x) and k(x,x) - k^T K^-1 k for the GP on rows X, values y with per-row noise."""
    K = covariance(kernel, alpha, lengths, X, X) + np.diag(row_noise)
    L = np.linalg.cholesky(K)
    mean = y.mean()
    beta = np.linalg.solve(L.T, np.linalg.solve(L, y - mean))
    k = covariance(kernel, alpha, lengths, X, x)[:, 0]
    v = np.linalg.solve(L, k)
    return mean + k @ beta, alpha - v @ v


def one_point_ei(best, mu, var):
    sigma = math.sqrt(max(np.finfo(float).tiny, var))
    t = best - mu
    z = t / sigma
    return max(0.0, t * 0.5 * math.erfc(-z / math.sqrt(2.0)) + sigma * math.exp(-0.5 * z * z) / math.sqrt(2 * math.pi))


def rounds(kernel, alpha, lengths, X, y, gp_noise, points, fantasy_values, policy_noise, best):
    """(mu, var, ei) at points[r] on the GP extended by points[:r] with fantasy_values[:r] (noise policy_noise)."""
    out = []
    for r, x in enumerate(points):
        Xr = np.vstack([X, points[:r]])
        yr = np.concatenate([y, fantasy_values[:r]])
        nz = np.concatenate([np.full(len(X), gp_noise), np.full(r, policy_noise)])
        mu, var = posterior(kernel, alpha, lengths, Xr, yr, nz, x[None])
        out.append((mu, var, one_point_ei(best, mu, var)))
    return out

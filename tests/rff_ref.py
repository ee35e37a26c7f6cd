"""NumPy restatement of the random-feature sampler's contract (cmoe_gp_sample_rff_optima, DESIGN.md K14), including the
pathwise M < F branch, and access to the golden fixture tests/golden/reference_rff.npz."""
import os

import numpy as np
import scipy.linalg as spla

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_rff.npz")


def golden_cases():
    z = np.load(GOLDEN)
    out = []
    for name in z["names"]:
        p = f"{name}/"
        out.append((str(name), {k[len(p):]: z[k] for k in z.files if k.startswith(p)}))
    return out


def design(X, Y, noise, derivs, alpha, lengths, omega, b):
    """(Phi [F, M], y' [M], W [F, d], c): value columns first, then one block per derivative type."""
    F = omega.shape[0]
    W = omega / lengths
    c = np.sqrt(2.0 * alpha / F)
    A = W @ X.T + b[:, None]
    cols = [c * np.cos(A) / np.sqrt(noise[0])]
    for k, j in enumerate(derivs):
        cols.append(-c * W[:, [j]] * np.sin(A) / np.sqrt(noise[k + 1]))
    Phi = np.concatenate(cols, axis=1)
    yp = (Y / np.sqrt(noise)).flatten("F")
    return Phi, yp, W, c


def theta(Phi, yp, z, eps=None):
    """The header's two branches: M < F pathwise (eps [M] needed), M >= F through the reversed Cholesky factor."""
    F, M = Phi.shape
    if M < F:
        L = np.linalg.cholesky(np.eye(M) + Phi.T @ Phi)
        r = Phi @ yp + z
        v = spla.cho_solve((L, True), Phi.T @ r + eps)
        return r - Phi @ v
    J = np.arange(F)[::-1]
    B = np.eye(F) + Phi @ Phi.T
    L = np.linalg.cholesky(B[np.ix_(J, J)])
    q = (Phi @ yp)[J]
    w = spla.solve_triangular(L, q, lower=True) + z[J]
    return spla.solve_triangular(L.T, w, lower=False)[J]


def posterior_cov(Phi):
    F = Phi.shape[0]
    return np.linalg.inv(np.eye(F) + Phi @ Phi.T)


def pathwise_cov(Phi):
    """Covariance of the M < F draw z - Phi A^-1 (Phi^T z + eps): (I - Phi A^-1 Phi^T)^2 + Phi A^-2 Phi^T."""
    F, M = Phi.shape
    A = np.eye(M) + Phi.T @ Phi
    G = Phi @ np.linalg.solve(A, np.eye(M))
    P = np.eye(F) - G @ Phi.T
    return P @ P.T + G @ G.T


def f_value(x, W, b, th, c):
    return c * np.cos(np.atleast_2d(x) @ W.T + b) @ th


def f_grad(x, W, b, th, c):
    return -c * (th * np.sin(W @ x + b)) @ W


def kkt_residual(x, g, lo, hi):
    return np.max(np.abs(x - np.clip(x - g, lo, hi)))

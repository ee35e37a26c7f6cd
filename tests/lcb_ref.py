"""CPU restatements of the reference's LCB batch selection (lower_confidence_bound.py:52-80).

``reference_loop`` makes the reference routine's calls on a CPU GP (the compiled reference or the C oracle): the value
mean, the [0,0] entry of the Cholesky variance of every one-point set (carrying the GP's derivative rows), and a refit
with the previous point appended (zero values, the GP's noise) before each further round.

``bordered`` restates the device algorithm (DESIGN.md K13) in NumPy, fed the backend's kernel blocks: no refit, one
block row of the bordered factor of M = Sigma0(S, S) + D per round, and w_j(x) = L_jj^-1 (c0(s_j, x) - R_j w_<j(x)).
"""
import os

import numpy as np


class LcbSingular(Exception):
    def __init__(self, info, cand=None):
        super().__init__(f"singular: info={info} candidate={cand}")
        self.info = info
        self.cand = cand


def _margin_min(values, best, coords, winner):
    """Relative gap between the winning value and the best value at other coordinates (inf if there is none)."""
    others = np.array([v for v, c in zip(values, coords) if not np.array_equal(c, coords[winner])])
    if others.size == 0:
        return np.inf
    return np.min(np.abs(others - best)) / max(abs(best), 1e-300)


def reference_loop(backend, kernel, alpha, lengths, X, y, noise, derivs, cand, q):
    X = np.array(X, dtype=np.float64)
    cand = np.array(cand, dtype=np.float64)
    derivs = np.asarray(derivs if derivs is not None else [], dtype=np.int32)
    b = 1 + len(derivs)
    y = np.asarray(y, dtype=np.float64).ravel()

    def fit(Xf, yf):
        gp, lm = backend.gp(kernel, alpha, lengths, Xf, yf, noise, derivs)
        if gp is None:
            raise LcbSingular(lm)
        return gp

    def sigmas(gp, pts, idx):
        out = np.empty(len(idx))
        for k, i in enumerate(idx):
            r = gp.posterior(pts[i], derivs, want=("chol_var",))
            if r["rc"] != 0 or not r["chol_var"][0] > 0.0:
                raise LcbSingular(1, int(i))
            out[k] = r["chol_var"][0]
        return out

    gp = fit(X, y)
    mean = gp.posterior(cand, None, want=("mean",))["mean"].copy()
    sd = sigmas(gp, cand, range(len(cand)))
    target, ucb = mean - sd, mean + sd
    first = int(np.argmin(target))
    upper = np.min(ucb)
    sat = np.nonzero(target <= upper)[0]
    margins = [_margin_min(target, target[first], cand, first)]
    inside = np.abs(target - upper) / max(abs(upper), 1e-300)
    margins.append(float(np.min(inside)))
    selected = [first]
    rounds = []
    Xa, ya = X, y
    for _ in range(1, q):
        Xa = np.vstack([Xa, cand[selected[-1]][None]])
        ya = np.concatenate([ya, np.zeros(b)])
        gp = fit(Xa, ya)
        s = sigmas(gp, cand, sat)
        rounds.append(s)
        j = int(np.argmax(s))
        margins.append(_margin_min(s, s[j], cand[sat], j))
        selected.append(int(sat[j]))
    return dict(selected=np.array(selected), mean=mean, sd=sd, sat=sat, rounds=rounds, margins=np.array(margins),
                num_sampled=Xa.shape[0])


def bordered(backend, kernel, alpha, lengths, X, y, noise, derivs, cand, q):
    """The bordered update; same return keys as reference_loop (margins omitted)."""
    X = np.array(X, dtype=np.float64)
    cand = np.array(cand, dtype=np.float64)
    derivs = np.asarray(derivs if derivs is not None else [], dtype=np.int32)
    b = 1 + len(derivs)
    N = X.shape[0]
    noise = np.asarray(noise, dtype=np.float64).ravel()
    y = np.asarray(y, dtype=np.float64).ravel()

    def block(p1, d1, p2, d2):
        return backend.covariance(kernel, alpha, lengths, p1, d1, p2, d2).reshape(1 + len(d2), 1 + len(d1)).T

    def rows_vs_data(p, d):  # K(p rows, X rows): (1+len(d)) x n
        return np.hstack([block(p, d, X[j], derivs) for j in range(N)])

    K = np.vstack([rows_vs_data(X[i], derivs) for i in range(N)]) + np.diag(np.tile(noise, N))
    L = np.linalg.cholesky(K)
    yc = y.copy()
    mu0 = np.mean(y[::b])
    yc[::b] -= mu0
    beta = np.linalg.solve(K, yc)
    kx = np.vstack([rows_vs_data(c, []) for c in cand])  # C x n
    mean = mu0 + kx @ beta
    V = np.linalg.solve(L, kx.T)
    s2 = np.array([block(c, [], c, [])[0, 0] for c in cand]) - np.sum(V * V, axis=0)
    for i, v in enumerate(s2):
        if not v > 1e-16:
            raise LcbSingular(1, i)
    sd = np.sqrt(s2)
    target, ucb = mean - sd, mean + sd
    first = int(np.argmin(target))
    sat = np.nonzero(target <= np.min(ucb))[0]
    selected, rounds = [first], []
    s2 = s2[sat]
    Ws = np.zeros((len(sat), 0))
    LM = np.zeros((0, 0))
    Ts, pts = [], []
    n0 = N * b
    for _ in range(1, q):
        s = cand[selected[-1]]
        pts.append(s)
        Ksx = rows_vs_data(s, derivs)  # b x n
        T = np.linalg.solve(L, Ksx.T)  # n x b
        Bk = np.linalg.solve(K, Ksx.T)
        Ts.append(T)
        Kp = np.hstack([block(s, derivs, p, derivs) for p in pts])  # b x (k+1) b, prior
        Kp[:, -b:] += np.diag(noise)
        Mrow = Kp - T.T @ np.hstack(Ts)
        kb = LM.shape[0]
        R = np.linalg.solve(LM, Mrow[:, :kb].T).T if kb else np.zeros((b, 0))
        S = Mrow[:, kb:] - R @ R.T
        Lkk = np.zeros((b, b))
        for jj in range(b):  # unblocked Cholesky with the reference's pivot test
            d = S[jj, jj] - Lkk[jj, :jj] @ Lkk[jj, :jj]
            if not d > 1e-16:
                raise LcbSingular(n0 + kb + jj + 1)
            Lkk[jj, jj] = np.sqrt(d)
            for ii in range(jj + 1, b):
                Lkk[ii, jj] = (S[ii, jj] - Lkk[ii, :jj] @ Lkk[jj, :jj]) / Lkk[jj, jj]
        LM = np.block([[LM, np.zeros((kb, b))], [R, Lkk]])
        c0 = np.array([block(s, derivs, cand[i], [])[:, 0] for i in sat]) - kx[sat] @ Bk  # C' x b
        w = np.linalg.solve(Lkk, (c0 - Ws @ R.T).T).T
        Ws = np.hstack([Ws, w])
        s2 = s2 - np.sum(w * w, axis=1)
        for k, v in enumerate(s2):
            if not v > 1e-16:
                raise LcbSingular(1, int(sat[k]))
        sig = np.sqrt(s2)
        rounds.append(sig)
        selected.append(int(sat[int(np.argmax(sig))]))
    return dict(selected=np.array(selected), mean=mean, sd=sd, sat=sat, rounds=rounds)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_lcb.npz")


def golden_cases():
    """(name, {field: array}) for every case of the reference run stored by tests/golden/make_lcb_golden.py."""
    z = np.load(GOLDEN)
    return [(str(name), {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(f"{name}/")}) for name in z["names"]]


def pivot_failure_problem():
    """Gradient observations with zero noise: at a training point the posterior derivative variance is zero (up to
    rounding far below 1e-16 at alpha = 1e-6), while the value variance keeps its noise.  Selecting that point makes the
    first derivative row of the enlarged matrix fail its pivot: info = n + 2."""
    from synth import make_problem
    pr = make_problem(8, 2, (0, 1), seed=21, noise=0.0, alpha=1e-6, length=0.3)
    pr["noise"] = np.array([1e-8, 0.0, 0.0])
    return pr, pr["X"][2:3].copy()

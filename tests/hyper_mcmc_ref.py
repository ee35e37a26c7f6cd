"""NumPy restatement of the hyper-parameter MCMC of the reference's GaussianProcessLogLikelihoodMCMC.train
(moe/optimal_learning/python/cpp_wrappers/log_likelihood_mcmc.py:170-239): emcee 2.2.1's EnsembleSampler.sample with the
stretch move (a = 2), the target density compute_log_likelihood (:277-312) and DefaultPrior
(moe/optimal_learning/python/default_priors.py:27-37).  emcee is neither installed nor in the reference tree, so its
loop is restated from the 2.2.1 release (ensemble.py: sample, _propose_stretch, _get_lnprob).

The likelihood is a callable `lml(H)` on linear-scale sets [alpha, lengths..., noise...] (rows of H), e.g.
cmoe_log_marginal_likelihood_list, or `numpy_lml_matern52` below for runs without a device."""
import numpy as np
from scipy import stats

STRETCH_A = 2.0
LOG_NOISE_FREE = float(np.log(np.array([1.0e-8]))[0])  # numpy.log((1 + g) * [1.e-8]), log_likelihood_mcmc.py:289


def default_prior_lnprob(theta, num_noise):
    """DefaultPrior(n_dims, num_noise).lnprob (default_priors.py:27-37), term by term in its order."""
    lp = 0
    lp += stats.norm.pdf(theta[0], scale=1.0, loc=0.0)  # NormalPrior.lnprob returns the pdf (base_prior.py:338-354)
    lengths = theta[1:-num_noise]
    lp += -np.inf if (np.any(lengths < -2) or np.any(lengths > 3)) else 0  # TophatPrior(-2, 3) (:104-123)
    for i in range(num_noise, 0, -1):  # HorseshoePrior(0.1) (:183-201)
        t = theta[-i]
        lp += np.inf if t == 0.0 else np.log(np.log(1 + 3.0 * (0.1 / t) ** 2))
    return lp


def log_prob(P, lml, dim, g, noisy, default_prior):
    """compute_log_likelihood (log_likelihood_mcmc.py:277-312) on every row of P.  Rows are modified in place, as the
    row views emcee 2.2.1's _get_lnprob hands to the function are: with noisy False the noise entries of every row in
    the box become log(1e-8).  The likelihoods of the rows that need one come from one lml() call."""
    out = np.full(len(P), -np.inf)
    need, priors = [], []
    for i, h in enumerate(P):
        if np.any((-20 > h) + (h > 20)):
            continue
        if not noisy:
            h[(dim + 1):] = np.log((1 + g) * [1.e-8])
        posterior = 1
        if default_prior:
            posterior = default_prior_lnprob(h, 1 + g)
        if posterior == -np.inf:
            continue
        need.append(i)
        priors.append(posterior)
    if need:
        out[need] = np.asarray(priors) + np.asarray(lml(np.exp(P[need])))
    return out


def random_state_tables(rs, num_steps, num_walkers):
    """Draws of a numpy RandomState in emcee's order (per half-step: rand(Ns), randint(Nc, size=Ns), rand(Ns)) as the
    three [num_steps, num_walkers] tables of cmoe_hyperparameter_mcmc; entry [step, w] belongs to walker w."""
    half = num_walkers // 2
    tz = np.empty((num_steps, num_walkers))
    tp = np.empty((num_steps, num_walkers), dtype=np.int32)
    tu = np.empty((num_steps, num_walkers))
    for s in range(num_steps):
        for h in range(2):
            sl = slice(h * half, (h + 1) * half)
            tz[s, sl] = rs.rand(half)
            tp[s, sl] = rs.randint(half, size=(half,))
            tu[s, sl] = rs.rand(half)
    return tz, tp, tu


def stretch_chain(p0, num_steps, lnprob_fn, tables, omit_volume_term=False):
    """EnsembleSampler.sample (emcee 2.2.1) for num_steps steps from p0, random numbers from `tables`.  Returns
    (positions, lnprob, accepts [num_steps, W], margins [num_steps, W]), margin = |lnpdiff - log u| of each decision
    (inf where lnpdiff is not finite, which no rounding can flip).  omit_volume_term drops (ndim - 1) log z: a wrong
    sampler, for showing that the stationary check rejects it."""
    p = np.array(p0, dtype=np.float64)
    k, ndim = p.shape
    if k % 2 or k < 2 * ndim:
        raise ValueError("emcee: the number of walkers must be even and at least twice the dimension")
    tz, tp, tu = tables
    halfk = k // 2
    lnprob = lnprob_fn(p)
    first, second = slice(halfk), slice(halfk, k)
    accepts = np.zeros((num_steps, k), dtype=bool)
    margins = np.full((num_steps, k), np.inf)
    for step in range(num_steps):
        for S0, S1 in [(first, second), (second, first)]:
            s, c = p[S0], p[S1]
            zz = ((STRETCH_A - 1.) * tz[step, S0] + 1) ** 2. / STRETCH_A
            rint = tp[step, S0]
            q = c[rint] - zz[:, np.newaxis] * (c[rint] - s)
            newlnprob = lnprob_fn(q)
            vol = 0.0 if omit_volume_term else (ndim - 1.) * np.log(zz)
            with np.errstate(invalid="ignore", divide="ignore"):  # -inf - -inf: nan, never accepted, as in emcee
                lnpdiff = vol + newlnprob - lnprob[S0]
                logu = np.log(tu[step, S0])
            acc = lnpdiff > logu
            with np.errstate(invalid="ignore"):
                margins[step, S0] = np.where(np.isfinite(lnpdiff), np.abs(lnpdiff - logu), np.inf)
            accepts[step, S0] = acc
            if np.any(acc):
                lnprob[S0][acc] = newlnprob[acc]
                p[S0][acc] = q[acc]
    return p, lnprob, accepts, margins


def numpy_lml_matern52(X, y):
    """log marginal likelihood of the Matern-5/2 GP (no derivative observations) at linear-scale sets H [sets, 2 + dim]
    with 1e-6 added to the noise and the mean of y as the prior mean: the value of cmoe_log_marginal_likelihood_list,
    restated for runs without a device (-inf where the Cholesky fails)."""
    X = np.asarray(X, dtype=np.float64)
    r = np.asarray(y, dtype=np.float64) - np.mean(y)
    n, dim = X.shape

    def lml(H):
        H = np.atleast_2d(H)
        alpha, lengths, noise = H[:, 0], H[:, 1:1 + dim], H[:, 1 + dim] + 1.0e-6
        D = (X[None, :, None, :] - X[None, None, :, :]) / lengths[:, None, None, :]
        dist = np.sqrt(np.sum(D * D, axis=-1))
        a = np.sqrt(5.0) * dist
        K = alpha[:, None, None] * (1.0 + a + a * a / 3.0) * np.exp(-a) + noise[:, None, None] * np.eye(n)
        # Cholesky of every set at once, column by column; a pivot that is not > 0 makes the set -inf
        L = np.zeros_like(K)
        ok = np.ones(len(H), dtype=bool)
        for j in range(n):
            d = K[:, j, j] - np.sum(L[:, j, :j] ** 2, axis=1)
            ok &= d > 0.0
            L[:, j, j] = np.sqrt(np.where(d > 0.0, d, 1.0))
            L[:, j + 1:, j] = (K[:, j + 1:, j] - np.einsum("sik,sk->si", L[:, j + 1:, :j], L[:, j, :j])) / L[:, j, j, None]
        z = np.zeros((len(H), n))
        for i in range(n):
            z[:, i] = (r[i] - np.einsum("sk,sk->s", L[:, i, :i], z[:, :i])) / L[:, i, i]
        val = -0.5 * np.sum(z * z, axis=1) - np.sum(np.log(np.diagonal(L, axis1=1, axis2=2)), axis=1) \
            - 0.5 * n * np.log(2 * np.pi)
        return np.where(ok, val, -np.inf)

    return lml


# ---- the stationary-distribution check ---------------------------------------------------------------------------
# d = 1, N = 5, the default prior, noisy True.  With noisy False the pinned noise entry is the same in every walker, so
# the ensemble spans nh - 1 dimensions while emcee's volume factor is z^(nh - 1), the factor of nh: the chain then
# does not sample the posterior (its spread is about 20 % too wide on this problem), for the reference as here.  With
# noisy True the walkers span all three coordinates (log alpha, log length, log noise) and the chain must reproduce
# the posterior.
def stationary_problem():
    rng = np.random.default_rng(7)
    X = np.sort(rng.uniform(0.0, 1.0, size=(5, 1)), axis=0)
    y = np.sin(3.0 * X[:, 0]) + 0.1 * rng.standard_normal(5)
    return X, y


def grid_moments(lml):
    """Posterior mean and standard deviation of (log alpha, log length, log noise) by quadrature of exp(lnp) over the
    region where the target is not -inf: log alpha and log noise in [-20, 20] (the box), log length in [-2, 3] (the
    tophat).  Midpoint rule; the log noise midpoints avoid the horseshoe's integrable singularity at 0."""
    ga = np.linspace(-20.0, 20.0, 321)
    ga = 0.5 * (ga[1:] + ga[:-1])
    gl = np.linspace(-2.0, 3.0, 101)
    gl = 0.5 * (gl[1:] + gl[:-1])
    gn = ga
    A, L = np.meshgrid(ga, gl, indexing="ij")
    lp = np.empty((ga.size, gl.size, gn.size))
    for k, t in enumerate(gn):  # one likelihood call per noise value
        H = np.exp(np.stack([A.ravel(), L.ravel(), np.full(A.size, t)], axis=1))
        prior = stats.norm.pdf(A.ravel()) + np.log(np.log(1 + 3.0 * (0.1 / t) ** 2))
        lp[:, :, k] = (prior + np.asarray(lml(H))).reshape(A.shape)
    w = np.exp(lp - lp.max())
    w /= w.sum()
    grids = np.meshgrid(ga, gl, gn, indexing="ij")
    mean = np.array([np.sum(w * G) for G in grids])
    sd = np.sqrt(np.array([np.sum(w * (G - m) ** 2) for G, m in zip(grids, mean)]))
    return mean, sd


# Pooled walkers of 64 chains over 4000 steps after a 1000-step burn-in.  log alpha and log length mix within tens of
# steps, but the log noise has a heavy tail down to the box edge (the horseshoe density falls as 1 / theta^2 there and
# the likelihood is flat), so its autocorrelation time is hundreds of steps and its pooled mean and spread carry errors
# of about 0.1 sd.  The bounds are 0.25 sd for the means and 25 % for the standard deviations: about twice the error of
# the correct NumPy sampler on this problem (0.13 sd, 12 %), while a sampler without the (ndim - 1) log z term misses
# them (0.45 sd, 37 %).
MEAN_TOL_SD = 0.25
SD_TOL_REL = 0.25


def stationary_check(samples, mean, sd):
    """(ok, sample mean, sample sd) of pooled samples [*, 3] against the quadrature's moments."""
    m = samples.mean(axis=0)
    s = samples.std(axis=0)
    ok = bool(np.all(np.abs(m - mean) <= MEAN_TOL_SD * sd) and np.all(np.abs(s - sd) <= SD_TOL_REL * sd))
    return ok, m, s


def initial_walkers(rng, num_walkers, dim, g):
    """Walkers spread like DefaultPrior.sample_from_prior (default_priors.py:38-51): log alpha ~ N(0, 1), log lengths
    ~ U(-2, 3), log noise = log |N(0, 1) |Cauchy| 0.1|."""
    p = np.empty((num_walkers, 2 + dim + g))
    p[:, 0] = rng.standard_normal(num_walkers)
    p[:, 1:1 + dim] = rng.uniform(-2.0, 3.0, size=(num_walkers, dim))
    p[:, 1 + dim:] = np.log(np.abs(rng.standard_normal((num_walkers, 1 + g)) *
                                   np.abs(rng.standard_cauchy((num_walkers, 1 + g))) * 0.1))
    return p

"""NumPy restatement of GaussianProcessLogLikelihoodMCMC.optimize's objective (log_likelihood_mcmc.py:241-312):
nll(theta) = -compute_log_likelihood(theta), and its analytic gradient, on top of tests/hyper_mcmc_ref.py's prior.
The likelihood is a callable on one linear-scale set [alpha, lengths..., noise...]; its gradient callable returns
d log p / d (the same set)."""
import numpy as np

import hyper_mcmc_ref as R


def pinned(theta, dim, noisy):
    h = np.array(theta, dtype=np.float64)
    if not noisy:
        h[dim + 1:] = R.LOG_NOISE_FREE
    return h


def nll(theta, lml, dim, g, noisy, default_prior):
    """compute_log_likelihood's order: the box, the pinning (on a copy), the prior, the likelihood."""
    h = np.array(theta, dtype=np.float64)
    if np.any((-20 > h) + (h > 20)):
        return np.inf
    h = pinned(h, dim, noisy)
    prior = R.default_prior_lnprob(h, 1 + g) if default_prior else 1
    if prior == -np.inf:
        return np.inf
    return -(prior + lml(np.exp(h)))


def default_prior_grad(h, dim, g, noisy):
    """d DefaultPrior.lnprob / d theta as the lnprob is written: -theta_0 pdf(theta_0), 0 inside the tophat, and
    d/dt log(log(1 + 3 (0.1 / t)^2)) per noise entry (0 for pinned entries)."""
    d = np.zeros(len(h))
    d[0] = -h[0] * np.exp(-h[0] ** 2 / 2.0) / np.sqrt(2.0 * np.pi)
    if noisy:
        for t in range(1 + dim, len(h)):
            r2 = (0.1 / h[t]) ** 2
            d[t] = -6.0 * r2 / (h[t] * (1.0 + 3.0 * r2) * np.log(1.0 + 3.0 * r2))
    return d


def nll_grad(theta, lml_grad, dim, g, noisy, default_prior):
    """The analytic gradient of nll at theta inside the box with a finite prior."""
    h = pinned(theta, dim, noisy)
    d = default_prior_grad(h, dim, g, noisy) if default_prior else np.zeros(len(h))
    gl = np.exp(h) * np.asarray(lml_grad(np.exp(h)), dtype=np.float64)
    out = -(d + gl)
    if not noisy:
        out[1 + dim:] = 0.0
    return out


def central_diff(f, x, h=1e-6):
    x = np.array(x, dtype=np.float64)
    out = np.empty(len(x))
    for k in range(len(x)):
        e = np.zeros(len(x))
        e[k] = h
        out[k] = (f(x + e) - f(x - e)) / (2.0 * h)
    return out

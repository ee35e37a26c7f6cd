"""CPU run of the stationary check of tests/test_gpu_hyper_mcmc.py on the NumPy restatement (tests/hyper_mcmc_ref.py)
with a NumPy likelihood, once as emcee samples and once without the (ndim - 1) log z term of the stretch move: the
check accepts the first and rejects the second.  No device needed; takes a few minutes."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import hyper_mcmc_ref as R  # noqa: E402

X, y = R.stationary_problem()
lml = R.numpy_lml_matern52(X, y)
mean, sd = R.grid_moments(lml)
print("quadrature mean", mean, "sd", sd)
for omit in (False, True):
    rs = np.random.RandomState(11)
    p = R.initial_walkers(np.random.default_rng(3), 64, 1, 0)
    lp = lambda P: R.log_prob(P, lml, 1, 0, True, True)  # noqa: E731
    p, _, _, _ = R.stretch_chain(p, 1000, lp, R.random_state_tables(rs, 1000, 64), omit_volume_term=omit)
    pool = []
    for c in range(400):
        p, _, _, _ = R.stretch_chain(p, 10, lp, R.random_state_tables(rs, 10, 64), omit_volume_term=omit)
        pool.append(p.copy())
    ok, m, s = R.stationary_check(np.concatenate(pool), mean, sd)
    print(f"{'without' if omit else 'with'} the volume term: check {'passes' if ok else 'fails'}; "
          f"mean error / sd {np.round((m - mean) / sd, 3)}, sd error {np.round(s / sd - 1, 3)}")

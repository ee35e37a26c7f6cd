"""Host restatement of the ensemble posterior-mean path (cmoe_posterior_mean_mcmc, cmoe_posterior_mean_mcmc_optimization)
for the parity tests, driven by per-member means from a CPU checker.

* ``ensemble_objective``: PosteriorMeanMCMC.compute_objective_function / compute_grad_objective_function
  (cpp_wrappers/knowledge_gradient_mcmc.py:72-157): the members' -mu_m (fidelity coordinates pinned to 1.0) added to 0
  in ascending order, then divided by M.
* ``gradient_descent``: python_version GradientDescentOptimizer.optimize (optimization.py:444-527) on a tensor-product
  box with compute_update_restricted_to_domain (python_version/domain.py:158-202), and _get_averaging_range (:415-442).
  The average adds the points in ascending step order, then divides by their number.
* ``multistart``: MultistartOptimizer.optimize (optimization.py:565-606): best value from -inf, best point from
  starts[0], strict `>` in start order.
* ``recommend``: the recommendation block of examples/main.py:243-260.
"""
import numpy as np


def averaging_range(num_steps_averaged, num_steps_total):
    if num_steps_averaged < 0 or num_steps_averaged > num_steps_total:
        num_steps_averaged = num_steps_total
    elif num_steps_averaged == 0:
        num_steps_averaged = 1
    return num_steps_total - num_steps_averaged + 1, num_steps_total + 1


def ensemble_objective(means, grad_means, dim, num_fidelity):
    """means[m](x_full) -> mu_m(x); grad_means[m](x_full) -> d mu_m / dx [dim].  Returns (f, grad_f) on the free
    coordinates."""
    ps = dim - num_fidelity

    def full(x):
        out = np.ones(dim)
        out[:ps] = x
        return out

    def f(x):
        acc = 0.0
        for mu in means:
            acc = acc + (-mu(full(x)))
        return acc / len(means)

    def grad_f(x):
        acc = np.zeros(ps)
        for gmu in grad_means:
            acc = acc + (-np.asarray(gmu(full(x)), dtype=np.float64)[:ps])
        return acc / len(grad_means)

    return f, grad_f


def gradient_descent(grad_f, x0, params, bounds):
    """params: (max_num_steps, num_steps_averaged, gamma, pre_mult, max_relative_change); bounds [ps, 2].
    Returns the averaged point."""
    steps, nav, gamma, pre_mult, mrc = params
    bounds = np.asarray(bounds, dtype=np.float64).reshape(-1, 2)
    path = [np.array(x0, dtype=np.float64)]
    for k in range(1, steps + 1):
        alpha = pre_mult * np.power(float(k), -gamma)
        x = path[-1]
        step = grad_f(x) * alpha
        out = np.empty_like(x)
        for j, s in enumerate(step):
            dist = np.fmin(x[j] - bounds[j, 0], bounds[j, 1] - x[j])
            out[j] = np.copysign(mrc * dist, s) if np.fabs(s) > mrc * dist else s
        path.append(out + x)
    start, end = averaging_range(nav, steps)
    acc = path[start].copy()
    for k in range(start + 1, end):
        acc = acc + path[k]
    return acc / float(end - start)


def multistart(f, grad_f, starts, params, bounds):
    """(points [S, ps], values [S], best_point, best_value, best_index) with best_index = -1 if no start beat -inf."""
    starts = np.asarray(starts, dtype=np.float64)
    pts = np.array([gradient_descent(grad_f, s, params, bounds) for s in starts])
    vals = np.array([f(p) for p in pts])
    best_value, best_point, best_index = -np.inf, starts[0], -1
    for i, v in enumerate(vals):
        if v > best_value:
            best_value, best_point, best_index = v, pts[i], i
    return pts, vals, best_point, best_value, best_index


def recommend(f, grad_f, eval_pts, params, bounds):
    """(report point, index of the screened start, screening values f)."""
    screen = np.array([f(p) for p in eval_pts])
    test = -screen
    i0 = int(np.argmin(test))
    _, _, point, value, _ = multistart(f, grad_f, eval_pts[i0][None], params, bounds)
    return (eval_pts[i0].copy() if -value > np.min(test) else point), i0, screen

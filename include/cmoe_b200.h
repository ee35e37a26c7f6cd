/* cornell-moe_b200 — C ABI of the H100-native (sm_90a) GP-posterior + Monte-Carlo acquisition path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / CUDA types.  Every entry point
 * states which interface of the reference (wujian16/Cornell-MOE, paths relative to
 * moe/optimal_learning/cpp/) it replaces.  The pybind11 module `GPP` in cornell-moe_b200/csrc/gpp_module.cpp
 * re-exports the reference's `moe.build.GPP` names on top of exactly these calls; INTEGRATION.md shows the
 * binding a reference maintainer would add.
 *
 * Conventions are the reference's own (gpp_common.hpp:29,390; gpp_math.hpp:301-305):
 *   - all reals are IEEE double, all matrices column-major, point sets are [num_points][dim];
 *   - observations are interleaved per point: (value, d/dx_{derivatives[0]}, ...);
 *   - noise_variance has 1+num_derivatives entries and is indexed by observation TYPE, not by point
 *     (gpp_math.cpp:447-449);
 *   - host pointers in, host pointers out, no ownership transfer (gpp_python_common.cpp:37, 79-128).
 *
 * Errors: every function returns a status code; CMOE_ERR_* map 1:1 onto the reference's exception
 * classes (gpp_exception.hpp:170-509, gpp_python.cpp:189-206).  `info` receives the payload
 * (leading-minor index k+1 for CMOE_ERR_SINGULAR, exactly as gpp_linear_algebra.cpp:141-142 returns it).
 * There is NO CPU fallback: without a CUDA device every compute call returns CMOE_ERR_NO_DEVICE.
 *
 * Threading: like the reference's Python boundary (GIL held for the whole call) a handle is used by one host thread at a
 * time; calls on the same cmoe_gp are issued on that handle's CUDA stream and must be serialised by the caller.
 * Repeated cmoe_kg_eval calls with an unchanged configuration reuse a device workspace cached in the handle.
 */
#ifndef CMOE_B200_H_
#define CMOE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CMOE_OK 0
#define CMOE_ERR_SINGULAR 1      /* SingularMatrixException   (gpp_exception.hpp:465) */
#define CMOE_ERR_BOUNDS 2        /* BoundsException           (gpp_exception.hpp:243) */
#define CMOE_ERR_INVALID_VALUE 3 /* InvalidValueException     (gpp_exception.hpp:382) */
#define CMOE_ERR_RUNTIME 4       /* OptimalLearningException  (gpp_exception.hpp:170): CUDA / internal failure */
#define CMOE_ERR_NO_DEVICE 5     /* OptimalLearningException: no CUDA device; there is no CPU path */

#define CMOE_KERNEL_SQUARE_EXPONENTIAL 0 /* gpp_covariance.hpp:195 */
#define CMOE_KERNEL_MATERN_NU_2P5 1      /* gpp_covariance.hpp:313 */

#define CMOE_MAX_DIM 32

typedef struct cmoe_gp cmoe_gp; /* opaque; replaces optimal_learning::GaussianProcess (gpp_math.hpp:275) */

/* GradientDescentParameters, gpp_optimizer_parameters.hpp:81-135 (same field order as its constructor) */
typedef struct cmoe_gd_params {
  int num_multistarts;
  int max_num_steps;
  int max_num_restarts;
  int num_steps_averaged;
  double gamma;
  double pre_mult;
  double max_relative_change;
  double tolerance;
} cmoe_gd_params;

/* Work counters reported by the fused q-KG kernel (it counts what it actually executed). */
typedef struct cmoe_kg_stats {
  uint64_t mc_samples;         /* candidates * num_mc */
  uint64_t posterior_evals;    /* posterior-mean evaluations the reference's line search would have made for the
                                  same trajectory (trial points + domain-limited points + start points) */
  uint64_t line_search_steps;  /* accepted inner gradient steps */
  uint64_t point_evals;        /* executed: value+gradient evaluations at one query point */
  uint64_t line_batches;       /* executed: batched backtracking passes (SquareExponential fast path; all trial step
                                  sizes of one step share one pass over the training points) */
} cmoe_kg_stats;

/* Human-readable description of the last error on the calling thread. */
const char* cmoe_last_error(void);
const char* cmoe_version(void);
/* Number of visible CUDA devices (0 if none / driver missing). */
int cmoe_device_count(void);

/* ---- GaussianProcess --------------------------------------------------------------------------------------
 * cmoe_gp_create  replaces GaussianProcess::GaussianProcess (gpp_math.cpp:553-573) == covariance build
 *   (gpp_math.cpp:426-455) + Cholesky (gpp_linear_algebra.cpp:109-148) + K^-1 (y - mean) (gpp_math.cpp:481-511);
 *   Python boundary: make_gaussian_process, gpp_python_gaussian_process.cpp:42-62.
 *   hyperparameters = (alpha, lengths[dim]).  device = CUDA ordinal (the reference's dead `which_gpu`).
 *   On a singular K: returns CMOE_ERR_SINGULAR, *info = leading minor index, *gp_out = NULL. */
int cmoe_gp_create(int kernel, double alpha, const double* lengths, const double* points_sampled,
                   const double* points_sampled_value, const double* noise_variance, const int* derivatives,
                   int num_derivatives, int dim, int num_sampled, int device, cmoe_gp** gp_out, int* info);
/* log p(y | X, theta) = -1/2 (y-m)^T K^-1 (y-m) - sum_i log L_ii - n/2 log(2 pi) with K = K(X,X) + diag(noise by type)
 * + 1e-6 I: LogMarginalLikelihoodEvaluator::ComputeLogLikelihood with FillLogLikelihoodState
 * (gpp_model_selection.cpp:540-612); Python boundary compute_log_likelihood (gpp_python_model_selection.cpp:43-87) —
 * the call the hyper-parameter MCMC of the front end makes thousands of times per refit.  One GP fit on the device
 * (covariance build, Cholesky, K^-1 y) plus two reductions over n numbers.  A singular K yields -inf (the reference
 * ignores the failed factorisation, :551-553).  SURVEY.md 8f rank 2, value only (no hyper-parameter gradient yet). */
int cmoe_log_marginal_likelihood(int kernel, double alpha, const double* lengths, const double* points_sampled,
                                 const double* points_sampled_value, const double* noise_variance,
                                 const int* derivatives, int num_derivatives, int dim, int num_sampled, int device,
                                 double* log_likelihood, int* info);
/* d log p / d (alpha, l_1..l_dim, noise_0..noise_g): LogMarginalLikelihoodEvaluator::ComputeGradLogLikelihood
 * (gpp_model_selection.cpp:629-690) with HyperparameterGradCovariance (gpp_covariance.cpp:245-317, 461-489); Python
 * boundary compute_hyperparameter_grad_log_likelihood (gpp_python_model_selection.cpp:89-140).  grad[dim + 2 + g].
 * One device fit, K^-1 by the blocked solves, one fused 1/2 tr[(a a^T - K^-1) dK/d theta] contraction kernel.  Keeps the
 * reference's Matern quirk (only the value-value entry of a derivative block contributes).  Singular K: zeros. */
int cmoe_grad_log_marginal_likelihood(int kernel, double alpha, const double* lengths, const double* points_sampled,
                                      const double* points_sampled_value, const double* noise_variance,
                                      const int* derivatives, int num_derivatives, int dim, int num_sampled, int device,
                                      double* grad, int* info);
/* log p(y | X, theta_s) for num_sets hyper-parameter sets in one device call: EvaluateLogLikelihoodAtPointList
 * (gpp_model_selection.hpp:1274-1308); Python boundary evaluate_log_likelihood_at_hyperparameter_list
 * (gpp_python_model_selection.cpp:281-341, 520-556).  hyperparameters[num_sets][2 + dim + g], each set
 * (alpha, lengths[dim], noise_variance[1 + g]), the reference's problem-size layout (gpp_model_selection.cpp:798-811).
 * Per set the value is cmoe_log_marginal_likelihood's: 1e-6 added to every noise entry, the prior mean = average of
 * the function values, -1/2 z^T z - sum_i log L_ii - n/2 log 2 pi with z = L^-1 (y - mean); a set whose Cholesky fails
 * gets -inf and leaves the others unaffected.  values[num_sets] in list order.  Unlike the reference, every set is
 * checked (alpha > 0, lengths > 0; CMOE_ERR_BOUNDS naming the set); num_sets >= 1, num_sampled (1 + g) <= 8192.
 * The sets are processed in chunks of at most 4096 sets and about 2 GiB of device workspace, which is kept per host
 * thread for the device of the last call.  A set's value does not depend on the rest of the list. */
int cmoe_log_marginal_likelihood_list(int kernel, const double* hyperparameters, int num_sets,
                                      const double* points_sampled, const double* points_sampled_value,
                                      const int* derivatives, int num_derivatives, int dim, int num_sampled, int device,
                                      double* values, int* info);
/* Value and hyper-parameter gradient at num_sets sets in one device call (DESIGN.md K11), in the layout and with the
 * size contract and checks of cmoe_log_marginal_likelihood_list.  values[num_sets] are bit for bit that call's;
 * grads[num_sets][2 + dim + g] = d log p / d (alpha, lengths..., noise by observation type), defined as
 * cmoe_grad_log_marginal_likelihood's (1e-6 added to the noise; the Matern-5/2 value-entry-only quirk).  A set whose
 * Cholesky fails gets value -inf and a zero gradient.  A set's outputs do not depend on the rest of the list. */
int cmoe_grad_log_marginal_likelihood_list(int kernel, const double* hyperparameters, int num_sets,
                                           const double* points_sampled, const double* points_sampled_value,
                                           const int* derivatives, int num_derivatives, int dim, int num_sampled,
                                           int device, double* values, double* grads, int* info);
/* The exact hyper-parameter gradient: cmoe_grad_log_marginal_likelihood_list's signature, layout, checks and values,
 * with grads the true d log p / d (alpha, lengths..., noise by observation type).  For Matern-5/2 with derivative
 * observations every entry of each (1 + g) x (1 + g) derivative block contributes, coincident points included, where
 * the quirk-keeping call uses the value-value entry only.  With g = 0, and for SquareExponential (whose branch is exact),
 * the results equal cmoe_grad_log_marginal_likelihood_list's bit for bit. */
int cmoe_grad_log_marginal_likelihood_list_exact(int kernel, const double* hyperparameters, int num_sets,
                                                 const double* points_sampled, const double* points_sampled_value,
                                                 const int* derivatives, int num_derivatives, int dim, int num_sampled,
                                                 int device, double* values, double* grads, int* info);
/* Maximum-likelihood fit of the hyper-parameters by restarted gradient ascent from every one of num_starts starts
 * [num_starts][nh], nh = 2 + dim + g, on the linear-space box bounds[nh][2]: MultistartGradientDescentHyperparameter-
 * Optimization (gpp_model_selection.hpp:1063-1103) with one thread, every start descending in lock step with one
 * cmoe_grad_log_marginal_likelihood_list call per step.  best_point[nh] / best_value: the best start (first maximum of
 * the start values) unless some end value beats it, then the first maximum of the end values; found_flag: whether one
 * did.  end_points[num_starts][nh] / end_values[num_starts] (each may be NULL): every start's result.  Unlike the
 * reference, a set whose Cholesky fails mid-descent has a zero gradient, so that start stops where it is. */
int cmoe_hyperparameter_gradient_descent(int kernel, const cmoe_gd_params* gd_params, const double* bounds,
                                         const double* starts, int num_starts, const double* points_sampled,
                                         const double* points_sampled_value, const int* derivatives,
                                         int num_derivatives, int dim, int num_sampled, int device,
                                         double* best_point, double* best_value, int* found_flag,
                                         double* end_points, double* end_values, int* info);
/* Priors of cmoe_hyperparameter_mcmc: the two the reference's GaussianProcessLogLikelihoodMCMC front end uses. */
#define CMOE_HYPER_PRIOR_NONE 0    /* prior = None: the constant 1 (log_likelihood_mcmc.py:291) */
#define CMOE_HYPER_PRIOR_DEFAULT 1 /* DefaultPrior(nh, 1 + g) (default_priors.py:27-37) */
/* Host-supplied random numbers of cmoe_hyperparameter_mcmc, each [num_steps][num_walkers] and indexed by the step of
 * the call and the walker: the uniform of the stretch factor, the partner (an index into the other half of the
 * ensemble, in [0, num_walkers / 2)) and the acceptance uniform.  Entries of the half that does not move are unused. */
typedef struct cmoe_mcmc_table {
  const double* z_uniform;
  const int* partner;
  const double* accept_uniform;
} cmoe_mcmc_table;
/* Hyper-parameter MCMC (DESIGN.md K12): num_steps steps of emcee 2.2.1's EnsembleSampler.sample (stretch move, a = 2)
 * on the log-probability of GaussianProcessLogLikelihoodMCMC.compute_log_likelihood (log_likelihood_mcmc.py:277-312),
 * the whole chain on the device in one call.  A walker is theta = (log alpha, log l_1..l_dim, log noise_0..noise_g),
 * nh = 2 + dim + g entries; its log-probability is -inf outside [-20, 20]^nh, else (with noisy == 0 the noise entries
 * are first set to log(1e-8) in the walker itself, so the pinned values persist in the chain) prior + the value of
 * cmoe_log_marginal_likelihood_list at exp(theta), -inf if the prior is -inf or the Cholesky fails.
 * initial_positions[num_walkers][nh]; the initial log-probabilities are evaluated first, as run_mcmc does.  Random
 * numbers: table == NULL draws them from Philox4x32-10 keyed by seed, a pure function of (seed, first_step + step,
 * walker), so a chain split over several calls (first_step = steps done so far) is bit-identical to one call; else
 * from *table.  Outputs: positions[num_walkers][nh] and log_probabilities[num_walkers] after the last step.
 * Bounds (CMOE_ERR_BOUNDS, before any device work): num_walkers even and >= 2 nh, num_steps >= 1, the K10 size
 * contract (dim <= CMOE_MAX_DIM, num_sampled (1 + g) <= 8192) and num_walkers / 2 sets within one K10 chunk (4096
 * sets and about 2 GiB: 3 sets at n = 8192).  Non-finite initial positions are CMOE_ERR_INVALID_VALUE (emcee raises). */
int cmoe_hyperparameter_mcmc(int kernel, int prior, int noisy, const double* initial_positions, int num_walkers,
                             int num_steps, uint64_t seed, uint64_t first_step, const cmoe_mcmc_table* table,
                             const double* points_sampled, const double* points_sampled_value, const int* derivatives,
                             int num_derivatives, int dim, int num_sampled, int device, double* positions,
                             double* log_probabilities, int* info);
/* Options of cmoe_hyperparameter_map; NULL gives the defaults. */
typedef struct cmoe_map_opts {
  double gtol;         /* stop at ||gradient||_inf <= gtol (scipy's default 1e-5); >= 0 */
  int max_iterations;  /* BFGS iterations per start; 0 = 200 nh (scipy's default) */
} cmoe_map_opts;
/* Hyper-parameter MAP fit (DESIGN.md K19): GaussianProcessLogLikelihoodMCMC.optimize (log_likelihood_mcmc.py:241-275),
 * scipy.optimize.minimize(nll, p0) with BFGS, from every one of num_starts starts[num_starts][nh] in one call, with the
 * analytic gradient instead of finite differences.  theta = (log alpha, log l_1..l_dim, log noise_0..noise_g), nh =
 * 2 + dim + g, and nll(theta) = -compute_log_likelihood(theta): +inf outside [-20, 20]^nh; with noisy == 0 the noise
 * entries of a copy of theta are log(1e-8) (their gradient entries are 0 and positions keep the start's values); then
 * minus (the prior, CMOE_HYPER_PRIOR_NONE = 1 or CMOE_HYPER_PRIOR_DEFAULT, plus the value of
 * cmoe_log_marginal_likelihood_list at exp(theta)).  The likelihood gradient is the exact one of
 * cmoe_grad_log_marginal_likelihood_list_exact.  BFGS as scipy's _minimize_bfgs (H0 = I, the first step from
 * old_old_fval = f + ||g||_2 / 2, rho = 1000 when y^T s == 0) with scipy's strong-Wolfe line_search_wolfe2 (c1 = 1e-4,
 * c2 = 0.9, 10 bracketing steps, at most 10 zoom trials; a +inf or NaN trial fails sufficient decrease).
 * Outputs per start: positions[num_starts][nh], values[num_starts] = nll there, gradients[num_starts][nh],
 * iterations, evaluations (value-and-gradient evaluations, the start's included) and status: 0 converged
 * (||g||_inf <= gtol), 1 max_iterations, 2 line search failed or objective not finite (scipy's warnflag 2; a start
 * outside the box gives value +inf), 3 NaN.  A start's results do not depend on the other starts.
 * Bounds (CMOE_ERR_BOUNDS, before any device work): the K10 size contract (dim <= CMOE_MAX_DIM, so nh <= 2 + 2
 * CMOE_MAX_DIM; num_sampled (1 + g) <= 8192), num_starts >= 1 and all starts within one K11 chunk (4096 sets and about
 * 2 GiB).  NULL pointers, a kernel, prior or noisy value outside the defined ones and bad opts: CMOE_ERR_INVALID_VALUE. */
int cmoe_hyperparameter_map(int kernel, int prior, int noisy, const double* starts, int num_starts,
                            const cmoe_map_opts* opts, const double* points_sampled,
                            const double* points_sampled_value, const int* derivatives, int num_derivatives,
                            int dim, int num_sampled, int device, double* positions, double* values,
                            double* gradients, int* iterations, int* evaluations, int* status, int* info);
/* Run-time switches between kernel generations (also read once from the environment: CMOE_LEGACY_LINALG, CMOE_COV_TMA):
 *   "legacy_linalg" 1 = round-1 launch-per-step Cholesky / chained trsv for large n (default 0: cooperative kernels);
 *   "cov_tma"       1 = TMA / DMMA covariance build with tensor-map tile stores (default 0: LDGSTS kernel, faster at d ~ 10);
 *   "ensemble_members_in_flight"  k >= 1 = at most k members of an ensemble run at once on the large-union q-KG / q-EI
 *                   stages (default 0: as many as the 2 GiB workspace holds).  Results do not depend on it. */
int cmoe_set_option(const char* name, int value);
void cmoe_gp_destroy(cmoe_gp* gp);
int cmoe_gp_dim(const cmoe_gp* gp);
int cmoe_gp_device(const cmoe_gp* gp);
int cmoe_gp_num_sampled(const cmoe_gp* gp);
int cmoe_gp_num_derivatives(const cmoe_gp* gp);
/* Copies out K_chol_ (n*n, lower triangle valid), K_inv_y_ (n) and mean_ (gpp_math.hpp:838-867); any may be NULL. */
int cmoe_gp_get_state(const cmoe_gp* gp, double* K_chol, double* K_inv_y, double* mean);
/* GaussianProcess::AddPointsToGP (gpp_math.cpp:1699-1718): append and refit. */
int cmoe_gp_add_sampled_points(cmoe_gp* gp, const double* new_points, const double* new_points_value,
                               int num_new_points, int* info);
/* Timings of the last fit, microseconds of device time: {covariance build, Cholesky, K^-1 y solve}. */
int cmoe_gp_fit_timings(const cmoe_gp* gp, double* usec3);

/* ---- posterior queries, batched over point sets -------------------------------------------------------------
 * Replaces ComputeMeanOfPoints (gpp_math.cpp:662), ComputeGradMeanOfPoints (:721), ComputeVarianceOfPoints (:924),
 * ComputeGradVarianceOfPoints (:1366), ComputeGradCholeskyVarianceOfPoints (:1466) and the q*q Cholesky; Python
 * boundary gpp_python_gaussian_process.cpp:64-236.  `sets` = [num_sets][num_pts][dim]; each point carries the
 * derivative rows derivs_s[g_s] (Q = num_pts*(1+g_s)).  Outputs per set, reference layouts:
 *   mean[Q]; grad_mean[Q][dim] (d fastest); var[Q*Q] col-major (full symmetric); chol_var[Q*Q] (lower, upper zeroed);
 *   grad_var / grad_chol [num_pts][Q][Q][dim] (d fastest; grad_chol in the reference's transposed storage,
 *   gpp_math.cpp:1416-1417).  Any output may be NULL.  chol failure -> CMOE_ERR_SINGULAR, *info = index. */
int cmoe_gp_posterior(const cmoe_gp* gp, const double* sets, int num_sets, int num_pts, const int* derivs_s, int g_s,
                      double* mean, double* grad_mean, double* var, double* chol_var, double* grad_var,
                      double* grad_chol, int* info);
/* Largest Q = num_pts (1 + g_s) of cmoe_gp_posterior's variance outputs and largest q + p of cmoe_ei_eval. */
#define CMOE_MAX_SET_ROWS 96
/* Largest Q of cmoe_gp_posterior_large and largest q + p of cmoe_ei_eval_large. */
#define CMOE_MAX_LARGE_SET_ROWS 8192
/* Largest Q = (q + p)(1 + num_derivatives) of cmoe_kg_eval and the cmoe_kg_plan_* API. */
#define CMOE_MAX_KG_ROWS 32
/* cmoe_gp_posterior's mean, var and chol_var for 1 <= Q = num_pts (1 + g_s) <= 8192, in its layouts (any output may be
 * NULL).  Computed by the stages of cmoe_gp_sample_joint: Var = K(P,P) - V^T V with V = L^-1 K(X,P), factored by the
 * batched blocked Cholesky (the reference's (K^-1 K*)^T K* differs by rounding).  Sets run in chunks that fit the handle's
 * 2 GiB sampling workspace; a set's result does not depend on the chunking.  chol failure -> CMOE_ERR_SINGULAR,
 * *info = leading minor of the first failing set.  The gradients of Var and of its factor are not offered here: they
 * hold num_pts Q^2 dim doubles per set (8.6 GB at Q = 512, dim = 8). */
int cmoe_gp_posterior_large(const cmoe_gp* gp, const double* sets, int num_sets, int num_pts, const int* derivs_s,
                            int g_s, double* mean, double* var, double* chol_var, int* info);

/* ---- joint posterior draws, batched over point sets ------------------------------------------------------------
 * Joint posterior draws over point sets: GaussianProcess::SamplePointsFromGP (gpp_math.cpp:1803-1848) batched over sets;
 * SamplePointFromGP (:1761-1798) is the one-point case carrying the GP's derivative rows.  Python boundary
 * SamplePointFromGPWrapper (gpp_python_gaussian_process.cpp:255-269).
 * sets [num_sets][num_pts][dim]; each point carries derivative rows derivs_s[g_s]; Q = num_pts*(1+g_s) <= 8192.
 * Set b draws Q normals: Philox draw (first_draw + b), exactly cmoe_philox_normals(seed, first_draw + b, 1, Q),
 * or row b of normals_table [num_sets][Q] when it is not NULL (NormalRNG replay for parity).
 * jitter >= 0 is added to the diagonal before factorisation (0 = the reference).
 * samples [num_sets][Q]; argmin [num_sets] = index of the point with the smallest value row (ties: lowest index);
 * mean [num_sets][Q]; chol [num_sets][Q*Q] (lower, upper zeroed). Every output may be NULL.
 * The posterior covariance is K(P,P) - V^T V with V = L^-1 K(X,P) (one triangular solve; the reference uses
 * (K^-1 K*)^T K*, which differs by rounding).  Sets are processed in chunks that fit a 2 GiB device workspace (or one
 * set, if larger); a set's result does not depend on the chunking.  The workspace is kept on the handle (grown on demand,
 * released by cmoe_gp_destroy), as the q-KG workspace is.
 * A failed factorisation (pivot <= 1e-16) -> CMOE_ERR_SINGULAR, *info = leading minor of the first failing set.
 * (The reference ignores the failure and applies the partial factor; its argmin starts at -1 with a strict `<`, so a
 * minimum at point 0 yields -1 there and 0 here.) */
int cmoe_gp_sample_joint(const cmoe_gp* gp, const double* sets, int num_sets, int num_pts, const int* derivs_s, int g_s,
                         uint64_t seed, uint64_t first_draw, const double* normals_table, double jitter,
                         double* samples, int* argmin, double* mean, double* chol, int* info);
/* Latin hypercube in a box (ComputeLatinHypercubePointsInDomain, gpp_random.cpp:173-194): out [num_sets][num_pts][dim].
 * domain_bounds [dim][2] = (min, max), min <= max; num_pts <= 8192.  Set b is a pure function of (seed, first_draw + b):
 * the strata of each dimension are permuted by ranking Philox uniforms (counter word 3 = 1, the normals use 0). */
int cmoe_latin_hypercube(uint64_t seed, uint64_t first_draw, int num_sets, int num_pts, int dim,
                         const double* domain_bounds, double* out, int device);
/* SampleGlobalOptimaFromGP (gpp_math.cpp:1854-1870): optimum b = argmin of one joint draw over the Latin hypercube
 * cmoe_latin_hypercube(seed, first_draw + b, 1, inner_number, ...). points_optima [num_optima][dim].
 * Python boundary SampleGlobalOptimaFromGPWrapper (gpp_python_gaussian_process.cpp:271-286). */
int cmoe_gp_sample_global_optima(const cmoe_gp* gp, int num_optima, int inner_number, const double* domain_bounds,
                                 uint64_t seed, uint64_t first_draw, double jitter, double* points_optima, int* info);

/* ---- random-feature Thompson sampling of the global minimum ------------------------------------------------------
 * sample_from_global_optima (moe/optimal_learning/python/random_features.py:29-175) in one call: num_points samples of
 * the GP drawn as random-Fourier-feature functions, each minimised over the grid and then locally inside the domain.
 * The handle holds n points X (raw coordinates), values y[n][1+g], partials derivs[g], per-type noise nu[1+g] and
 * alpha = sigma^2, lengths l[d].  M = n (1 + g), F = num_features, c = sqrt(2 sigma^2 / F).  For sample s:
 *   features    W = Omega / l (Omega F x d standard normals), b = 2 pi u (u F uniforms); always the spectral density of
 *               SquareExponential, whatever the handle's kernel;
 *   design      Phi (F x M), value columns first: column i = c cos(W x_i + b) / sqrt(nu_0), then one block per derivative
 *               type k (partial j = derivs[k]): -c W[:, j] sin(W x_i + b) / sqrt(nu_{k+1}); y' = y[:, t] / sqrt(nu_t)
 *               flattened type-major.  The raw values are used with a zero prior mean (the GP's mean is not subtracted);
 *   posterior   theta ~ N(m, (I + Phi Phi^T)^-1), m = (I + Phi Phi^T)^-1 Phi y'.  Branch by size, as the reference:
 *               M < F  (Woodbury): A = I_M + Phi^T Phi = L L^T, theta = r - Phi A^-1 (Phi^T r + eps), r = Phi y' + z,
 *                      z in R^F and eps in R^M standard normals.  This pathwise update has exactly the target
 *                      distribution; the reference applies the symmetric square root of A from an eigensolver instead, so
 *                      this branch matches it in distribution, not draw for draw;
 *               M >= F: B = I_F + Phi Phi^T = U U^T (U upper, the lower factor of the order-reversed B), m = B^-1 Phi y',
 *                      theta = m + U^-T z: the reference's z^T cholesky(B^-1, upper), draw for draw given (Omega, u, z);
 *   function    f(x) = c sum_f theta_f cos(W_f x + b_f);
 *   grid        argmin of f over grid[num_grid][d] (shared by all samples), ties to the lowest index;
 *   local       projected Newton inside domain_bounds from the grid argmin (clamped into the box), one warp per sample:
 *               exact d x d Hessian; a variable within eps_k = min(1e-3 (hi_k - lo_k), ||x - P(x - grad f)||_inf) of a
 *               bound whose gradient points outward is held and steps along -grad f (Bertsekas' epsilon-active set); a
 *               free variable at a bound drops an outward Newton component; the free block is shifted to positive definite (H + tau I, tau doubled from 1e-3 max|H_ii| until its Cholesky succeeds);
 *               Armijo backtracking along the projected arc (sufficient decrease 1e-4, up to 60 halvings, rounding slack
 *               1e-13 (1 + |f|)); at most 100 iterations; stops when ||x - P(x - grad f(x))||_inf <= 1e-9 (1 + |f(x)|).
 *               The end point is kept only if f there is strictly below the grid minimum, else the grid point is
 *               returned (random_features.py:164).  The reference uses SLSQP here.
 * points[num_points][d], values[num_points] (f at the returned point).  omega[num_points][F][d] (the frequencies W =
 * Omega / l), b[num_points][F] and theta[num_points][F] may be NULL; they return each sample function.
 * Randomness: sample s is a pure function of (seed, first_draw + s): Omega (row-major), then z, then eps (M < F only) are
 * the normals 0 .. F d + F + M - 1 of Philox draw first_draw + s (cmoe_philox_normals), and u_f comes from the Philox
 * call (draw, f / 2) with counter word 3 = 2 (words 0, 1 for even f, 2, 3 for odd f, as 53-bit uniforms).  With a table,
 * the table's numbers replace Philox: omega[P][F][d] (Omega), b[P][F] (b itself), z[P][F], eps[P][M] (read only when
 * M < F).  Samples run in chunks that fit the handle's 2 GiB sampling workspace; a sample's result does not depend on
 * num_points or the chunking.  The caller's GP is not modified.
 * Errors (before any device work, the first two before gp is read): CMOE_ERR_BOUNDS unless num_features, num_points,
 * num_grid >= 1; CMOE_ERR_INVALID_VALUE for a NULL gp; CMOE_ERR_BOUNDS unless min(F, M) <= 8192 and
 * (F M + min(F, M)^2) doubles fit in 2 GiB; CMOE_ERR_INVALID_VALUE for NULL arguments, non-finite grid points or bounds,
 * min > max, or a noise variance that is not > 0.  A failed factorisation (non-finite data) -> CMOE_ERR_SINGULAR. */
typedef struct cmoe_rff_table {
  const double* omega; /* [P][F][d] standard normals */
  const double* b;     /* [P][F] phases */
  const double* z;     /* [P][F] */
  const double* eps;   /* [P][M], read only when M < F */
} cmoe_rff_table;

int cmoe_gp_sample_rff_optima(const cmoe_gp* gp, int num_features, int num_points, const double* domain_bounds,
                              const double* grid, int num_grid, uint64_t seed, uint64_t first_draw,
                              const cmoe_rff_table* table, double* points, double* values, double* omega, double* b,
                              double* theta, int* info);

/* ---- kernel-matched random features, the sample functions alone, and their evaluation -----------------------------
 * opts->spectral selects the frequencies' distribution:
 *   CMOE_RFF_SPECTRAL_REFERENCE (the default, and opts == NULL): W = Omega / l whatever the kernel, the reference's draw;
 *   CMOE_RFF_SPECTRAL_KERNEL: the handle's own kernel.  For Matern-5/2, k = alpha (1 + sqrt5 r + 5 r^2 / 3) e^(-sqrt5 r)
 *     with r = ||(x - x') / l||, whose spectral measure is a multivariate Student-t with 5 degrees of freedom:
 *     W_f = (Omega_f / l) sqrt(5 / g_f), g_f ~ chi^2_5, computed as __dmul_rn(Omega / l, sqrt(5 / g)) (each operation
 *     rounded once).  g_f = -2 ln u0 - 2 ln u1 + (-2 ln u2) cos^2(2 pi v2), the sum of squares of five Box-Muller normals
 *     (a pair's squares sum to -2 ln u), from the Philox calls (draw, 2f) -> (u0, u1) and (draw, 2f + 1) -> (u2, v2)
 *     with counter word 3 = 3 (53-bit uniforms as for b).  Omega, b, z and eps are the reference mode's numbers, so a
 *     matched sample differs from the reference-mode sample of the same (seed, draw) only by the per-row factor.  For a
 *     SquareExponential handle the matched draw is the reference draw.
 * opts->chi2[P][F] replaces g in table mode; it is read only when a table is given and the draw is the Matern one, and
 * then each entry must be finite and > 0.  The design matrix, both posterior branches, the grid stage and the local
 * optimiser are those of cmoe_gp_sample_rff_optima. */
#define CMOE_RFF_SPECTRAL_REFERENCE 0
#define CMOE_RFF_SPECTRAL_KERNEL 1
typedef struct cmoe_rff_opts {
  int spectral;        /* CMOE_RFF_SPECTRAL_* */
  const double* chi2;  /* [P][F], table mode with the Matern draw only */
} cmoe_rff_opts;

/* cmoe_gp_sample_rff_optima with options; opts == NULL gives cmoe_gp_sample_rff_optima's results bit for bit.  An
 * unknown opts->spectral -> CMOE_ERR_INVALID_VALUE (after the size checks). */
int cmoe_gp_sample_rff_optima_ex(const cmoe_gp* gp, int num_features, int num_points, const double* domain_bounds,
                                 const double* grid, int num_grid, uint64_t seed, uint64_t first_draw,
                                 const cmoe_rff_table* table, const cmoe_rff_opts* opts, double* points, double* values,
                                 double* omega, double* b, double* theta, int* info);

/* sample_gp_with_random_features (random_features.py:29-133): the sample functions of num_points draws without the grid
 * and the local optimiser.  omega[P][F][d], b[P][F] and theta[P][F] (none may be NULL) are bit for bit those
 * cmoe_gp_sample_rff_optima_ex returns for the same (gp, F, P, seed, first_draw, table, opts).  Errors as for
 * cmoe_gp_sample_rff_optima_ex, without those of the grid and the bounds. */
int cmoe_gp_sample_rff_functions(const cmoe_gp* gp, int num_features, int num_points, uint64_t seed,
                                 uint64_t first_draw, const cmoe_rff_table* table, const cmoe_rff_opts* opts,
                                 double* omega, double* b, double* theta, int* info);

/* The g[num_draws][num_features] of the Matern draw for Philox draws first_draw .. first_draw + num_draws - 1, as
 * rff_features_kernel forms them (so that a table can replay a Philox run, as cmoe_philox_normals does for the normals).
 * num_draws <= 65535. */
int cmoe_rff_chi2_draws(uint64_t seed, uint64_t first_draw, int num_draws, int num_features, double* out, int device);

/* The sample functions' values and gradients (the reference's wrapper(x, gradient)):
 *   values[p][j]   = c sum_f theta[p][f] cos(omega[p][f] . x_pj + b[p][f]),
 *   grads[p][j][k] = -c sum_f theta[p][f] sin(omega[p][f] . x_pj + b[p][f]) omega[p][f][k],
 * with c = sqrt(2 alpha / F) as the sampler uses it.  points are [num_points][dim], shared by all functions
 * (per_function = 0), or [num_functions][num_points][dim] (per_function != 0).  values or grads may be NULL, not both.
 * Each sum runs over the features in ascending order, one point per thread, so a result depends only on its function
 * and its point, not on num_functions, num_points, the chunking or whether the other output is requested; the values
 * are the sampler's grid-stage arithmetic, bit for bit.  Runs in chunks of (functions x points) that fit 2 GiB.
 * Errors (before any device work): CMOE_ERR_BOUNDS unless dim in [1, 32], num_features, num_functions, num_points >= 1
 * and one function's features and one point fit in 2 GiB; CMOE_ERR_INVALID_VALUE for NULL inputs, both outputs NULL,
 * or non-finite omega, b, theta, c or points. */
int cmoe_rff_evaluate(int dim, int num_features, int num_functions, const double* omega, const double* b,
                      const double* theta, double c, const double* points, int num_points, int per_function,
                      double* values, double* grads, int device, int* info);

/* ---- lower-confidence-bound batch selection ----------------------------------------------------------------------
 * lower_confidence_bound_optimization (moe/optimal_learning/python/cpp_wrappers/lower_confidence_bound.py:52-80) in one
 * call.  candidates [num_candidates][dim].  mu(x) is the value mean, sigma(x) the square root of the value variance.
 *   selected[0] = argmin(mu - sigma) (first occurrence); the satisfied set is {x : mu - sigma <= min(mu + sigma)} in
 *   candidate order; selected[i], i = 1 .. num_to_sample - 1, = argmax over the satisfied set (first occurrence) of
 *   sigma on the GP to which selected[0 .. i-1] have been added as noisy observations with the GP's own derivative rows
 *   and per-type noise (the reference's refit; here a bordered update, the handle is not modified).  A point may be
 *   selected again.  selected[num_to_sample] holds indices into `candidates`.
 * mean[num_candidates], sd[num_candidates] (the round-0 mu and sigma) and *num_satisfied may be NULL.
 * Candidates are screened in chunks of max(1, floor(2^31 / (8 n))) (n = num_sampled (1 + num_derivatives)) in the
 * handle's sampling workspace; a candidate's mu and sigma do not depend on the chunking.
 * Errors: a candidate variance that is not > 1e-16 (round 0, or on a surviving candidate in a later round) ->
 * CMOE_ERR_SINGULAR, *info = 1, the lowest such candidate index in cmoe_last_error(); a pivot of the enlarged matrix
 * that is not > 1e-16 -> CMOE_ERR_SINGULAR, *info = its leading minor counted from the GP's n rows, as
 * cmoe_gp_add_sampled_points counts it.  Limits (CMOE_ERR_BOUNDS): (num_to_sample - 1)(1 + num_derivatives) <= 1024,
 * and num_satisfied (num_to_sample - 1)(1 + num_derivatives) <= 2^28 (checked after the screen).  Non-finite
 * candidates -> CMOE_ERR_INVALID_VALUE. */
int cmoe_lcb_select(const cmoe_gp* gp, const double* candidates, int num_candidates, int num_to_sample, int* selected,
                    double* mean, double* sd, int* num_satisfied, int* info);

/* ---- heuristic batch EI (DESIGN.md K20) ------------------------------------------------------------------------
 * Replaces the reference's ComputeHeuristicPointsToSample loop (gpp_python_expected_improvement.cpp:602-659, the
 * policies :445-486): q rounds of one-point EI optimisation, each point fed back to a private copy of the GP with an
 * estimated value.  Round r is cmoe_multistart_ei with q = 1, p = 0 and the start block starts[r] on the GP extended
 * by rounds 0..r-1 (gd == NULL: the random search of the kNull branch, best -1 and strict `<` over the screen); its
 * restarted descent runs on the device in one launch per round.  After round r the chosen point is appended with the
 * policy's value and noise_variance on its diagonal:
 *   Constant Liar      value = policy->value (the lie)
 *   Kriging Believer   value = mu(x) + policy->value * sqrt(max(sigma^2(x), 0)), mu and sigma^2 (no noise) of round r
 * best_so_far is held fixed over the rounds.  The caller's GP is never modified.  Outputs: points [q][dim],
 * fantasy_values [q], ei_values [q] (the chosen point's 1-EI in its round, -1 if no start was found) and found [q]
 * (each may be NULL except points).  CMOE_ERR_BOUNDS: q < 1, num_starts < 1, a GP with derivative observations,
 * max_num_steps > 2^20, an empty box, or more than the descent's shared-memory rows (num_sampled + q - 1, about 13500
 * on an H100).  CMOE_ERR_INVALID_VALUE: a NULL argument, an unknown policy, a non-finite value or noise_variance < 0.
 * A fantasy that makes the factor singular: CMOE_ERR_SINGULAR, *info = its leading minor. */
#define CMOE_ESTIMATION_CONSTANT_LIAR 0
#define CMOE_ESTIMATION_KRIGING_BELIEVER 1
typedef struct cmoe_estimation_policy {
  int policy;            /* CMOE_ESTIMATION_* */
  double value;          /* Constant Liar: the lie; Kriging Believer: std_deviation_coef (finite) */
  double noise_variance; /* >= 0: noise of each fantasy row */
} cmoe_estimation_policy;
int cmoe_heuristic_ei(const cmoe_gp* gp, const cmoe_estimation_policy* policy, const cmoe_gd_params* gd,
                      const double* domain_bounds, const double* starts, int num_starts, int q, double best_so_far,
                      double* points, double* fantasy_values, double* ei_values, int* found, int* info);

/* ---- q-EI Monte Carlo, batched over candidates ----------------------------------------------------------------
 * Replaces ExpectedImprovementEvaluator::ComputeExpectedImprovement / ComputeGradExpectedImprovement
 * (gpp_math.cpp:1991-2126); Python boundary compute_expected_improvement / compute_grad_expected_improvement /
 * evaluate_EI_at_point_list (gpp_python_expected_improvement.cpp:44-109, 401-441).
 * candidates = [num_candidates][q][dim]; points_being_sampled = [p][dim] shared by all candidates.
 * Normals: Philox4x32-10 + Box-Muller keyed by `seed` (same stream for every candidate = common random numbers,
 * the device analogue of ResetToMostRecentSeed, gpp_random.cpp:130-135), or, if normals_table != NULL, the table
 * is replayed exactly like NormalRNGSimulator (gpp_random.hpp:314): (q+p) normals per iteration.
 * ei[num_candidates]; grad_ei[num_candidates][q][dim] or NULL. */
int cmoe_ei_eval(const cmoe_gp* gp, const double* candidates, int num_candidates, int q,
                 const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                 const double* normals_table, double* ei, double* grad_ei, int* info);
/* cmoe_ei_eval for 1 <= U = q + p <= 8192 (CMOE_ERR_BOUNDS past it, or when the num_mc U normals exceed 2 GiB), same
 * arguments, same draws: sample s uses the normals 2k, 2k+1 of Philox call (seed, draw s, k), or row s of the
 * [num_mc][U] table.  At U <= 96 the two calls differ only in summation order.  y - mu = C W runs as FP64 tensor-core
 * tiles; the gradient is taken in reverse mode through the Cholesky factor (DESIGN.md K16), so no q U^2 dim tensor is
 * formed: O(n U + U^2) device memory per candidate.  The call's device workspace (the num_mc U normals and chunks of
 * candidates) is at most 2 GiB, kept on the handle; the table, when given, is uploaded beside it.  A candidate's result
 * does not depend on the batch or the chunking.  A failed factorisation -> CMOE_ERR_SINGULAR, *info = leading minor of the first failing
 * candidate.  The multistart q-EI drivers (cmoe_multistart_ei(_ex), cmoe_ei_gradient_descent) evaluate through this
 * call's stages when q + p > CMOE_MAX_SET_ROWS and through cmoe_ei_eval's otherwise. */
int cmoe_ei_eval_large(const cmoe_gp* gp, const double* candidates, int num_candidates, int q,
                       const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                       const double* normals_table, double* ei, double* grad_ei, int* info);

/* ---- q-KG / d-KG Monte Carlo, batched over candidates -----------------------------------------------------------
 * Replaces KnowledgeGradientEvaluator::ComputeKnowledgeGradient / ComputeGradKnowledgeGradient
 * (gpp_knowledge_gradient_optimization.cpp:69-227) including KnowledgeGradientState::PreCompute (:292-317),
 * ComputeOptimalPosteriorMean (:420-472), the line-search gradient descent (gpp_optimization.hpp:708-828) and
 * TensorProductDomain::LimitUpdate (gpp_domain.cpp:64-104); Python boundary compute_knowledge_gradient /
 * compute_grad_knowledge_gradient / evaluate_KG_at_point_list (gpp_python_knowledge_gradient.cpp:77-154, 352-397).
 * inner_bounds = [dim-num_fidelity][2]; discrete_pts = [num_pts][dim-num_fidelity].
 * Normals as for EI but (q+p)(1+g) per EVEN iteration; odd iterations are antithetic (:88-97).
 * kg[num_candidates]; grad_kg[num_candidates][q][dim] or NULL; stats may be NULL. */
int cmoe_kg_eval(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds,
                 const double* discrete_pts, int num_pts, const double* candidates, int num_candidates, int q,
                 const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                 const double* normals_table, double* kg, double* grad_kg, cmoe_kg_stats* stats, int* info);
/* Largest Q = (q + p)(1 + num_derivatives) of cmoe_kg_eval_large. */
#define CMOE_MAX_KG_LARGE_ROWS 1024
/* cmoe_kg_eval for 1 <= Q = (q + p)(1 + g) <= CMOE_MAX_KG_LARGE_ROWS: same arguments, same draws, same argument checks
 * (g <= 31, distinct partials past 8).  The fantasised posterior of each sample is a GP mean over the training points
 * followed by the union points with per-sample weights (DESIGN.md K17), so the union size only sizes dense products;
 * the inner optimiser is cmoe_kg_eval's line-search descent, and the gradient is taken in reverse mode through the union's
 * Cholesky factor.  The call's device workspace (the draws, the inner optimiser's scratch, chunks of candidates) is at
 * most 2 GiB, kept on the handle; a candidate's value and gradient do not depend on num_candidates or the chunking.
 * CMOE_ERR_BOUNDS, before any device work, when one candidate's workspace does not fit.  A singular union covariance -> CMOE_ERR_SINGULAR, *info = leading minor of
 * the first failing candidate.  stats: mc_samples exact, posterior_evals and line_search_steps as cmoe_kg_stats,
 * point_evals and line_batches what this call's kernel executed.  num_mc <= 65535 * 64.  The multistart q-KG drivers
 * (cmoe_multistart_kg(_ex), cmoe_kg_gradient_descent(_ex)) and the ensemble calls (cmoe_kg_eval_mcmc,
 * cmoe_multistart_kg_mcmc, cmoe_kg_gradient_descent_mcmc) evaluate through these stages when (q + p)(1 + g) >
 * CMOE_MAX_KG_ROWS and through the plans / cmoe_kg_eval otherwise.  The cmoe_kg_plan_* API keeps the
 * CMOE_MAX_KG_ROWS bound of cmoe_kg_eval. */
int cmoe_kg_eval_large(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds,
                       const double* discrete_pts, int num_pts, const double* candidates, int num_candidates, int q,
                       const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                       const double* normals_table, double* kg, double* grad_kg, cmoe_kg_stats* stats, int* info);

/* ---- device-resident plan for the q-KG path (what bench.py times as `value`) ------------------------------------
 * Same computation as cmoe_kg_eval, split so that inputs can be made resident in HBM before the timed region:
 *   create -> upload (H2D of candidates) -> run (kernels only, asynchronous on the plan's stream) -> download (D2H).
 * cmoe_kg_plan_elapsed_ms returns CUDA-event time of the last run; cmoe_kg_plan_kernel_ms the time spent in the
 * fused MC kernel alone (events recorded around it on the launching stream); *_launches the kernel launches issued. */
typedef struct cmoe_kg_plan cmoe_kg_plan;
int cmoe_kg_plan_create(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds,
                        const double* discrete_pts, int num_pts, int max_candidates, int q,
                        const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                        int want_grad, cmoe_kg_plan** plan_out);
void cmoe_kg_plan_destroy(cmoe_kg_plan* plan);
/* Optional table replay (NormalRNGSimulator semantics): ((num_mc+1)/2)*(q+p) normals; replaces the Philox stream. */
int cmoe_kg_plan_set_table(cmoe_kg_plan* plan, const double* normals_table, int table_len);
/* Reference-driver compatibility: the multistart drivers of the reference evaluate every start and every descent step
 * through ONE KnowledgeGradientState per thread, constructed with the first start; SetCurrentPoint refreshes the GP
 * quantities but NOT discretized_set (gpp_knowledge_gradient_optimization.cpp:233-243 vs :259-261), so the set the
 * per-sample inner optimiser starts from keeps the FIRST start's q points instead of the current ones.  Passing those
 * q points here ([q][dim]; NULL clears) makes a plan evaluate exactly that; cmoe_multistart_kg(_ex) does it itself. */
int cmoe_kg_plan_set_stale_union(cmoe_kg_plan* plan, const double* points_to_sample);
int cmoe_kg_plan_upload(cmoe_kg_plan* plan, const double* candidates, int num_candidates);
int cmoe_kg_plan_run(cmoe_kg_plan* plan);
int cmoe_kg_plan_sync(cmoe_kg_plan* plan, int* info);
int cmoe_kg_plan_download(cmoe_kg_plan* plan, double* kg, double* grad_kg, cmoe_kg_stats* stats);
int cmoe_kg_plan_timings(const cmoe_kg_plan* plan, double* total_ms, double* mc_kernel_ms, int* launches);

/* ---- multistart optimisation (the data-parallel axis) -------------------------------------------------------------
 * Replaces ComputeKGOptimalPointsToSampleViaMultistartGradientDescent (gpp_knowledge_gradient_optimization.hpp:859-935):
 * KG at every start -> keep the best 20 (hard-coded `k = 20`, :901) -> restarted gradient descent with LimitUpdate on
 * each (gpp_optimization.hpp:620-705, 1144-1185) -> strict-> argmax (gpp_optimization.hpp:1511, 1540).
 * Python boundary multistart_knowledge_gradient_optimization (gpp_python_knowledge_gradient.cpp:243-304).
 * This entry point runs the whole pipeline on one GPU.  With one process per GPU the same pipeline is sharded over
 * the starts by cornell_moe_b200/multigpu.py: cmoe_kg_eval on this rank's starts -> one all-gather of the values ->
 * identical top-20 on every rank -> cmoe_kg_gradient_descent on this rank's share -> one all-gather -> arg-max.
 * start_values (may be NULL) receives KG at every start.
 * best_value / best_point[q*dim] / found_flag follow OptimizationIOContainer (gpp_optimization.hpp:511). */
int cmoe_multistart_kg(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer, const cmoe_gd_params* inner,
                       const double* domain_bounds, const double* inner_bounds, const double* discrete_pts, int num_pts,
                       const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                       int num_mc, double best_so_far, uint64_t seed, double* start_values, double* best_point,
                       double* best_value, int* found_flag, int* info);
/* EI twin: ComputeOptimalPointsToSampleViaMultistartGradientDescent (gpp_math.hpp:1683-1802);
 * Python boundary multistart_expected_improvement_optimization (gpp_python_expected_improvement.cpp:221-276). */
int cmoe_multistart_ei(const cmoe_gp* gp, const cmoe_gd_params* outer, const double* domain_bounds,
                       const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                       int num_mc, double best_so_far, uint64_t seed, double* start_values, double* best_point,
                       double* best_value, int* found_flag, int* info);

/* Extended forms of the two drivers above (opts may be NULL = plain call):
 *   normals_table / table_len — standard normals replayed for every evaluation exactly like the reference's
 *     NormalRNG after ResetToMostRecentSeed (every q-KG / q-EI evaluation of a driver call rewinds its generator,
 *     gpp_knowledge_gradient_optimization.cpp:81,164, gpp_math.cpp:2011,2076): ((num_mc+1)/2)*(q+p)*(1+g) values for
 *     q-KG, num_mc*(q+p) for q-EI.  With the table drawn from a NormalRNG of the same seed the device path and
 *     ComputeKGOptimalPointsToSampleViaMultistartGradientDescent consume identical draws.
 *   devices / num_devices — the reference's parallel axis (OpenMP threads over starts, gpp_optimization.hpp:1472-1546)
 *     inside the call: the GP is replicated on every listed GPU (one host thread and stream set per device), starts
 *     are strided over the devices for the screening pass and for the gradient descent of the kept 20, values are
 *     gathered on the host.  Every start is evaluated by the same kernels with the same seed wherever it runs, so the
 *     result is bit-identical to the single-device call. */
typedef struct cmoe_multistart_opts {
  const double* normals_table;
  size_t table_len;
  const int* devices;
  int num_devices;
  int domain_type; /* CMOE_DOMAIN_TENSOR_PRODUCT (0) or CMOE_DOMAIN_SIMPLEX (1): the outer optimiser's domain */
  /* q-KG only.  0 (default): bug-compatible with the reference driver — the inner optimiser's discretisation set keeps
   * the q points of `stale_union` (NULL = the first start), see cmoe_kg_plan_set_stale_union.  1: every evaluation uses
   * its own current points (what a freshly constructed state, e.g. compute_knowledge_gradient, does). */
  int fresh_discretisation;
  const double* stale_union; /* [q][dim] or NULL */
} cmoe_multistart_opts;
/* DomainTypes, gpp_python_common.cpp:201-240.  CMOE_DOMAIN_SIMPLEX = unit simplex intersected with the box
 * (SimplexIntersectTensorProductDomain, gpp_domain.cpp:107-289): implemented for the q-EI drivers; q-KG needs the same
 * domain for its per-sample inner optimiser, which the fused kernel only has for the tensor product — it reports
 * CMOE_ERR_INVALID_VALUE. */
#define CMOE_DOMAIN_TENSOR_PRODUCT 0
#define CMOE_DOMAIN_SIMPLEX 1
/* One LimitUpdate of the outer optimiser's domain (host arithmetic, no device needed): update[dim] is limited in place.
 * TensorProductDomain::LimitUpdate gpp_domain.cpp:64-104 / SimplexIntersectTensorProductDomain::LimitUpdate :234-289. */
int cmoe_limit_update(int domain_type, const double* domain_bounds, int dim, double max_relative_change,
                      const double* current_point, double* update);
int cmoe_multistart_kg_ex(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer, const cmoe_gd_params* inner,
                          const double* domain_bounds, const double* inner_bounds, const double* discrete_pts,
                          int num_pts, const double* starts, int num_starts, int q, const double* points_being_sampled,
                          int p, int num_mc, double best_so_far, uint64_t seed, const cmoe_multistart_opts* opts,
                          double* start_values, double* best_point, double* best_value, int* found_flag, int* info);
int cmoe_multistart_ei_ex(const cmoe_gp* gp, const cmoe_gd_params* outer, const double* domain_bounds,
                          const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                          int num_mc, double best_so_far, uint64_t seed, const cmoe_multistart_opts* opts,
                          double* start_values, double* best_point, double* best_value, int* found_flag, int* info);

/* Restarted gradient descent from given starts only (the second half of the multistart drivers); used by the
 * multi-GPU host layer after the global top-20 has been agreed on.  values_out[num_starts], points_out[num_starts][q*dim]. */
/* (cmoe_kg_gradient_descent_ex: same, `stale_union` ([q][dim] or NULL) as in cmoe_multistart_opts — the sharded host
 * layer passes the global first start so that every rank reproduces the one-process driver.) */
int cmoe_kg_gradient_descent(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer,
                             const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                             const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                             const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                             double* values_out, double* points_out, int* info);
int cmoe_kg_gradient_descent_ex(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer,
                                const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                                const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                                const double* points_being_sampled, int p, int num_mc, double best_so_far,
                                uint64_t seed, const double* stale_union, double* values_out, double* points_out,
                                int* info);
int cmoe_ei_gradient_descent(const cmoe_gp* gp, const cmoe_gd_params* outer, const double* domain_bounds,
                             const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                             int num_mc, double best_so_far, uint64_t seed, double* values_out, double* points_out,
                             int* info);

/* Closed-form one-point EI and its gradient at num_points points (OnePotentialSampleExpectedImprovementEvaluator,
 * gpp_math.cpp:2196-2253) — what EvaluateEIAtPointList and the multistart driver use when q = 1, p = 0
 * (gpp_math.cpp:2317, gpp_math.hpp:1703-1749).  values[num_points]; grads[num_points][dim] or NULL. */
int cmoe_ei_analytic(const cmoe_gp* gp, const double* points, int num_points, double best_so_far, double* values,
                     double* grads, int* info);

/* ---- ensembles of GPs: "MCMC-averaged" acquisition, one GP per hyper-parameter sample ----------------------------
 * The reference's GaussianProcessMCMC is a list of GPs over the same data (gpp_knowledge_gradient_mcmc_optimization.cpp:
 * 24-48); here it is an array of cmoe_gp handles (same dim / derivative observations / device).
 * discrete_pts[num_gp][num_pts][dim-num_fidelity] and best_so_far[num_gp] are per member, as in the reference.
 *
 * cmoe_kg_eval_mcmc      KnowledgeGradientMCMCEvaluator::Compute{,Grad}KnowledgeGradient (..mcmc_optimization.cpp:137-180)
 *                        = mean_m KG_m / cost,  cost = max_i prod_{j>=dim-nf} x_ij (1 when num_fidelity = 0, :87-104);
 *                        gradient by the quotient rule (:162-180).  Python: compute_knowledge_gradient_mcmc,
 *                        compute_grad_knowledge_gradient_mcmc, evaluate_KG_mcmc_at_point_list
 *                        (gpp_python_knowledge_gradient_mcmc.cpp:80-198, 326-384).
 * cmoe_ei_eval_mcmc      ExpectedImprovementMCMCEvaluator (gpp_expected_improvement_mcmc_optimization.cpp:47-85):
 *                        mean_m of the Monte-Carlo q-EI; with analytic_single != 0 and q = 1, p = 0 the closed-form
 *                        1-EI per member instead, as EvaluateEIMCMCAtPointList does (..mcmc_optimization.cpp:251).  Python: compute_expected_improvement_mcmc, ..grad.., evaluate_EI_mcmc_at_point_list.
 * cmoe_multistart_*_mcmc ComputeKGMCMCOptimalPointsToSampleViaMultistartGradientDescent (..mcmc_optimization.hpp:665-745)
 *                        and ComputeEIMCMC... (gpp_expected_improvement_mcmc_optimization.hpp:860-980): screen, top-20,
 *                        restarted gradient descent, strict-> arg-max (initial best -inf for KG, 0.0 for EI; the EI
 *                        driver uses analytic 1-EI per member when q = 1, p = 0).
 * normals_table: as in cmoe_kg_eval / cmoe_ei_eval (NULL = Philox stream keyed by seed); shared by every member.
 *
 * Sizes: q-KG up to (q + p)(1 + g) = CMOE_MAX_KG_ROWS runs each member's cmoe_kg_eval (the drivers: its plans); past
 * it, up to CMOE_MAX_KG_LARGE_ROWS, each member's cmoe_kg_eval_large with num_mc, g and the inner optimiser bounded as
 * there.
 * q-EI up to q + p = CMOE_MAX_SET_ROWS runs each member's cmoe_ei_eval; past it, up to CMOE_MAX_LARGE_SET_ROWS, each
 * member's cmoe_ei_eval_large.  Past the per-set bounds the draws are made once per evaluation, the members run
 * together on their own streams, and the evaluation's large-stage workspace is at most 2 GiB per device whatever
 * num_gp is (kept on gps[0]'s handle); each member's value and gradient are those of its single large call, summed in
 * member order (a one-member sum is the member's own result).  q + p past the large bound -> CMOE_ERR_BOUNDS before
 * any handle is read.  A singular union ->
 * CMOE_ERR_SINGULAR, *info = leading minor of the first failing candidate of the first failing member. */
int cmoe_kg_eval_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* inner,
                      const double* inner_bounds, const double* discrete_pts, int num_pts, const double* candidates,
                      int num_candidates, int q, const double* points_being_sampled, int p, int num_mc,
                      const double* best_so_far, uint64_t seed, const double* normals_table, double* values,
                      double* grads, int* info);
int cmoe_ei_eval_mcmc(const cmoe_gp* const* gps, int num_gp, const double* candidates, int num_candidates, int q,
                      const double* points_being_sampled, int p, int num_mc, const double* best_so_far, uint64_t seed,
                      const double* normals_table, int analytic_single, double* values, double* grads, int* info);
int cmoe_multistart_kg_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* outer,
                            const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                            const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                            const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                            uint64_t seed, double* start_values, double* best_point, double* best_value,
                            int* found_flag, int* info);
int cmoe_multistart_ei_mcmc(const cmoe_gp* const* gps, int num_gp, const cmoe_gd_params* outer,
                            const double* domain_bounds, const double* starts, int num_starts, int q,
                            const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                            uint64_t seed, double* start_values, double* best_point, double* best_value,
                            int* found_flag, int* info);

/* The restarted gradient descent of the MCMC drivers alone (RestartedGradientDescentKGMCMCOptimization,
 * gpp_knowledge_gradient_mcmc_optimization.hpp:576-600, and its EI twin): every start is optimised, no top-20 selection.
 * values_out[num_starts], points_out[num_starts][q][dim].  Used by the multi-GPU layer, which shards the kept starts. */
int cmoe_kg_gradient_descent_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* outer,
                                  const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                                  const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                                  const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                                  uint64_t seed, double* values_out, double* points_out, int* info);
int cmoe_ei_gradient_descent_mcmc(const cmoe_gp* const* gps, int num_gp, const cmoe_gd_params* outer,
                                  const double* domain_bounds, const double* starts, int num_starts, int q,
                                  const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                                  uint64_t seed, double* values_out, double* points_out, int* info);

/* posterior_mean_optimization (gpp_python_knowledge_gradient.cpp:306-350): ComputeOptimalPosteriorMean
 * (gpp_knowledge_gradient_optimization.cpp:420-472) from ONE start on the un-fantasised GP — line-search gradient
 * descent on -mu(x) over the dim-num_fidelity free coordinates (fidelity coordinates pinned to 1.0).
 * best_point[dim-num_fidelity]; best_value = -min mu found (the reference's best_function_value).
 * With max_num_restarts <= 0 nothing is written and *found_flag = 0, as in the reference (:424-426). */
int cmoe_posterior_mean_optimization(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* params,
                                     const double* domain_bounds, const double* initial_guess, double* best_point,
                                     double* best_value, int* found_flag);

/* ---- ensemble posterior mean: the recommendation step of the MCMC loop ---------------------------------------------
 * PosteriorMeanMCMC (moe/optimal_learning/python/cpp_wrappers/knowledge_gradient_mcmc.py:25-157) over an ensemble
 * (gps[num_gp], as for the *_mcmc calls above): f(x) = -(1/M) sum_m mu_m(x), the members summed in ascending order and
 * then divided by M; fidelity coordinates are pinned to 1.0.  Members may have different numbers of sampled points.
 *
 * cmoe_posterior_mean_mcmc   f at num_points points [num_points][dim-num_fidelity] in one call (the screening loop of
 *                            examples/main.py:243-252): values[num_points]; grads[num_points][dim-num_fidelity] (grad f
 *                            on the free coordinates) or NULL; member_values[num_gp][num_points] = -mu_m or NULL.
 * cmoe_posterior_mean_mcmc_optimization
 *                            The Python GradientDescentOptimizer (python_version/optimization.py:392-528) on f from every
 *                            start (MultistartOptimizer, :565-610): for k = 1..max_num_steps, s = pre_mult k^-gamma grad f,
 *                            each coordinate limited by TensorProductDomain.compute_update_restricted_to_domain
 *                            (python_version/domain.py:158-202, no half-step fallback), x += s; then the Polyak-Ruppert
 *                            average over _get_averaging_range (:415-442).  points_out[num_starts][dim-num_fidelity] and
 *                            values_out[num_starts] (f at the average) may be NULL.  best: strict > in start order from
 *                            -inf, best_point starting as starts[0].  max_num_restarts, tolerance and num_multistarts are
 *                            ignored, as the Python optimiser ignores them.  max_num_steps < 1 (where the Python optimiser
 *                            averages an empty range), an empty box, num_fidelity outside [0, dim) and num_starts < 1 are
 *                            CMOE_ERR_BOUNDS.  One CTA per start; a start's result does not depend on the batch. */
int cmoe_posterior_mean_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const double* points,
                             int num_points, double* values, double* grads, double* member_values, int* info);
int cmoe_posterior_mean_mcmc_optimization(const cmoe_gp* const* gps, int num_gp, int num_fidelity,
                                          const cmoe_gd_params* params, const double* domain_bounds,
                                          const double* starts, int num_starts, double* points_out,
                                          double* values_out, double* best_point, double* best_value, int* info);

/* ---- per-member posterior-mean optima: the discretisation step of the MCMC q-KG loop ---------------------------------
 * examples/main.py:172-197 and KnowledgeGradientMCMC's best_so_far (cpp_wrappers/knowledge_gradient_mcmc.py:386-393) for
 * every member of an ensemble (gps[num_gp], same rules as cmoe_posterior_mean_mcmc: members may have different numbers
 * of sampled points, fidelity coordinates are pinned to 1.0, ps = dim - num_fidelity free coordinates) in one call.
 * For every member m, independently:
 *   1. screen   mu_m at points[num_points][ps] (shared by the members) or, with points_per_member != 0, at the member's
 *               own list points[num_gp][num_points][ps]; with include_sampled != 0 also at the first ps coordinates of
 *               the member's N_m sampled points, which follow the given points in the member's screen list.
 *   2. argmin   the least value and its first index (numpy.argmin): screen_min[m], start_index[m], start x0_m.  The
 *               screened values are bit for bit -member_values of cmoe_posterior_mean_mcmc on the same points.
 *   3. descent  ComputeOptimalPosteriorMean from x0_m: what cmoe_posterior_mean_optimization computes, with the same
 *               params and domain_bounds[ps][2].  A member with N_m (1 + g) >= 128 rows spreads them over up to 8 warps
 *               (the count depends on the member's rows only) and adds the warps' sums in ascending order, so its end
 *               point agrees with the single-GP call to rounding; a smaller member returns that call's bits.
 *   4. fallback if mu_m at the end point is greater than screen_min[m] the optimum is x0_m and kept_start[m] = 1.
 *               max_num_restarts <= 0: the reference's descent returns without moving, so the optimum is x0_m and
 *               kept_start[m] = 1 (the single-GP call writes nothing then; here the screen always gives an answer).
 *   5. baseline discrete_pts[m] = [shared_discrete[num_shared][ps] ; optimum_m] and best_so_far[m] = the least mu_m over
 *               it (values as cmoe_gp_posterior returns them): the discrete_pts (num_pts = num_shared + 1) and
 *               best_so_far arguments of cmoe_kg_eval_mcmc / cmoe_multistart_kg_mcmc.  shared_discrete may be NULL with
 *               num_shared = 0.
 * A member's result depends on that member, its screen points, params and the bounds only: not on num_gp, on the other
 * members, or on how the screen is split into chunks.  The screen runs in chunks whose given points and values fit a
 * 64 MiB workspace (at least one screen index per chunk); num_gp (num_points + N) is not bounded by a grid dimension,
 * num_points + N must fit an int.  A screen point outside the box is allowed (the reference does not check).
 * Outputs (all but optima may be NULL): optima[num_gp][ps]; optimum_means[num_gp] = mu_m at the returned point;
 * start_index[num_gp]; kept_start[num_gp]; screen_min[num_gp]; discrete_pts[num_gp][num_shared + 1][ps];
 * best_so_far[num_gp].
 * Errors, all before any device work: NULL params / domain_bounds / points / optima (or shared_discrete with
 * num_shared > 0) and non-finite points are CMOE_ERR_INVALID_VALUE; num_points < 1, num_shared < 0, num_fidelity outside
 * [0, dim), max_num_steps > 2^20 and an empty box are CMOE_ERR_BOUNDS; ensemble mismatches as in the other *_mcmc calls. */
int cmoe_posterior_mean_optima_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity,
                                    const cmoe_gd_params* params, const double* domain_bounds, const double* points,
                                    int num_points, int points_per_member, int include_sampled,
                                    const double* shared_discrete, int num_shared, double* optima,
                                    double* optimum_means, int* start_index, int* kept_start, double* screen_min,
                                    double* discrete_pts, double* best_so_far, int* info);

/* ---- building blocks exposed for parity tests and micro-benchmarks ------------------------------------------------ */
/* Covariance build alone on device-resident inputs: returns device time (usec) of `repeats` builds of the n*n matrix. */
int cmoe_bench_cov_build(const cmoe_gp* gp, int repeats, double* usec_per_build);
/* Blocked Cholesky alone (re-factors a fresh copy of K each repeat). */
int cmoe_bench_cholesky(const cmoe_gp* gp, int repeats, double* usec_per_factor);
/* The batched Cholesky of cmoe_gp_sample_joint alone on num_mats device-resident Q x Q matrices (mats
 * [num_mats][Q*Q] column-major, uploaded once), against a loop of the single-matrix blocked Cholesky over the same
 * matrices: device time per call of each, averaged over `repeats` after one warm-up. */
int cmoe_bench_cholesky_batched(const double* mats, int num_mats, int Q, int repeats, int device, double* usec_batched,
                                double* usec_loop, int* info);
/* Measured FP64 peaks of this GPU: tflops[0] = DFMA vector pipe, tflops[1] = DMMA tensor pipe (m8n8k4). */
int cmoe_bench_fp64_peaks(int device, double* tflops);
/* tflops[0] = total FP64 TFLOP/s when every warp interleaves DFMA and DMMA 1:1 by flops (do the vector pipe and the
 * tensor sub-pipe overlap?). */
int cmoe_bench_fp64_mixed(int device, double* tflops);
/* latency microbenchmarks behind the Cholesky pivot chain: out[11] (cycles), see microbench_chain.cu */
int cmoe_bench_chain_latencies(int device, double* out);
/* In-place lower Cholesky of a host matrix through the device path (ComputeCholeskyFactorL, gpp_linear_algebra.cpp:109). */
int cmoe_cholesky(int n, double* a, int device, int* info);
/* Solve (L L^T) X = B for nrhs right-hand sides (CholeskyFactorLMatrixMatrixSolve, gpp_linear_algebra.hpp:247). */
int cmoe_potrs(int n, int nrhs, const double* chol, double* x, int device);
/* Philox4x32-10 + Box-Muller normals exactly as the kernels draw them: out[num_draws][per_draw]. */
int cmoe_philox_normals(uint64_t seed, uint64_t first_draw, int num_draws, int per_draw, double* out, int device);

#ifdef __cplusplus
}
#endif
#endif /* CMOE_B200_H_ */

// `GPP`: drop-in for the reference's Boost.Python module `moe.build.GPP` (gpp_python.cpp:453-600) for the GP-posterior
// + Monte-Carlo acquisition hot path, built with pybind11 (Boost.Python is not available) on top of the C ABI in
// include/cmoe_b200.h.  Same names, positional signatures, flat-list conventions, status-dict keys and exception
// classes as the reference, so `moe.optimal_learning.python.cpp_wrappers.*` can `import ... GPP as C_GP` unchanged:
//
//   GaussianProcess(hyperparameters, points_sampled, points_sampled_value, noise_variance, derivatives,
//                   num_derivatives, dim, num_sampled)                     gpp_python_gaussian_process.cpp:42-62, 295
//     .compute_mean_of_points / compute_mean_of_additional_points / compute_grad_mean_of_points /
//     .compute_variance_of_points / compute_cholesky_variance_of_points / compute_grad_variance_of_points /
//     .compute_grad_cholesky_variance_of_points / add_sampled_points / ...   :64-253, 456-463
//   compute_expected_improvement, compute_grad_expected_improvement, multistart_expected_improvement_optimization,
//   evaluate_EI_at_point_list                                             gpp_python_expected_improvement.cpp:44-441
//   heuristic_expected_improvement_optimization, ConstantLiarEstimationPolicy, KrigingBelieverEstimationPolicy
//                                                                         gpp_python_expected_improvement.cpp:445-659
//   compute_posterior_mean, compute_grad_posterior_mean, compute_knowledge_gradient, compute_grad_knowledge_gradient,
//   multistart_knowledge_gradient_optimization, posterior_mean_optimization, evaluate_KG_at_point_list
//                                                                         gpp_python_knowledge_gradient.cpp:44-397
//   GaussianProcessMCMC, compute_{,grad_}knowledge_gradient_mcmc, multistart_knowledge_gradient_mcmc_optimization,
//   evaluate_KG_mcmc_at_point_list                                        gpp_python_knowledge_gradient_mcmc.cpp:49-384
//   compute_{,grad_}expected_improvement_mcmc, multistart_expected_improvement_mcmc_optimization,
//   evaluate_EI_mcmc_at_point_list                                        gpp_python_expected_improvement_mcmc.cpp:46-300
//   compute_posterior_mean_of_points, compute_{,grad_}posterior_mean_mcmc_of_points, posterior_mean_mcmc_optimization,
//   posterior_mean_optima_mcmc,
//   sample_hyperparameters_mcmc                                           batched forms, not in the reference module
//   GradientDescentParameters, NewtonParameters, RandomnessSourceContainer, OptimizerTypes, DomainTypes,
//   LogLikelihoodTypes                                                    gpp_python_common.cpp:201-370
//   OptimalLearningException, BoundsException, InvalidValueException, SingularMatrixException   gpp_python.cpp:189-206
//
// Differences that are inherent to the device path and documented in INTEGRATION.md:
//   * normals come from Philox4x32-10 keyed by the RandomnessSourceContainer's seed (not boost mt19937);
//   * `max_num_threads` is accepted and validated against the container but the parallel axis is the GPU;
//   * `use_gpu` / `which_gpu` (dead arguments in the reference) select the device.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <limits>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "cmoe_b200.h"

namespace py = pybind11;

namespace {

PyObject* g_exc_base = nullptr;
PyObject* g_exc_bounds = nullptr;
PyObject* g_exc_invalid = nullptr;
PyObject* g_exc_singular = nullptr;

[[noreturn]] void raise_status(int rc, int info) {
  PyObject* type = g_exc_base;
  if (rc == CMOE_ERR_SINGULAR) type = g_exc_singular;
  if (rc == CMOE_ERR_BOUNDS) type = g_exc_bounds;
  if (rc == CMOE_ERR_INVALID_VALUE) type = g_exc_invalid;
  std::string msg = cmoe_last_error();
  if (rc == CMOE_ERR_SINGULAR) msg += " (leading minor index " + std::to_string(info) + ")";
  PyErr_SetString(type, msg.c_str());
  throw py::error_already_set();
}

void check(int rc, int info = 0) {
  if (rc != CMOE_OK) raise_status(rc, info);
}

std::vector<double> to_vec(const py::list& l, size_t n) {
  if (static_cast<size_t>(py::len(l)) < n) {
    PyErr_SetString(g_exc_bounds, "input list shorter than the size implied by the dimension arguments");
    throw py::error_already_set();
  }
  std::vector<double> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = l[i].cast<double>();
  return v;
}

std::vector<int> to_ivec(const py::list& l, size_t n) {
  std::vector<int> v(n);
  for (size_t i = 0; i < n; ++i) v[i] = l[i].cast<int>();
  return v;
}

py::list to_list(const std::vector<double>& v) {
  py::list out;
  for (double x : v) out.append(x);
  return out;
}

// One random-feature sample function of sample_gp_with_random_features, callable as the reference's wrapper(x, gradient):
// x is one point [dim] or points [X][dim] (a numpy array); gradient = False returns f at the points (a float for one
// point), gradient = True only the gradient ([dim] for one point, else [X][dim]), as random_features.py:113-131.
struct RandomFeatureSample {
  int dim = 0, F = 0, device = 0;
  double c = 0.0;
  std::vector<double> omega, b, theta;
  py::array_t<double> array(const std::vector<double>& v, std::vector<py::ssize_t> shape) const {
    py::array_t<double> a(shape);
    std::copy(v.begin(), v.end(), a.mutable_data());
    return a;
  }
  py::object call(const py::object& x, bool gradient) const;
};

// ---- parameter structs (gpp_optimizer_parameters.hpp:46-200) -------------------------------------------------------
struct GradientDescentParameters {
  cmoe_gd_params p;
  GradientDescentParameters(int num_multistarts, int max_num_steps, int max_num_restarts, int num_steps_averaged,
                            double gamma, double pre_mult, double max_relative_change, double tolerance)
      : p{num_multistarts, max_num_steps, max_num_restarts, num_steps_averaged, gamma, pre_mult, max_relative_change,
          tolerance} {}
};

struct NewtonParameters {
  int num_multistarts, max_num_steps;
  double gamma, time_factor, max_relative_change, tolerance;
  NewtonParameters(int a, int b, double c, double d, double e, double f)
      : num_multistarts(a), max_num_steps(b), gamma(c), time_factor(d), max_relative_change(e), tolerance(f) {}
};

enum class OptimizerTypes { kNull = 0, kGradientDescent = 1, kNewton = 2 };
enum class DomainTypes { kTensorProduct = 0, kSimplex = 1 };
enum class LogLikelihoodTypes { kLogMarginalLikelihood = 0, kLeaveOneOutLogLikelihood = 1 };

// ---- RandomnessSourceContainer (gpp_python_common.hpp:146-230) ------------------------------------------------------
struct RandomnessSourceContainer {
  static constexpr uint32_t kUniformDefaultSeed = 314, kNormalDefaultSeed = 314;
  std::mt19937 uniform_engine;
  uint32_t uniform_seed = kUniformDefaultSeed;
  std::vector<uint64_t> normal_seeds;  // one per "thread", as in the reference
  explicit RandomnessSourceContainer(int num_threads)
      : uniform_engine(kUniformDefaultSeed), normal_seeds(std::max(0, num_threads)) {
    SetExplicitNormalRNGSeed(kNormalDefaultSeed);
  }
  void SetExplicitUniformGeneratorSeed(uint32_t seed) { uniform_seed = seed; uniform_engine.seed(seed); }
  void SetRandomizedUniformGeneratorSeed(uint32_t seed) { SetExplicitUniformGeneratorSeed(mix(seed, 0)); }
  void ResetUniformGeneratorState() { uniform_engine.seed(uniform_seed); }
  void SetExplicitNormalRNGSeed(uint32_t seed) {
    for (size_t i = 0; i < normal_seeds.size(); ++i) normal_seeds[i] = static_cast<uint64_t>(seed) + i;
  }
  void SetRandomizedNormalRNGSeed(uint32_t seed) {
    for (size_t i = 0; i < normal_seeds.size(); ++i) normal_seeds[i] = mix(seed, static_cast<int>(i));
  }
  bool SetNormalRNGSeedPythonList(const py::list& seeds, const py::list& flags) {
    if (py::len(seeds) != py::len(flags) || py::len(seeds) != normal_seeds.size()) return false;
    for (size_t i = 0; i < normal_seeds.size(); ++i)
      if (flags[i].cast<int>()) normal_seeds[i] = static_cast<uint64_t>(seeds[i].cast<int64_t>());
    return true;
  }
  void ResetNormalRNGState() {}  // the Philox stream is a pure function of (seed, sample index): nothing to rewind
  void PrintState() const {
    std::printf("Uniform seed: %u\n", uniform_seed);
    for (size_t i = 0; i < normal_seeds.size(); ++i)
      std::printf("NormalRNG %zu: Philox4x32-10 key %llu\n", i, static_cast<unsigned long long>(normal_seeds[i]));
  }
  uint64_t seed0() const { return normal_seeds.empty() ? kNormalDefaultSeed : normal_seeds[0]; }
  static uint32_t mix(uint32_t seed, int thread_id) {
    std::random_device rd;
    return seed ^ (rd() + 0x9e3779b9u + (seed << 6) + (seed >> 2)) ^ static_cast<uint32_t>(thread_id * 2654435761u);
  }
};

void require_threads(int max_num_threads, const RandomnessSourceContainer& r) {
  if (max_num_threads > static_cast<int>(r.normal_seeds.size())) {
    PyErr_SetString(g_exc_bounds, "Fewer randomness_sources than max_num_threads.");
    throw py::error_already_set();
  }
}

// ---- GaussianProcess ------------------------------------------------------------------------------------------------
struct GaussianProcess {
  cmoe_gp* h = nullptr;
  int dim_ = 0, num_derivatives_ = 0;
  double alpha_ = 0.0;  // the kernel amplitude sigma^2 (the random features' c = sqrt(2 alpha / F))
  std::vector<int> derivatives_;
  GaussianProcess(const py::list& hyperparameters, const py::list& points_sampled, const py::list& points_sampled_value,
                  const py::list& noise_variance, const py::list& derivatives, int num_derivatives, int dim,
                  int num_sampled, const std::string& kernel, int which_gpu) {
    const double alpha = hyperparameters[0].cast<double>();
    alpha_ = alpha;
    const std::vector<double> lengths = to_vec(hyperparameters[1].cast<py::list>(), dim);
    const std::vector<double> X = to_vec(points_sampled, static_cast<size_t>(dim) * num_sampled);
    const std::vector<double> y = to_vec(points_sampled_value, static_cast<size_t>(num_sampled) * (1 + num_derivatives));
    const std::vector<double> noise = to_vec(noise_variance, 1 + num_derivatives);
    derivatives_ = to_ivec(derivatives, num_derivatives);
    dim_ = dim;
    num_derivatives_ = num_derivatives;
    // The reference's Python boundary hard-wires MaternNu2p5 (gpp_python_gaussian_process.cpp:53); SE is opt-in.
    const int kid = (kernel == "square_exponential") ? CMOE_KERNEL_SQUARE_EXPONENTIAL : CMOE_KERNEL_MATERN_NU_2P5;
    int info = 0;
    check(cmoe_gp_create(kid, alpha, lengths.data(), X.data(), y.data(), noise.data(), derivatives_.data(),
                         num_derivatives, dim, num_sampled, which_gpu, &h, &info),
          info);
  }
  ~GaussianProcess() { cmoe_gp_destroy(h); }
  // Randomness of the sampling methods: Philox key `seed_`, next unused draw `next_draw_`.  Construction behaves like
  // set_randomized_seed(0), as the reference's constructor does (gpp_python_gaussian_process.cpp:60).
  uint64_t seed_ = RandomnessSourceContainer::mix(0, 0), next_draw_ = 0;
  void set_explicit_seed(uint32_t s) { seed_ = s; next_draw_ = 0; }
  void set_randomized_seed(uint32_t s) { seed_ = RandomnessSourceContainer::mix(s, 0); next_draw_ = 0; }
  void reset_to_most_recent_seed() { next_draw_ = 0; }
  // SamplePointFromGPWrapper (gpp_python_gaussian_process.cpp:255-269): one joint draw of the value and the GP's
  // derivative rows at one point, without noise; uses one draw.
  py::list sample_point_from_gp(const py::list& point_to_sample) {
    const auto P = to_vec(point_to_sample, dim_);
    std::vector<double> out(1 + num_derivatives_);
    int info = 0;
    check(cmoe_gp_sample_joint(h, P.data(), 1, 1, derivatives_.data(), num_derivatives_, seed_, next_draw_, nullptr,
                               0.0, out.data(), nullptr, nullptr, nullptr, &info), info);
    ++next_draw_;
    return to_list(out);
  }
  // SampleGlobalOptimaFromGPWrapper (:271-286): num_optima * dim values; uses num_optima draws.
  py::list sample_global_optima(int num_optima, int inner_number, const py::list& domain_bounds) {
    const auto B = to_vec(domain_bounds, 2 * static_cast<size_t>(dim_));
    std::vector<double> out(static_cast<size_t>(std::max(num_optima, 0)) * dim_);
    int info = 0;
    check(cmoe_gp_sample_global_optima(h, num_optima, inner_number, B.data(), seed_, next_draw_, 0.0, out.data(),
                                       &info), info);
    next_draw_ += static_cast<uint64_t>(num_optima);
    return to_list(out);
  }
  GaussianProcess(const GaussianProcess&) = delete;
  GaussianProcess& operator=(const GaussianProcess&) = delete;
  int dim() const { return dim_; }
  int num_sampled() const { return cmoe_gp_num_sampled(h); }
  int Qs(int n) const { return n * (1 + num_derivatives_); }

  py::list mean(const py::list& pts, int n) const {  // GetMeanWrapper :64-79 (no derivative rows)
    const auto P = to_vec(pts, static_cast<size_t>(n) * dim_);
    std::vector<double> out(n);
    int info = 0;
    check(cmoe_gp_posterior(h, P.data(), 1, n, nullptr, 0, out.data(), nullptr, nullptr, nullptr, nullptr, nullptr, &info), info);
    return to_list(out);
  }
  py::list grad_mean(const py::list& pts, int n) const {  // GetGradMeanWrapper :98-116 (GP's derivative rows)
    const auto P = to_vec(pts, static_cast<size_t>(n) * dim_);
    std::vector<double> out(static_cast<size_t>(dim_) * Qs(n));
    int info = 0;
    check(cmoe_gp_posterior(h, P.data(), 1, n, derivatives_.data(), num_derivatives_, nullptr, out.data(), nullptr,
                            nullptr, nullptr, nullptr, &info), info);
    return to_list(out);
  }
  py::list variance(const py::list& pts, int n) const {  // GetVarWrapper :118-154: full symmetric, row by row
    const auto P = to_vec(pts, static_cast<size_t>(n) * dim_);
    const int Q = Qs(n);
    std::vector<double> v(static_cast<size_t>(Q) * Q);
    int info = 0;
    if (Q > CMOE_MAX_SET_ROWS)
      check(cmoe_gp_posterior_large(h, P.data(), 1, n, derivatives_.data(), num_derivatives_, nullptr, v.data(), nullptr,
                                    &info), info);
    else
      check(cmoe_gp_posterior(h, P.data(), 1, n, derivatives_.data(), num_derivatives_, nullptr, nullptr, v.data(),
                              nullptr, nullptr, nullptr, &info), info);
    py::list out;
    for (int i = 0; i < Q; ++i)
      for (int j = 0; j < Q; ++j) out.append(v[static_cast<size_t>(j) * Q + i]);
    return out;
  }
  py::list chol_variance(const py::list& pts, int n) const {  // GetCholVarWrapper :156-187
    const auto P = to_vec(pts, static_cast<size_t>(n) * dim_);
    const int Q = Qs(n);
    std::vector<double> v(static_cast<size_t>(Q) * Q);
    int info = 0;
    if (Q > CMOE_MAX_SET_ROWS)
      check(cmoe_gp_posterior_large(h, P.data(), 1, n, derivatives_.data(), num_derivatives_, nullptr, nullptr,
                                    v.data(), &info), info);
    else
      check(cmoe_gp_posterior(h, P.data(), 1, n, derivatives_.data(), num_derivatives_, nullptr, nullptr, nullptr,
                              v.data(), nullptr, nullptr, &info), info);
    py::list out;
    for (int i = 0; i < Q; ++i)
      for (int j = 0; j < Q; ++j) out.append(v[static_cast<size_t>(j) * Q + i]);
    return out;
  }
  py::list grad_variance(const py::list& pts, int n, int num_derivatives, bool chol) const {  // :189-236
    const auto P = to_vec(pts, static_cast<size_t>(n) * dim_);
    const int Q = Qs(n);
    std::vector<double> g(static_cast<size_t>(dim_) * Q * Q * n);
    int info = 0;
    check(cmoe_gp_posterior(h, P.data(), 1, n, derivatives_.data(), num_derivatives_, nullptr, nullptr, nullptr, nullptr,
                            chol ? nullptr : g.data(), chol ? g.data() : nullptr, &info), info);
    g.resize(static_cast<size_t>(dim_) * Q * Q * std::min(n, std::max(0, num_derivatives)));
    return to_list(g);
  }
  void add_sampled_points(const py::list& pts, const py::list& vals, int n) {  // AddPointsToGPWrapper :238-253
    const auto P = to_vec(pts, static_cast<size_t>(n) * dim_);
    const auto V = to_vec(vals, static_cast<size_t>(n) * (1 + num_derivatives_));
    int info = 0;
    check(cmoe_gp_add_sampled_points(h, P.data(), V.data(), n, &info), info);
  }
};

cmoe_gd_params gd_of(const py::object& optimizer_parameters) {
  return optimizer_parameters.attr("optimizer_parameters").cast<const GradientDescentParameters&>().p;
}

// a GaussianProcess, or a wrapper holding one as `_gaussian_process` (the reference's python_version objects)
GaussianProcess& unwrap_gp(const py::object& gaussian_process) {
  py::object o = gaussian_process;
  if (!py::isinstance<GaussianProcess>(o) && py::hasattr(o, "_gaussian_process")) o = o.attr("_gaussian_process");
  return o.cast<GaussianProcess&>();
}

py::object RandomFeatureSample::call(const py::object& x, bool gradient) const {
  const auto xa = py::array_t<double, py::array::c_style | py::array::forcecast>::ensure(x);
  if (!xa || (xa.ndim() != 1 && xa.ndim() != 2) || xa.shape(xa.ndim() - 1) != dim) {
    PyErr_SetString(g_exc_bounds, "x must be a point [dim] or points [num_points][dim]");
    throw py::error_already_set();
  }
  const int X = xa.ndim() == 1 ? 1 : static_cast<int>(xa.shape(0));
  std::vector<double> out(static_cast<size_t>(std::max(X, 0)) * (gradient ? dim : 1));
  int info = 0;
  check(cmoe_rff_evaluate(dim, F, 1, omega.data(), b.data(), theta.data(), c, xa.data(), X, 0,
                          gradient ? nullptr : out.data(), gradient ? out.data() : nullptr, device, &info),
        info);
  if (gradient) return xa.ndim() == 1 ? array(out, {dim}) : array(out, {X, dim});
  if (X == 1) return py::float_(out[0]);
  return array(out, {X});
}

std::vector<double> full_bounds(const py::list& domain_bounds, int dim) { return to_vec(domain_bounds, 2 * static_cast<size_t>(dim)); }

// ---- EI ---------------------------------------------------------------------------------------------------------------
// The q-EI evaluator for a union of q + p rows: the per-set kernels up to CMOE_MAX_SET_ROWS, the tiled path past them.
using EiEvalFn = int (*)(const cmoe_gp*, const double*, int, int, const double*, int, int, double, uint64_t,
                         const double*, double*, double*, int*);
EiEvalFn ei_eval_for(int q, int p) { return q + p > CMOE_MAX_SET_ROWS ? cmoe_ei_eval_large : cmoe_ei_eval; }

double compute_expected_improvement(const GaussianProcess& gp, const py::list& pts, const py::list& being, int q, int p,
                                    int max_int_steps, double best_so_far, bool /*force_monte_carlo*/,
                                    RandomnessSourceContainer& rnd) {
  const auto X = to_vec(pts, static_cast<size_t>(q) * gp.dim_);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * gp.dim_);
  double ei = 0.0;
  int info = 0;
  check(ei_eval_for(q, p)(gp.h, X.data(), 1, q, Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(), nullptr, &ei, nullptr,
                     &info), info);
  return ei;
}

py::list compute_grad_expected_improvement(const GaussianProcess& gp, const py::list& pts, const py::list& being, int q,
                                           int p, int max_int_steps, double best_so_far, bool /*force_monte_carlo*/,
                                           RandomnessSourceContainer& rnd) {
  const auto X = to_vec(pts, static_cast<size_t>(q) * gp.dim_);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * gp.dim_);
  double ei = 0.0;
  std::vector<double> g(static_cast<size_t>(q) * gp.dim_);
  int info = 0;
  check(ei_eval_for(q, p)(gp.h, X.data(), 1, q, Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(), nullptr, &ei, g.data(),
                     &info), info);
  return to_list(g);
}

// Latin hypercube starts in a repeated tensor-product domain (gpp_random.cpp:173-197, gpp_domain.hpp:490-515)
std::vector<double> lhc_starts(const std::vector<double>& bounds, int dim, int q, int num, std::mt19937& eng) {
  std::vector<double> out(static_cast<size_t>(num) * q * dim);
  std::vector<int> idx(num);
  for (int rep = 0; rep < q; ++rep) {
    for (int d = 0; d < dim; ++d) {
      const double edge = (bounds[2 * d + 1] - bounds[2 * d]) / static_cast<double>(num);
      for (int j = 0; j < num; ++j) idx[j] = j;
      std::shuffle(idx.begin(), idx.end(), eng);
      std::uniform_real_distribution<double> u(0.0, edge);
      for (int j = 0; j < num; ++j)
        out[(static_cast<size_t>(j) * q + rep) * dim + d] = bounds[2 * d] + edge * idx[j] + u(eng);
    }
  }
  return out;
}

// Starts inside the unit simplex intersected with the box, by rejection from the (clipped) box as
// SimplexIntersectTensorProductDomain::GeneratePointInDomain does (gpp_domain.cpp:153-163): every one of the q points of a
// start is drawn until it lies in the simplex (at most 10000 attempts each, then the last draw is kept).
std::vector<double> simplex_starts(const std::vector<double>& bounds, int dim, int q, int num, std::mt19937& eng) {
  std::vector<double> out(static_cast<size_t>(num) * q * dim);
  for (size_t pt = 0; pt < static_cast<size_t>(num) * q; ++pt) {
    double* x = out.data() + pt * dim;
    for (int attempt = 0; attempt < 10000; ++attempt) {
      double sum = 0.0;
      for (int d = 0; d < dim; ++d) {
        const double lo = std::max(bounds[2 * d], 0.0), hi = std::min(bounds[2 * d + 1], 1.0);
        x[d] = std::uniform_real_distribution<double>(lo, hi)(eng);
        sum += x[d];
      }
      if (sum <= 1.0) break;
    }
  }
  return out;
}

// The reference's parallel axis is `max_num_threads` OpenMP threads over the multistart starts; here that knob selects
// how many GPUs share the starts inside ONE call: min(max_num_threads, visible devices, $CMOE_MAX_DEVICES), beginning
// with the GP's own device.  One device (the default when CMOE_MAX_DEVICES is unset) keeps the single-GPU path.
std::vector<int> devices_for(int home_device, int max_num_threads) {
  int cap = 1;
  if (const char* e = std::getenv("CMOE_MAX_DEVICES")) cap = std::max(1, std::atoi(e));
  const int count = cmoe_device_count();
  const int n = std::max(1, std::min(std::min(max_num_threads, cap), count));
  std::vector<int> devs{home_device};
  for (int d = 0; d < count && static_cast<int>(devs.size()) < n; ++d)
    if (d != home_device) devs.push_back(d);
  return devs;
}

py::list multistart_expected_improvement_optimization(const py::object& optimizer_parameters, const GaussianProcess& gp,
                                                      const py::list& domain_bounds, const py::list& being, int q, int p,
                                                      double best_so_far, int max_int_steps, int max_num_threads,
                                                      bool /*use_gpu*/, int /*which_gpu*/, RandomnessSourceContainer& rnd,
                                                      py::dict& status) {
  require_threads(max_num_threads, rnd);
  const int dim = gp.dim_;
  const auto bounds = full_bounds(domain_bounds, dim);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const auto domain_type = optimizer_parameters.attr("domain_type").cast<DomainTypes>();
  const auto opt_type = optimizer_parameters.attr("optimizer_type").cast<OptimizerTypes>();
  const bool simplex = domain_type == DomainTypes::kSimplex;
  auto make_starts = [&](int n) {
    return simplex ? simplex_starts(bounds, dim, q, n, rnd.uniform_engine) : lhc_starts(bounds, dim, q, n, rnd.uniform_engine);
  };
  std::vector<double> best(static_cast<size_t>(q) * dim, 0.0);
  double best_value = 0.0;
  int found = 0, info = 0;
  if (opt_type == OptimizerTypes::kNull) {
    const int n = optimizer_parameters.attr("num_random_samples").cast<int>();
    const auto starts = make_starts(n);
    std::vector<double> vals(n);
    check(ei_eval_for(q, p)(gp.h, starts.data(), n, q, Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(), nullptr,
                       vals.data(), nullptr, &info), info);
    double bv = -1.0;
    std::copy(starts.begin(), starts.begin() + static_cast<size_t>(q) * dim, best.begin());
    for (int i = 0; i < n; ++i)
      if (bv < vals[i]) {
        bv = vals[i];
        found = 1;
        std::copy(starts.begin() + static_cast<size_t>(i) * q * dim, starts.begin() + static_cast<size_t>(i + 1) * q * dim, best.begin());
      }
    status[simplex ? "lhc_simplex_domain_found_update" : "lhc_tensor_product_domain_found_update"] = static_cast<bool>(found);
  } else if (opt_type == OptimizerTypes::kGradientDescent) {
    const cmoe_gd_params gd = gd_of(optimizer_parameters);
    const auto starts = make_starts(gd.num_multistarts);
    const std::vector<int> devs = devices_for(cmoe_gp_device(gp.h), max_num_threads);
    const cmoe_multistart_opts opts{nullptr, 0, devs.data(), static_cast<int>(devs.size()),
                                    simplex ? CMOE_DOMAIN_SIMPLEX : CMOE_DOMAIN_TENSOR_PRODUCT};
    check(cmoe_multistart_ei_ex(gp.h, &gd, bounds.data(), starts.data(), gd.num_multistarts, q, Xp.data(), p,
                                max_int_steps, best_so_far, rnd.seed0(), &opts, nullptr, best.data(), &best_value, &found,
                                &info), info);
    status[simplex ? "gradient_descent_simplex_domain_found_update" : "gradient_descent_tensor_product_domain_found_update"] = static_cast<bool>(found);
  } else {
    PyErr_SetString(g_exc_base, "ERROR: invalid optimizer choice. Setting all coordinates to 0.0.");
    throw py::error_already_set();
  }
  return to_list(best);
}

py::list evaluate_EI_at_point_list(const GaussianProcess& gp, const py::list& initial_guesses, const py::list& being,
                                   int num_multistarts, int q, int p, double best_so_far, int max_int_steps,
                                   int max_num_threads, RandomnessSourceContainer& rnd, py::dict& status) {
  require_threads(max_num_threads, rnd);
  const auto starts = to_vec(initial_guesses, static_cast<size_t>(num_multistarts) * q * gp.dim_);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * gp.dim_);
  std::vector<double> vals(num_multistarts);
  int info = 0;
  if (q == 1 && p == 0)  // closed-form 1-EI, as EvaluateEIAtPointList does (gpp_math.cpp:2317)
    check(cmoe_ei_analytic(gp.h, starts.data(), num_multistarts, best_so_far, vals.data(), nullptr, &info), info);
  else
    check(ei_eval_for(q, p)(gp.h, starts.data(), num_multistarts, q, Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(),
                       nullptr, vals.data(), nullptr, &info), info);
  bool found = false;
  for (double v : vals) found = found || (v > -1.0);
  status["evaluate_EI_at_point_list"] = found;
  return to_list(vals);
}

// ---- heuristic EI (DESIGN.md K20) -----------------------------------------------------------------------------------
// The estimation policies of gpp_python_expected_improvement.cpp:445-486, with their positional constructors.
struct ObjectiveEstimationPolicyInterface {
  cmoe_estimation_policy p{};
  virtual ~ObjectiveEstimationPolicyInterface() = default;
};
struct ConstantLiarEstimationPolicy : ObjectiveEstimationPolicyInterface {
  ConstantLiarEstimationPolicy(double lie_value, double lie_noise_variance) {
    p = {CMOE_ESTIMATION_CONSTANT_LIAR, lie_value, lie_noise_variance};
  }
};
struct KrigingBelieverEstimationPolicy : ObjectiveEstimationPolicyInterface {
  KrigingBelieverEstimationPolicy(double std_deviation_coef, double kriging_noise_variance) {
    p = {CMOE_ESTIMATION_KRIGING_BELIEVER, std_deviation_coef, kriging_noise_variance};
  }
};

// HeuristicExpectedImprovementOptimizationWrapper (gpp_python_expected_improvement.cpp:278-400, 602-659): q rounds of
// one-point EI optimisation with the policy's fantasy fed back after each round (cmoe_heuristic_ei).  Round r's starts
// are the r-th Latin-hypercube block drawn from the uniform engine; the draws do not depend on results, so all q blocks
// are drawn up front in round order.  The status flag is the AND of the rounds' found flags.
py::list heuristic_expected_improvement_optimization(const py::object& optimizer_parameters,
                                                     const py::object& gaussian_process, const py::list& domain_bounds,
                                                     const ObjectiveEstimationPolicyInterface& estimation_policy,
                                                     int num_to_sample, double best_so_far, int /*max_num_threads*/,
                                                     RandomnessSourceContainer& rnd, py::dict& status) {
  const GaussianProcess& gp = unwrap_gp(gaussian_process);
  const int dim = gp.dim_, q = num_to_sample;
  const auto domain_type = optimizer_parameters.attr("domain_type").cast<DomainTypes>();
  const auto opt_type = optimizer_parameters.attr("optimizer_type").cast<OptimizerTypes>();
  if (domain_type == DomainTypes::kSimplex) {
    PyErr_SetString(g_exc_base, "heuristic_expected_improvement_optimization: only the tensor_product domain is "
                                "implemented");
    throw py::error_already_set();
  }
  if (opt_type != OptimizerTypes::kNull && opt_type != OptimizerTypes::kGradientDescent) {
    PyErr_SetString(g_exc_base, "ERROR: invalid optimizer choice. Setting all coordinates to 0.0.");
    throw py::error_already_set();
  }
  if (q < 1) {
    PyErr_SetString(g_exc_bounds, "num_to_sample must be >= 1");
    throw py::error_already_set();
  }
  const auto bounds = full_bounds(domain_bounds, dim);
  const bool null_opt = opt_type == OptimizerTypes::kNull;
  cmoe_gd_params gd{};
  if (!null_opt) gd = gd_of(optimizer_parameters);
  const int n = null_opt ? optimizer_parameters.attr("num_random_samples").cast<int>() : gd.num_multistarts;
  if (n < 1) {
    PyErr_SetString(g_exc_bounds, "num_multistarts must be > 1");
    throw py::error_already_set();
  }
  std::vector<double> starts;
  for (int r = 0; r < q; ++r) {
    const auto block = lhc_starts(bounds, dim, 1, n, rnd.uniform_engine);
    starts.insert(starts.end(), block.begin(), block.end());
  }
  std::vector<double> pts(static_cast<size_t>(q) * dim);
  std::vector<int> found(q);
  int info = 0;
  check(cmoe_heuristic_ei(gp.h, &estimation_policy.p, null_opt ? nullptr : &gd, bounds.data(), starts.data(), n, q,
                          best_so_far, pts.data(), nullptr, nullptr, found.data(), &info),
        info);
  bool all = true;
  for (int f : found) all = all && f != 0;
  status[null_opt ? "lhc_tensor_product_domain_found_update" : "gradient_descent_tensor_product_domain_found_update"] =
      all;
  return to_list(pts);
}

// ---- posterior mean / KG ----------------------------------------------------------------------------------------------
std::vector<double> pad_fidelity(const std::vector<double>& pt, int dim) {
  std::vector<double> full(dim, 1.0);  // fidelity coordinates pinned to 1.0 (...knowledge_gradient_optimization.cpp:365)
  std::copy(pt.begin(), pt.end(), full.begin());
  return full;
}

double compute_posterior_mean(const GaussianProcess& gp, int num_fidelity, const py::list& pt) {
  const auto x = pad_fidelity(to_vec(pt, gp.dim_ - num_fidelity), gp.dim_);
  double m = 0.0;
  int info = 0;
  check(cmoe_gp_posterior(gp.h, x.data(), 1, 1, nullptr, 0, &m, nullptr, nullptr, nullptr, nullptr, nullptr, &info), info);
  return -m;  // the evaluator maximises -mu (...cpp:334-340)
}

// Batched form of compute_posterior_mean (not in the reference module): the examples screen 1e3-1e4 points with a
// Python loop of single-point calls (examples/main.py:147-152, 180-186); this evaluates all of them in ONE device call.
py::list compute_posterior_mean_of_points(const GaussianProcess& gp, int num_fidelity, const py::list& pts,
                                          int num_points) {
  const int ps = gp.dim_ - num_fidelity;
  const auto flat = to_vec(pts, static_cast<size_t>(num_points) * ps);
  std::vector<double> full(static_cast<size_t>(num_points) * gp.dim_, 1.0);
  for (int i = 0; i < num_points; ++i)
    std::copy(flat.begin() + static_cast<size_t>(i) * ps, flat.begin() + static_cast<size_t>(i + 1) * ps,
              full.begin() + static_cast<size_t>(i) * gp.dim_);
  std::vector<double> m(num_points);
  int info = 0;
  check(cmoe_gp_posterior(gp.h, full.data(), num_points, 1, nullptr, 0, m.data(), nullptr, nullptr, nullptr, nullptr,
                          nullptr, &info), info);
  for (double& v : m) v = -v;
  return to_list(m);
}

py::list compute_grad_posterior_mean(const GaussianProcess& gp, int num_fidelity, const py::list& pt) {
  const auto x = pad_fidelity(to_vec(pt, gp.dim_ - num_fidelity), gp.dim_);
  std::vector<double> g(gp.dim_);
  int info = 0;
  check(cmoe_gp_posterior(gp.h, x.data(), 1, 1, nullptr, 0, nullptr, g.data(), nullptr, nullptr, nullptr, nullptr, &info), info);
  std::vector<double> out(gp.dim_ - num_fidelity);
  for (size_t i = 0; i < out.size(); ++i) out[i] = -g[i];
  return to_list(out);
}

// ---- q-KG ---------------------------------------------------------------------------------------------------------------
// The q-KG evaluator for a union of (q + p)(1 + g) rows: cmoe_kg_eval up to CMOE_MAX_KG_ROWS, cmoe_kg_eval_large past it.
using KgEvalFn = int (*)(const cmoe_gp*, int, const cmoe_gd_params*, const double*, const double*, int, const double*,
                         int, int, const double*, int, int, double, uint64_t, const double*, double*, double*,
                         cmoe_kg_stats*, int*);
KgEvalFn kg_eval_for(const GaussianProcess& gp, int q, int p) {
  return static_cast<long long>(q + p) * (1 + gp.num_derivatives_) > CMOE_MAX_KG_ROWS ? cmoe_kg_eval_large
                                                                                       : cmoe_kg_eval;
}

double compute_knowledge_gradient(const GaussianProcess& gp, int num_fidelity, const py::object& optimizer_parameters,
                                  const py::list& domain_bounds, const py::list& discrete_pts, const py::list& pts,
                                  const py::list& being, int num_pts, int q, int p, int max_int_steps, double best_so_far,
                                  RandomnessSourceContainer& rnd) {
  const int dim = gp.dim_, ps = dim - num_fidelity;
  const auto inner_bounds = to_vec(domain_bounds, 2 * static_cast<size_t>(ps));
  const auto D = to_vec(discrete_pts, static_cast<size_t>(num_pts) * ps);
  const auto X = to_vec(pts, static_cast<size_t>(q) * dim);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const cmoe_gd_params inner = gd_of(optimizer_parameters);
  double kg = 0.0;
  int info = 0;
  check(kg_eval_for(gp, q, p)(gp.h, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts, X.data(), 1, q,
                              Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(), nullptr, &kg, nullptr, nullptr,
                              &info),
        info);
  return kg;
}

py::list compute_grad_knowledge_gradient(const GaussianProcess& gp, int num_fidelity,
                                         const py::object& optimizer_parameters, const py::list& domain_bounds,
                                         const py::list& discrete_pts, const py::list& pts, const py::list& being,
                                         int num_pts, int q, int p, int max_int_steps, double best_so_far,
                                         RandomnessSourceContainer& rnd) {
  const int dim = gp.dim_, ps = dim - num_fidelity;
  const auto inner_bounds = to_vec(domain_bounds, 2 * static_cast<size_t>(ps));
  const auto D = to_vec(discrete_pts, static_cast<size_t>(num_pts) * ps);
  const auto X = to_vec(pts, static_cast<size_t>(q) * dim);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const cmoe_gd_params inner = gd_of(optimizer_parameters);
  double kg = 0.0;
  std::vector<double> g(static_cast<size_t>(q) * dim);
  int info = 0;
  check(kg_eval_for(gp, q, p)(gp.h, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts, X.data(), 1, q,
                              Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(), nullptr, &kg, g.data(), nullptr,
                              &info),
        info);
  return to_list(g);
}

py::list multistart_knowledge_gradient_optimization(const py::object& optimizer_parameters,
                                                    const py::object& optimizer_parameters_inner,
                                                    const GaussianProcess& gp, int num_fidelity,
                                                    const py::list& domain_bounds, const py::list& discrete_pts,
                                                    const py::list& being, int num_pts, int q, int p, double best_so_far,
                                                    int max_int_steps, int max_num_threads,
                                                    RandomnessSourceContainer& rnd, py::dict& status) {
  require_threads(max_num_threads, rnd);
  const int dim = gp.dim_, ps = dim - num_fidelity;
  const auto bounds = full_bounds(domain_bounds, dim);
  const std::vector<double> inner_bounds(bounds.begin(), bounds.begin() + 2 * ps);
  const auto D = to_vec(discrete_pts, static_cast<size_t>(num_pts) * ps);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const auto domain_type = optimizer_parameters.attr("domain_type").cast<DomainTypes>();
  const auto opt_type = optimizer_parameters.attr("optimizer_type").cast<OptimizerTypes>();
  if (domain_type != DomainTypes::kTensorProduct) {
    PyErr_SetString(g_exc_base, "only the tensor_product domain is implemented on the GPU path");
    throw py::error_already_set();
  }
  const cmoe_gd_params inner = gd_of(optimizer_parameters_inner);
  std::vector<double> best(static_cast<size_t>(q) * dim, 0.0);
  double best_value = 0.0;
  int found = 0, info = 0;
  if (opt_type == OptimizerTypes::kNull) {
    const int n = optimizer_parameters.attr("num_random_samples").cast<int>();
    const auto starts = lhc_starts(bounds, dim, q, n, rnd.uniform_engine);
    std::vector<double> vals(n);
    check(kg_eval_for(gp, q, p)(gp.h, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts, starts.data(), n,
                                q, Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(), nullptr, vals.data(), nullptr,
                                nullptr, &info),
          info);
    double bv = -INFINITY;
    std::copy(starts.begin(), starts.begin() + static_cast<size_t>(q) * dim, best.begin());
    for (int i = 0; i < n; ++i)
      if (bv < vals[i]) {
        bv = vals[i];
        found = 1;
        std::copy(starts.begin() + static_cast<size_t>(i) * q * dim, starts.begin() + static_cast<size_t>(i + 1) * q * dim, best.begin());
      }
    status["lhc_tensor_product_domain_found_update"] = static_cast<bool>(found);
  } else if (opt_type == OptimizerTypes::kGradientDescent) {
    const cmoe_gd_params gd = gd_of(optimizer_parameters);
    const auto starts = lhc_starts(bounds, dim, q, gd.num_multistarts, rnd.uniform_engine);
    const std::vector<int> devs = devices_for(cmoe_gp_device(gp.h), max_num_threads);
    const cmoe_multistart_opts opts{nullptr, 0, devs.data(), static_cast<int>(devs.size())};
    check(cmoe_multistart_kg_ex(gp.h, num_fidelity, &gd, &inner, bounds.data(), inner_bounds.data(), D.data(), num_pts,
                                starts.data(), gd.num_multistarts, q, Xp.data(), p, max_int_steps, best_so_far,
                                rnd.seed0(), &opts, nullptr, best.data(), &best_value, &found, &info), info);
    status["gradient_descent_tensor_product_domain_found_update"] = static_cast<bool>(found);
  } else {
    PyErr_SetString(g_exc_base, "ERROR: invalid optimizer choice. Setting all coordinates to 0.0.");
    throw py::error_already_set();
  }
  return to_list(best);
}

py::list evaluate_KG_at_point_list(const GaussianProcess& gp, int num_fidelity, const py::object& optimizer_parameters,
                                   const py::list& domain_bounds, const py::list& discrete_being_sampled,
                                   const py::list& initial_guesses, int num_multistarts, int num_pts, int q, int p,
                                   double best_so_far, int max_int_steps, int max_num_threads,
                                   RandomnessSourceContainer& rnd, py::dict& status) {
  require_threads(max_num_threads, rnd);
  const int dim = gp.dim_, ps = dim - num_fidelity;
  const auto bounds = full_bounds(domain_bounds, dim);
  const std::vector<double> inner_bounds(bounds.begin(), bounds.begin() + 2 * ps);
  // [discrete_pts (num_pts x dim) ; points_being_sampled (p x dim)], as the reference wrapper slices it (:376-390)
  const auto both = to_vec(discrete_being_sampled, static_cast<size_t>(num_pts + p) * dim);
  std::vector<double> D(static_cast<size_t>(num_pts) * ps);
  for (int j = 0; j < num_pts; ++j)
    for (int d = 0; d < ps; ++d) D[static_cast<size_t>(j) * ps + d] = both[static_cast<size_t>(j) * dim + d];
  const std::vector<double> Xp(both.begin() + static_cast<size_t>(num_pts) * dim, both.end());
  const auto starts = to_vec(initial_guesses, static_cast<size_t>(num_multistarts) * q * dim);
  const cmoe_gd_params inner = gd_of(optimizer_parameters);
  std::vector<double> vals(num_multistarts);
  int info = 0;
  check(kg_eval_for(gp, q, p)(gp.h, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts, starts.data(),
                              num_multistarts, q, Xp.data(), p, max_int_steps, best_so_far, rnd.seed0(), nullptr,
                              vals.data(), nullptr, nullptr, &info),
        info);
  bool found = false;
  for (double v : vals) found = found || std::isfinite(v);
  status["evaluate_KG_at_point_list"] = found;
  return to_list(vals);
}

// ---- GaussianProcessMCMC + MCMC-averaged acquisition ---------------------------------------------------------------------
// (gpp_python_knowledge_gradient_mcmc.cpp:49-384, gpp_python_expected_improvement_mcmc.cpp:46-300)
struct GaussianProcessMCMC {
  std::vector<cmoe_gp*> members;
  int dim_ = 0, num_derivatives_ = 0, num_sampled_ = 0;
  std::vector<int> derivatives_;
  GaussianProcessMCMC(const py::list& hyperparameters_list, const py::list& noise_variance_list,
                      const py::list& points_sampled, const py::list& points_sampled_value, const py::list& derivatives,
                      int num_mcmc, int num_derivatives, int dim, int num_sampled, const std::string& kernel,
                      int which_gpu) {
    // hyperparameters_list: num_mcmc x (alpha, length_1..length_dim) flat; noise_variance_list: num_mcmc x (1+g) flat
    const auto hyp = to_vec(hyperparameters_list, static_cast<size_t>(num_mcmc) * (dim + 1));
    const auto noise = to_vec(noise_variance_list, static_cast<size_t>(num_mcmc) * (1 + num_derivatives));
    const auto X = to_vec(points_sampled, static_cast<size_t>(dim) * num_sampled);
    const auto y = to_vec(points_sampled_value, static_cast<size_t>(num_sampled) * (1 + num_derivatives));
    derivatives_ = to_ivec(derivatives, num_derivatives);
    dim_ = dim;
    num_derivatives_ = num_derivatives;
    num_sampled_ = num_sampled;
    const int kid = (kernel == "square_exponential") ? CMOE_KERNEL_SQUARE_EXPONENTIAL : CMOE_KERNEL_MATERN_NU_2P5;
    for (int m = 0; m < num_mcmc; ++m) {
      cmoe_gp* h = nullptr;
      int info = 0;
      const int rc = cmoe_gp_create(kid, hyp[static_cast<size_t>(m) * (dim + 1)], hyp.data() + static_cast<size_t>(m) * (dim + 1) + 1,
                                    X.data(), y.data(), noise.data() + static_cast<size_t>(m) * (1 + num_derivatives),
                                    derivatives_.data(), num_derivatives, dim, num_sampled, which_gpu, &h, &info);
      if (rc != CMOE_OK) {
        for (cmoe_gp* g : members) cmoe_gp_destroy(g);
        members.clear();
        check(rc, info);
      }
      members.push_back(h);
    }
  }
  ~GaussianProcessMCMC() {
    for (cmoe_gp* g : members) cmoe_gp_destroy(g);
  }
  GaussianProcessMCMC(const GaussianProcessMCMC&) = delete;
  GaussianProcessMCMC& operator=(const GaussianProcessMCMC&) = delete;
  int num_mcmc() const { return static_cast<int>(members.size()); }
  const cmoe_gp* const* handles() const { return members.data(); }
};

double compute_knowledge_gradient_mcmc(const GaussianProcessMCMC& gp, int num_fidelity, const py::object& optimizer_parameters,
                                       const py::list& domain_bounds, const py::list& discrete_pts, const py::list& pts,
                                       const py::list& being, int num_pts, int q, int p, int max_int_steps,
                                       const py::list& best_so_far, RandomnessSourceContainer& rnd) {
  const int dim = gp.dim_, ps = dim - num_fidelity, M = gp.num_mcmc();
  const auto inner_bounds = to_vec(domain_bounds, 2 * static_cast<size_t>(ps));
  const auto D = to_vec(discrete_pts, static_cast<size_t>(M) * num_pts * ps);
  const auto X = to_vec(pts, static_cast<size_t>(q) * dim);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const auto best = to_vec(best_so_far, M);
  const cmoe_gd_params inner = gd_of(optimizer_parameters);
  double kg = 0.0;
  int info = 0;
  check(cmoe_kg_eval_mcmc(gp.handles(), M, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts, X.data(), 1, q,
                          Xp.data(), p, max_int_steps, best.data(), rnd.seed0(), nullptr, &kg, nullptr, &info), info);
  return kg;
}

py::list compute_grad_knowledge_gradient_mcmc(const GaussianProcessMCMC& gp, int num_fidelity,
                                              const py::object& optimizer_parameters, const py::list& domain_bounds,
                                              const py::list& discrete_pts, const py::list& pts, const py::list& being,
                                              int num_pts, int q, int p, int max_int_steps, const py::list& best_so_far,
                                              RandomnessSourceContainer& rnd) {
  const int dim = gp.dim_, ps = dim - num_fidelity, M = gp.num_mcmc();
  const auto inner_bounds = to_vec(domain_bounds, 2 * static_cast<size_t>(ps));
  const auto D = to_vec(discrete_pts, static_cast<size_t>(M) * num_pts * ps);
  const auto X = to_vec(pts, static_cast<size_t>(q) * dim);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const auto best = to_vec(best_so_far, M);
  const cmoe_gd_params inner = gd_of(optimizer_parameters);
  double kg = 0.0;
  std::vector<double> g(static_cast<size_t>(q) * dim);
  int info = 0;
  check(cmoe_kg_eval_mcmc(gp.handles(), M, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts, X.data(), 1, q,
                          Xp.data(), p, max_int_steps, best.data(), rnd.seed0(), nullptr, &kg, g.data(), &info), info);
  return to_list(g);
}

template <typename EvalAll, typename Multistart>
py::list mcmc_optimization_common(const py::object& optimizer_parameters, const std::vector<double>& bounds, int dim,
                                  int q, double init_best, RandomnessSourceContainer& rnd, py::dict& status,
                                  EvalAll&& eval_all, Multistart&& multistart) {
  const auto domain_type = optimizer_parameters.attr("domain_type").cast<DomainTypes>();
  const auto opt_type = optimizer_parameters.attr("optimizer_type").cast<OptimizerTypes>();
  if (domain_type != DomainTypes::kTensorProduct) {
    PyErr_SetString(g_exc_base, "only the tensor_product domain is implemented on the GPU path");
    throw py::error_already_set();
  }
  std::vector<double> best(static_cast<size_t>(q) * dim, 0.0);
  int found = 0;
  if (opt_type == OptimizerTypes::kNull) {
    const int n = optimizer_parameters.attr("num_random_samples").cast<int>();
    const auto starts = lhc_starts(bounds, dim, q, n, rnd.uniform_engine);
    std::vector<double> vals(n);
    eval_all(starts, n, vals);
    double bv = init_best;
    std::copy(starts.begin(), starts.begin() + static_cast<size_t>(q) * dim, best.begin());
    for (int i = 0; i < n; ++i)
      if (bv < vals[i]) {
        bv = vals[i];
        found = 1;
        std::copy(starts.begin() + static_cast<size_t>(i) * q * dim, starts.begin() + static_cast<size_t>(i + 1) * q * dim, best.begin());
      }
    status["lhc_tensor_product_domain_found_update"] = static_cast<bool>(found);
  } else if (opt_type == OptimizerTypes::kGradientDescent) {
    const cmoe_gd_params gd = gd_of(optimizer_parameters);
    const auto starts = lhc_starts(bounds, dim, q, gd.num_multistarts, rnd.uniform_engine);
    multistart(gd, starts, best, found);
    status["gradient_descent_tensor_product_domain_found_update"] = static_cast<bool>(found);
  } else {
    PyErr_SetString(g_exc_base, "ERROR: invalid optimizer choice. Setting all coordinates to 0.0.");
    throw py::error_already_set();
  }
  return to_list(best);
}

py::list multistart_knowledge_gradient_mcmc_optimization(const py::object& optimizer_parameters,
                                                         const py::object& optimizer_parameters_inner,
                                                         const GaussianProcessMCMC& gp, int num_fidelity,
                                                         const py::list& domain_bounds, const py::list& discrete_pts,
                                                         const py::list& being, int num_pts, int q, int p,
                                                         const py::list& best_so_far, int max_int_steps,
                                                         int max_num_threads, RandomnessSourceContainer& rnd,
                                                         py::dict& status) {
  require_threads(max_num_threads, rnd);
  const int dim = gp.dim_, ps = dim - num_fidelity, M = gp.num_mcmc();
  const auto bounds = full_bounds(domain_bounds, dim);
  const std::vector<double> inner_bounds(bounds.begin(), bounds.begin() + 2 * ps);
  const auto D = to_vec(discrete_pts, static_cast<size_t>(M) * num_pts * ps);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const auto best = to_vec(best_so_far, M);
  const cmoe_gd_params inner = gd_of(optimizer_parameters_inner);
  return mcmc_optimization_common(
      optimizer_parameters, bounds, dim, q, -INFINITY, rnd, status,
      [&](const std::vector<double>& starts, int n, std::vector<double>& vals) {
        int info = 0;
        check(cmoe_kg_eval_mcmc(gp.handles(), M, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts,
                                starts.data(), n, q, Xp.data(), p, max_int_steps, best.data(), rnd.seed0(), nullptr,
                                vals.data(), nullptr, &info), info);
      },
      [&](const cmoe_gd_params& gd, const std::vector<double>& starts, std::vector<double>& out, int& found) {
        int info = 0;
        double bv = 0.0;
        check(cmoe_multistart_kg_mcmc(gp.handles(), M, num_fidelity, &gd, &inner, bounds.data(), inner_bounds.data(),
                                      D.data(), num_pts, starts.data(), gd.num_multistarts, q, Xp.data(), p,
                                      max_int_steps, best.data(), rnd.seed0(), nullptr, out.data(), &bv, &found, &info),
              info);
      });
}

py::list evaluate_KG_mcmc_at_point_list(const GaussianProcessMCMC& gp, int num_fidelity,
                                        const py::object& optimizer_parameters, const py::list& domain_bounds,
                                        const py::list& initial_guesses, const py::list& discrete_being_sampled,
                                        int num_multistarts, int num_pts, int q, int p, const py::list& best_so_far,
                                        int max_int_steps, int max_num_threads, RandomnessSourceContainer& rnd,
                                        py::dict& status) {
  require_threads(max_num_threads, rnd);
  const int dim = gp.dim_, ps = dim - num_fidelity, M = gp.num_mcmc();
  const auto bounds = full_bounds(domain_bounds, dim);
  const std::vector<double> inner_bounds(bounds.begin(), bounds.begin() + 2 * ps);
  // flat [num_mcmc x num_pts x (dim - nf) discrete points ; p x dim points being sampled], as the reference slices it (:349-374)
  const size_t nd = static_cast<size_t>(M) * num_pts * ps;
  const auto both = to_vec(discrete_being_sampled, nd + static_cast<size_t>(p) * dim);
  const std::vector<double> D(both.begin(), both.begin() + nd);
  const std::vector<double> Xp(both.begin() + nd, both.end());
  const auto starts = to_vec(initial_guesses, static_cast<size_t>(num_multistarts) * q * dim);
  const auto best = to_vec(best_so_far, M);
  const cmoe_gd_params inner = gd_of(optimizer_parameters);
  std::vector<double> vals(num_multistarts);
  int info = 0;
  check(cmoe_kg_eval_mcmc(gp.handles(), M, num_fidelity, &inner, inner_bounds.data(), D.data(), num_pts, starts.data(),
                          num_multistarts, q, Xp.data(), p, max_int_steps, best.data(), rnd.seed0(), nullptr, vals.data(),
                          nullptr, &info), info);
  bool found = false;
  for (double v : vals) found = found || (v > -INFINITY);
  status["evaluate_KG_at_point_list"] = found;
  return to_list(vals);
}

double compute_expected_improvement_mcmc(const GaussianProcessMCMC& gp, const py::list& pts, const py::list& being, int q,
                                         int p, int max_int_steps, const py::list& best_so_far,
                                         RandomnessSourceContainer& rnd) {
  const auto X = to_vec(pts, static_cast<size_t>(q) * gp.dim_);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * gp.dim_);
  const auto best = to_vec(best_so_far, gp.num_mcmc());
  double ei = 0.0;
  int info = 0;
  check(cmoe_ei_eval_mcmc(gp.handles(), gp.num_mcmc(), X.data(), 1, q, Xp.data(), p, max_int_steps, best.data(),
                          rnd.seed0(), nullptr, 0, &ei, nullptr, &info), info);
  return ei;
}

py::list compute_grad_expected_improvement_mcmc(const GaussianProcessMCMC& gp, const py::list& pts, const py::list& being,
                                                int q, int p, int max_int_steps, const py::list& best_so_far,
                                                RandomnessSourceContainer& rnd) {
  const auto X = to_vec(pts, static_cast<size_t>(q) * gp.dim_);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * gp.dim_);
  const auto best = to_vec(best_so_far, gp.num_mcmc());
  double ei = 0.0;
  std::vector<double> g(static_cast<size_t>(q) * gp.dim_);
  int info = 0;
  check(cmoe_ei_eval_mcmc(gp.handles(), gp.num_mcmc(), X.data(), 1, q, Xp.data(), p, max_int_steps, best.data(),
                          rnd.seed0(), nullptr, 0, &ei, g.data(), &info), info);
  return to_list(g);
}

py::list multistart_expected_improvement_mcmc_optimization(const py::object& optimizer_parameters,
                                                           const GaussianProcessMCMC& gp, const py::list& domain_bounds,
                                                           const py::list& being, int q, int p,
                                                           const py::list& best_so_far, int max_int_steps,
                                                           int max_num_threads, RandomnessSourceContainer& rnd,
                                                           py::dict& status) {
  require_threads(max_num_threads, rnd);
  const int dim = gp.dim_, M = gp.num_mcmc();
  const auto bounds = full_bounds(domain_bounds, dim);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * dim);
  const auto best = to_vec(best_so_far, M);
  return mcmc_optimization_common(
      optimizer_parameters, bounds, dim, q, 0.0, rnd, status,
      [&](const std::vector<double>& starts, int n, std::vector<double>& vals) {
        int info = 0;
        check(cmoe_ei_eval_mcmc(gp.handles(), M, starts.data(), n, q, Xp.data(), p, max_int_steps, best.data(),
                                rnd.seed0(), nullptr, 1, vals.data(), nullptr, &info), info);
      },
      [&](const cmoe_gd_params& gd, const std::vector<double>& starts, std::vector<double>& out, int& found) {
        int info = 0;
        double bv = 0.0;
        check(cmoe_multistart_ei_mcmc(gp.handles(), M, &gd, bounds.data(), starts.data(), gd.num_multistarts, q,
                                      Xp.data(), p, max_int_steps, best.data(), rnd.seed0(), nullptr, out.data(), &bv,
                                      &found, &info), info);
      });
}

py::list evaluate_EI_mcmc_at_point_list(const GaussianProcessMCMC& gp, const py::list& initial_guesses,
                                        const py::list& being, int num_multistarts, int q, int p,
                                        const py::list& best_so_far, int max_int_steps, int max_num_threads,
                                        RandomnessSourceContainer& rnd, py::dict& status) {
  require_threads(max_num_threads, rnd);
  const auto starts = to_vec(initial_guesses, static_cast<size_t>(num_multistarts) * q * gp.dim_);
  const auto Xp = to_vec(being, static_cast<size_t>(p) * gp.dim_);
  const auto best = to_vec(best_so_far, gp.num_mcmc());
  std::vector<double> vals(num_multistarts);
  int info = 0;
  check(cmoe_ei_eval_mcmc(gp.handles(), gp.num_mcmc(), starts.data(), num_multistarts, q, Xp.data(), p, max_int_steps,
                          best.data(), rnd.seed0(), nullptr, 1, vals.data(), nullptr, &info), info);
  bool found = false;
  for (double v : vals) found = found || (v > 0.0);
  status["evaluate_EI_at_point_list"] = found;
  return to_list(vals);
}

[[noreturn]] void not_on_path(const char* name) {
  PyErr_SetString(g_exc_base, (std::string(name) + " is outside the GPU hot path (SURVEY.md 8f) and is not provided by this build").c_str());
  throw py::error_already_set();
}

[[noreturn]] void raise_exc(PyObject* type, const char* msg) {
  PyErr_SetString(type, msg);
  throw py::error_already_set();
}

// ---- model selection (gpp_python_model_selection.cpp) ---------------------------------------------------------------
// The training data of the model-selection entries in PythonInterfaceInputContainer's order (gpp_python_common.cpp:
// 107-129): points, values, the noise of the entries that take one, then the derivative indices.
struct TrainingData {
  std::vector<double> X, y, noise;
  std::vector<int> derivs;
};

TrainingData training_data(const py::list& points_sampled, const py::list& points_sampled_value, int dim,
                           int num_sampled, const py::list& derivatives, int num_derivatives,
                           const py::list* noise_variance = nullptr) {
  TrainingData d;
  d.X = to_vec(points_sampled, static_cast<size_t>(dim) * num_sampled);
  d.y = to_vec(points_sampled_value, static_cast<size_t>(num_sampled) * (1 + num_derivatives));
  if (noise_variance) d.noise = to_vec(*noise_variance, 1 + num_derivatives);
  d.derivs = to_ivec(derivatives, num_derivatives);
  return d;
}

// (alpha, lengths...) of `hyperparameters` = [alpha, [lengths]], with MaternNu2p5's constructor checks
// (gpp_covariance.cpp:80-91)
std::vector<double> covariance_hyperparameters(const py::list& hyperparameters, int dim) {
  std::vector<double> h{hyperparameters[0].cast<double>()};
  const auto lengths = to_vec(hyperparameters[1].cast<py::list>(), dim);
  if (!(h[0] > 0.0)) raise_exc(g_exc_bounds, "Invalid hyperparameter (alpha).");
  for (double l : lengths)
    if (!(l > 0.0)) raise_exc(g_exc_bounds, "Invalid hyperparameter (length).");
  h.insert(h.end(), lengths.begin(), lengths.end());
  return h;
}

// ---- hyper-parameter optimisation (gpp_python_model_selection.cpp:150-279, 343-376) ---------------------------------
// The inputs of both entries in the reference's order: the input lists, the MaternNu2p5 constructor's checks, then the
// log10 domain copy.  start = (alpha, lengths..., noise by observation type).
struct HyperInputs : TrainingData {
  std::vector<double> start, log_bounds;
  int nh = 0;
};

HyperInputs hyper_inputs(const py::list& hyperparameter_domain, const py::list& points_sampled,
                         const py::list& points_sampled_value, int dim, int num_sampled,
                         const py::list& hyperparameters, const py::list& noise_variance, const py::list& derivatives,
                         int num_derivatives) {
  HyperInputs in;
  static_cast<TrainingData&>(in) = training_data(points_sampled, points_sampled_value, dim, num_sampled, derivatives,
                                                 num_derivatives, &noise_variance);
  in.start = covariance_hyperparameters(hyperparameters, dim);
  in.start.insert(in.start.end(), in.noise.begin(), in.noise.end());
  in.nh = dim + 2 + num_derivatives;
  in.log_bounds = to_vec(hyperparameter_domain, 2 * static_cast<size_t>(in.nh));
  return in;
}

std::vector<double> pow10(std::vector<double> v) {
  for (double& x : v) x = std::pow(10.0, x);
  return v;
}

// multistart_hyperparameter_optimization (:219-279): the MaternNu2p5 kernel hard-wired, as in the reference; starts
// drawn in log10 space from the uniform engine (ConvertFromLogToLinearDomainAndBuildInitialGuesses,
// gpp_model_selection.hpp:841-858).  `max_num_threads` is accepted and ignored: the starts run in parallel on one GPU.
py::list multistart_hyperparameter_optimization(const py::object& optimizer_parameters,
                                                const py::list& hyperparameter_domain, const py::list& points_sampled,
                                                const py::list& points_sampled_value, int dim, int num_sampled,
                                                const py::list& hyperparameters, const py::list& noise_variance,
                                                const py::list& derivatives, int num_derivatives,
                                                int /*max_num_threads*/, RandomnessSourceContainer& rnd,
                                                py::dict status) {
  const HyperInputs in = hyper_inputs(hyperparameter_domain, points_sampled, points_sampled_value, dim, num_sampled,
                                      hyperparameters, noise_variance, derivatives, num_derivatives);
  const auto opt_type = optimizer_parameters.attr("optimizer_type").cast<OptimizerTypes>();
  const auto objective = optimizer_parameters.attr("objective_type").cast<LogLikelihoodTypes>();
  if (objective != LogLikelihoodTypes::kLogMarginalLikelihood)  // leave-one-out is commented out (:258-267)
    raise_exc(g_exc_base, "ERROR: invalid objective type choice. Setting all hyperparameters to 1.0.");
  const int nh = in.nh;
  std::vector<double> best(nh);
  int info = 0;
  if (opt_type == OptimizerTypes::kNull) {
    // LatinHypercubeSearchHyperparameterOptimization (gpp_model_selection.hpp:1342-1363): the start values and the
    // strict-`<` arg-max from -inf of EvaluateLogLikelihoodAtPointList
    const int n = optimizer_parameters.attr("num_random_samples").cast<int>();
    if (n <= 0) raise_exc(g_exc_bounds, "num_multistarts must be > 1");
    const auto starts = pow10(lhc_starts(in.log_bounds, nh, 1, n, rnd.uniform_engine));
    std::vector<double> values(n);
    check(cmoe_log_marginal_likelihood_list(CMOE_KERNEL_MATERN_NU_2P5, starts.data(), n, in.X.data(), in.y.data(),
                                            in.derivs.data(), num_derivatives, dim, num_sampled, 0, values.data(),
                                            &info),
          info);
    double bv = -std::numeric_limits<double>::infinity();
    int bi = 0;
    bool found = false;
    for (int i = 0; i < n; ++i)
      if (bv < values[i]) {
        bv = values[i];
        bi = i;
        found = true;
      }
    std::copy(starts.begin() + static_cast<size_t>(bi) * nh, starts.begin() + static_cast<size_t>(bi + 1) * nh,
              best.begin());
    status["log_marginal_likelihood_lhc_found_update"] = found;
  } else if (opt_type == OptimizerTypes::kGradientDescent) {
    const cmoe_gd_params gd = gd_of(optimizer_parameters);
    if (gd.num_multistarts <= 0) raise_exc(g_exc_bounds, "num_multistarts must be > 1");
    const auto starts = pow10(lhc_starts(in.log_bounds, nh, 1, gd.num_multistarts, rnd.uniform_engine));
    const auto bounds = pow10(in.log_bounds);
    double bv = 0.0;
    int found = 0;
    check(cmoe_hyperparameter_gradient_descent(CMOE_KERNEL_MATERN_NU_2P5, &gd, bounds.data(), starts.data(),
                                               gd.num_multistarts, in.X.data(), in.y.data(), in.derivs.data(),
                                               num_derivatives, dim, num_sampled, 0, best.data(), &bv, &found, nullptr,
                                               nullptr, &info),
          info);
    status["log_marginal_likelihood_gradient_descent_found_update"] = found != 0;
  } else {  // kNewton is commented out at the reference's boundary (:194-206)
    raise_exc(g_exc_base, "ERROR: invalid optimizer choice. Setting all hyperparameters to 1.0.");
  }
  return to_list(best);
}

// restarted_hyperparameter_optimization (:343-376): one start from (hyperparameters, noise_variance) on the linear-space
// box; with max_num_restarts <= 0 the reference's driver returns before writing, so the result is its zero vector.
py::list restarted_hyperparameter_optimization(const py::object& optimizer_parameters,
                                               const py::list& hyperparameter_domain, const py::list& points_sampled,
                                               const py::list& points_sampled_value, int dim, int num_sampled,
                                               const py::list& hyperparameters, const py::list& noise_variance,
                                               const py::list& derivatives, int num_derivatives, py::dict /*status*/) {
  const HyperInputs in = hyper_inputs(hyperparameter_domain, points_sampled, points_sampled_value, dim, num_sampled,
                                      hyperparameters, noise_variance, derivatives, num_derivatives);
  const cmoe_gd_params gd = gd_of(optimizer_parameters);
  std::vector<double> out(in.nh, 0.0), best(in.nh);
  if (gd.max_num_restarts <= 0) return to_list(out);
  const auto bounds = pow10(in.log_bounds);
  int info = 0;
  check(cmoe_hyperparameter_gradient_descent(CMOE_KERNEL_MATERN_NU_2P5, &gd, bounds.data(), in.start.data(), 1,
                                             in.X.data(), in.y.data(), in.derivs.data(), num_derivatives, dim,
                                             num_sampled, 0, best.data(), nullptr, nullptr, out.data(), nullptr, &info),
        info);
  return to_list(out);
}

}  // namespace

// ---- ensemble posterior mean (not in the reference module) ------------------------------------------------------------
// The recommendation step of examples/main.py:243-260 evaluates PosteriorMeanMCMC point by point and runs the Python
// GradientDescentOptimizer on it.  These names do both in one device call each.  `gps` is a GaussianProcessMCMC or a
// Python list of GaussianProcess (what PosteriorMeanMCMC holds, as gp._gaussian_process; the wrapper objects themselves
// are accepted too).
std::vector<const cmoe_gp*> ensemble_handles(const py::object& gps) {
  if (py::isinstance<GaussianProcessMCMC>(gps)) {
    const auto& e = gps.cast<const GaussianProcessMCMC&>();
    return std::vector<const cmoe_gp*>(e.members.begin(), e.members.end());
  }
  std::vector<const cmoe_gp*> h;
  for (const py::handle& item : gps) {
    py::object o = py::reinterpret_borrow<py::object>(item);
    if (!py::isinstance<GaussianProcess>(o) && py::hasattr(o, "_gaussian_process")) o = o.attr("_gaussian_process");
    h.push_back(o.cast<const GaussianProcess&>().h);
  }
  return h;
}

// GPP.GradientDescentParameters or the reference's python_version GradientDescentParameters namedtuple, by attribute
cmoe_gd_params gd_by_attr(const py::object& p) {
  auto get_int = [&](const char* n) { return py::hasattr(p, n) ? p.attr(n).cast<int>() : 0; };
  auto get_dbl = [&](const char* n) { return py::hasattr(p, n) ? p.attr(n).cast<double>() : 0.0; };
  return cmoe_gd_params{get_int("num_multistarts"), p.attr("max_num_steps").cast<int>(), get_int("max_num_restarts"),
                        p.attr("num_steps_averaged").cast<int>(), p.attr("gamma").cast<double>(),
                        p.attr("pre_mult").cast<double>(), p.attr("max_relative_change").cast<double>(),
                        get_dbl("tolerance")};
}

int ensemble_dim(const std::vector<const cmoe_gp*>& h) { return h.empty() ? 0 : cmoe_gp_dim(h[0]); }

// values of PosteriorMeanMCMC.compute_objective_function, -(1/M) sum_m mu_m, at num_points points [num_points][dim-nf]
py::list compute_posterior_mean_mcmc_of_points(const py::object& gps, int num_fidelity, const py::list& pts,
                                               int num_points) {
  const auto h = ensemble_handles(gps);
  const auto flat = to_vec(pts, static_cast<size_t>(std::max(num_points, 0)) * std::max(ensemble_dim(h) - num_fidelity, 0));
  std::vector<double> v(std::max(num_points, 0));
  int info = 0;
  check(cmoe_posterior_mean_mcmc(h.data(), static_cast<int>(h.size()), num_fidelity, flat.data(), num_points, v.data(),
                                 nullptr, nullptr, &info), info);
  return to_list(v);
}

// compute_grad_objective_function of PosteriorMeanMCMC at every point, flat [num_points][dim-nf]
py::list compute_grad_posterior_mean_mcmc_of_points(const py::object& gps, int num_fidelity, const py::list& pts,
                                                    int num_points) {
  const auto h = ensemble_handles(gps);
  const size_t ps = std::max(ensemble_dim(h) - num_fidelity, 0), n = std::max(num_points, 0);
  const auto flat = to_vec(pts, n * ps);
  std::vector<double> v(n), g(n * ps);
  int info = 0;
  check(cmoe_posterior_mean_mcmc(h.data(), static_cast<int>(h.size()), num_fidelity, flat.data(), num_points, v.data(),
                                 g.data(), nullptr, &info), info);
  return to_list(g);
}

// multistart_optimize(GradientDescentOptimizer(RepeatedDomain(1, box), PosteriorMeanMCMC, params), starts):
// (best_point [dim-nf], function_values [num_starts]), as python_version.optimization.multistart_optimize returns them
py::tuple posterior_mean_mcmc_optimization(const py::object& gps, int num_fidelity, const py::object& optimizer_parameters,
                                           const py::list& domain_bounds, const py::list& starting_points,
                                           int num_starts) {
  const auto h = ensemble_handles(gps);
  const size_t ps = std::max(ensemble_dim(h) - num_fidelity, 0), n = std::max(num_starts, 0);
  const auto bounds = to_vec(domain_bounds, 2 * ps);
  const auto starts = to_vec(starting_points, n * ps);
  const cmoe_gd_params gd = gd_by_attr(optimizer_parameters);
  std::vector<double> vals(n), best(ps);
  double best_value = 0.0;
  int info = 0;
  check(cmoe_posterior_mean_mcmc_optimization(h.data(), static_cast<int>(h.size()), num_fidelity, &gd, bounds.data(),
                                              starts.data(), num_starts, nullptr, vals.data(), best.data(), &best_value,
                                              &info), info);
  return py::make_tuple(to_list(best), to_list(vals));
}

// The discretisation step of examples/main.py:172-197 for every member at once (not in the reference module):
// screen `points` (flat [num_points][dim-nf], shared by the members) and, if include_sampled, each member's own sampled
// points by posterior mean, descend from the argmin with posterior_mean_optimization's line search, keep the start if
// the descent ended higher.  Returns (discrete_pts flat [M][num_shared + 1][dim-nf] = shared_discrete_pts followed by
// the member's optimum, best_so_far [M] as KnowledgeGradientMCMC computes it, optima flat [M][dim-nf]).
py::tuple posterior_mean_optima_mcmc(const py::object& gps, int num_fidelity, const py::object& optimizer_parameters,
                                     const py::list& domain_bounds, const py::list& points, int num_points,
                                     const py::list& shared_discrete_pts, int num_shared, bool include_sampled) {
  const auto h = ensemble_handles(gps);
  const size_t ps = std::max(ensemble_dim(h) - num_fidelity, 0), n = std::max(num_points, 0), ns = std::max(num_shared, 0);
  const auto bounds = to_vec(domain_bounds, 2 * ps);
  const auto pts = to_vec(points, n * ps);
  const auto shared = to_vec(shared_discrete_pts, ns * ps);
  const cmoe_gd_params gd = gd_by_attr(optimizer_parameters);
  std::vector<double> optima(h.size() * ps), disc(h.size() * (ns + 1) * ps), best(h.size());
  int info = 0;
  check(cmoe_posterior_mean_optima_mcmc(h.data(), static_cast<int>(h.size()), num_fidelity, &gd, bounds.data(),
                                        pts.data(), num_points, 0, include_sampled ? 1 : 0,
                                        ns ? shared.data() : nullptr, num_shared, optima.data(), nullptr, nullptr,
                                        nullptr, nullptr, disc.data(), best.data(), &info), info);
  return py::make_tuple(to_list(disc), to_list(best), to_list(optima));
}

PYBIND11_MODULE(GPP, m) {
  m.doc() = "H100-native drop-in for moe.build.GPP (GP posterior + MC acquisition hot path)";
  g_exc_base = PyErr_NewExceptionWithDoc("GPP.OptimalLearningException",
                                         "Base exception class for errors raised from the optimal_learning library.",
                                         PyExc_Exception, nullptr);
  g_exc_bounds = PyErr_NewExceptionWithDoc("GPP.BoundsException", "value not in range [min, max].", g_exc_base, nullptr);
  g_exc_invalid = PyErr_NewExceptionWithDoc("GPP.InvalidValueException", "value != truth (+/- tolerance)", g_exc_base, nullptr);
  g_exc_singular = PyErr_NewExceptionWithDoc("GPP.SingularMatrixException", "num_rows X num_cols matrix is singular", g_exc_base, nullptr);
  m.attr("OptimalLearningException") = py::handle(g_exc_base);
  m.attr("BoundsException") = py::handle(g_exc_bounds);
  m.attr("InvalidValueException") = py::handle(g_exc_invalid);
  m.attr("SingularMatrixException") = py::handle(g_exc_singular);

  py::enum_<OptimizerTypes>(m, "OptimizerTypes")
      .value("null", OptimizerTypes::kNull)
      .value("gradient_descent", OptimizerTypes::kGradientDescent)
      .value("newton", OptimizerTypes::kNewton);
  py::enum_<DomainTypes>(m, "DomainTypes")
      .value("tensor_product", DomainTypes::kTensorProduct)
      .value("simplex", DomainTypes::kSimplex);
  py::enum_<LogLikelihoodTypes>(m, "LogLikelihoodTypes")
      .value("log_marginal_likelihood", LogLikelihoodTypes::kLogMarginalLikelihood)
      .value("leave_one_out_log_likelihood", LogLikelihoodTypes::kLeaveOneOutLogLikelihood);

  py::class_<GradientDescentParameters>(m, "GradientDescentParameters")
      .def(py::init<int, int, int, int, double, double, double, double>())
      .def_property("num_multistarts", [](const GradientDescentParameters& s) { return s.p.num_multistarts; },
                    [](GradientDescentParameters& s, int v) { s.p.num_multistarts = v; })
      .def_property("max_num_steps", [](const GradientDescentParameters& s) { return s.p.max_num_steps; },
                    [](GradientDescentParameters& s, int v) { s.p.max_num_steps = v; })
      .def_property("max_num_restarts", [](const GradientDescentParameters& s) { return s.p.max_num_restarts; },
                    [](GradientDescentParameters& s, int v) { s.p.max_num_restarts = v; })
      .def_property("num_steps_averaged", [](const GradientDescentParameters& s) { return s.p.num_steps_averaged; },
                    [](GradientDescentParameters& s, int v) { s.p.num_steps_averaged = v; })
      .def_property("gamma", [](const GradientDescentParameters& s) { return s.p.gamma; },
                    [](GradientDescentParameters& s, double v) { s.p.gamma = v; })
      .def_property("pre_mult", [](const GradientDescentParameters& s) { return s.p.pre_mult; },
                    [](GradientDescentParameters& s, double v) { s.p.pre_mult = v; })
      .def_property("max_relative_change", [](const GradientDescentParameters& s) { return s.p.max_relative_change; },
                    [](GradientDescentParameters& s, double v) { s.p.max_relative_change = v; })
      .def_property("tolerance", [](const GradientDescentParameters& s) { return s.p.tolerance; },
                    [](GradientDescentParameters& s, double v) { s.p.tolerance = v; });
  py::class_<NewtonParameters>(m, "NewtonParameters")
      .def(py::init<int, int, double, double, double, double>())
      .def_readwrite("num_multistarts", &NewtonParameters::num_multistarts)
      .def_readwrite("max_num_steps", &NewtonParameters::max_num_steps)
      .def_readwrite("gamma", &NewtonParameters::gamma)
      .def_readwrite("time_factor", &NewtonParameters::time_factor)
      .def_readwrite("max_relative_change", &NewtonParameters::max_relative_change)
      .def_readwrite("tolerance", &NewtonParameters::tolerance);
  py::class_<RandomnessSourceContainer>(m, "RandomnessSourceContainer")
      .def(py::init<int>())
      .def("SetExplicitUniformGeneratorSeed", &RandomnessSourceContainer::SetExplicitUniformGeneratorSeed)
      .def("SetRandomizedUniformGeneratorSeed", &RandomnessSourceContainer::SetRandomizedUniformGeneratorSeed)
      .def("ResetUniformRNGSeed", &RandomnessSourceContainer::ResetUniformGeneratorState)
      .def("SetExplicitNormalRNGSeed", &RandomnessSourceContainer::SetExplicitNormalRNGSeed)
      .def("SetRandomizedNormalRNGSeed", &RandomnessSourceContainer::SetRandomizedNormalRNGSeed)
      .def("SetNormalRNGSeedPythonList", &RandomnessSourceContainer::SetNormalRNGSeedPythonList)
      .def("ResetNormalRNGSeed", &RandomnessSourceContainer::ResetNormalRNGState)
      .def("PrintState", &RandomnessSourceContainer::PrintState);

  py::class_<GaussianProcess>(m, "GaussianProcess")
      .def(py::init<const py::list&, const py::list&, const py::list&, const py::list&, const py::list&, int, int, int,
                    const std::string&, int>(),
           py::arg("hyperparameters"), py::arg("points_sampled"), py::arg("points_sampled_value"),
           py::arg("noise_variance"), py::arg("derivatives"), py::arg("num_derivatives"), py::arg("dim"),
           py::arg("num_sampled"), py::arg("kernel") = "matern52", py::arg("which_gpu") = 0)
      .def_property_readonly("dim", &GaussianProcess::dim)
      .def_property_readonly("num_sampled", &GaussianProcess::num_sampled)
      .def("compute_mean_of_points", &GaussianProcess::mean)
      .def("compute_mean_of_additional_points", &GaussianProcess::mean)
      .def("compute_grad_mean_of_points", &GaussianProcess::grad_mean)
      .def("compute_variance_of_points", &GaussianProcess::variance)
      .def("compute_cholesky_variance_of_points", &GaussianProcess::chol_variance)
      .def("compute_grad_variance_of_points",
           [](const GaussianProcess& g, const py::list& pts, int n, int nd) { return g.grad_variance(pts, n, nd, false); })
      .def("compute_grad_cholesky_variance_of_points",
           [](const GaussianProcess& g, const py::list& pts, int n, int nd) { return g.grad_variance(pts, n, nd, true); })
      .def("add_sampled_points", &GaussianProcess::add_sampled_points)
      .def("sample_point_from_gp", &GaussianProcess::sample_point_from_gp, py::arg("point_to_sample"))
      .def("sample_global_optima", &GaussianProcess::sample_global_optima, py::arg("num_optima"),
           py::arg("inner_number"), py::arg("domain_bounds"))
      .def("set_explicit_seed", &GaussianProcess::set_explicit_seed, py::arg("seed"))
      .def("set_randomized_seed", &GaussianProcess::set_randomized_seed, py::arg("seed"))
      .def("reset_to_most_recent_seed", &GaussianProcess::reset_to_most_recent_seed)
      .def("print_historical_data", [](GaussianProcess&) {});

  m.def("compute_expected_improvement", &compute_expected_improvement);
  m.def("compute_grad_expected_improvement", &compute_grad_expected_improvement);
  m.def("multistart_expected_improvement_optimization", &multistart_expected_improvement_optimization);
  m.def("evaluate_EI_at_point_list", &evaluate_EI_at_point_list);
  m.def("compute_posterior_mean", &compute_posterior_mean);
  m.def("compute_grad_posterior_mean", &compute_grad_posterior_mean);
  m.def("compute_posterior_mean_of_points", &compute_posterior_mean_of_points);
  m.def("compute_knowledge_gradient", &compute_knowledge_gradient);
  m.def("compute_grad_knowledge_gradient", &compute_grad_knowledge_gradient);
  m.def("multistart_knowledge_gradient_optimization", &multistart_knowledge_gradient_optimization);
  m.def("evaluate_KG_at_point_list", &evaluate_KG_at_point_list);
  m.def("posterior_mean_optimization",
        [](const GaussianProcess& gp, int num_fidelity, const py::object& optimizer_parameters,
           const py::list& domain_bounds, const py::list& initial_guess, py::dict& status) -> py::list {
          const int ps = gp.dim_ - num_fidelity;
          const auto bounds = to_vec(domain_bounds, 2 * static_cast<size_t>(ps));
          const auto x0 = to_vec(initial_guess, ps);
          const cmoe_gd_params gd = gd_of(optimizer_parameters);
          std::vector<double> best(ps, 0.0);
          double value = 0.0;
          int found = 0;
          check(cmoe_posterior_mean_optimization(gp.h, num_fidelity, &gd, bounds.data(), x0.data(), best.data(), &value,
                                                 &found));
          (void)status;  // the reference leaves `status` untouched for this entry point (:306-350)
          return to_list(best);
        });
  py::class_<GaussianProcessMCMC>(m, "GaussianProcessMCMC")
      .def(py::init<const py::list&, const py::list&, const py::list&, const py::list&, const py::list&, int, int, int,
                    int, const std::string&, int>(),
           py::arg("hyperparameters_list"), py::arg("noise_variance_list"), py::arg("points_sampled"),
           py::arg("points_sampled_value"), py::arg("derivatives"), py::arg("num_mcmc"), py::arg("num_derivatives"),
           py::arg("dim"), py::arg("num_sampled"), py::arg("kernel") = "matern52", py::arg("which_gpu") = 0)
      .def_property_readonly("dim", [](const GaussianProcessMCMC& g) { return g.dim_; })
      .def_property_readonly("num_mcmc", &GaussianProcessMCMC::num_mcmc)
      .def_property_readonly("num_sampled", [](const GaussianProcessMCMC& g) { return g.num_sampled_; });
  m.def("compute_knowledge_gradient_mcmc", &compute_knowledge_gradient_mcmc);
  m.def("compute_grad_knowledge_gradient_mcmc", &compute_grad_knowledge_gradient_mcmc);
  m.def("multistart_knowledge_gradient_mcmc_optimization", &multistart_knowledge_gradient_mcmc_optimization);
  m.def("evaluate_KG_mcmc_at_point_list", &evaluate_KG_mcmc_at_point_list);
  m.def("compute_expected_improvement_mcmc", &compute_expected_improvement_mcmc);
  m.def("compute_grad_expected_improvement_mcmc", &compute_grad_expected_improvement_mcmc);
  m.def("multistart_expected_improvement_mcmc_optimization", &multistart_expected_improvement_mcmc_optimization);
  m.def("evaluate_EI_mcmc_at_point_list", &evaluate_EI_mcmc_at_point_list);
  m.def("compute_posterior_mean_mcmc_of_points", &compute_posterior_mean_mcmc_of_points, py::arg("gps"),
        py::arg("num_fidelity"), py::arg("points"), py::arg("num_points"));
  m.def("compute_grad_posterior_mean_mcmc_of_points", &compute_grad_posterior_mean_mcmc_of_points, py::arg("gps"),
        py::arg("num_fidelity"), py::arg("points"), py::arg("num_points"));
  m.def("posterior_mean_mcmc_optimization", &posterior_mean_mcmc_optimization, py::arg("gps"), py::arg("num_fidelity"),
        py::arg("optimizer_parameters"), py::arg("domain_bounds"), py::arg("starting_points"), py::arg("num_starts"));
  m.def("posterior_mean_optima_mcmc", &posterior_mean_optima_mcmc, py::arg("gps"), py::arg("num_fidelity"),
        py::arg("optimizer_parameters"), py::arg("domain_bounds"), py::arg("points"), py::arg("num_points"),
        py::arg("shared_discrete_pts"), py::arg("num_shared"), py::arg("include_sampled") = true);
  // names of the reference module whose arguments may match none of the signatures below (model selection): present, so
  // that an unmodified front end fails with the library's own exception class and a clear message rather than a
  // TypeError
  // compute_log_likelihood(points_sampled, points_sampled_value, dim, num_sampled, objective_type, hyperparameters,
  //                        derivatives, num_derivatives, noise_variance)   gpp_python_model_selection.cpp:43-87
  m.def("compute_log_likelihood",
        [](const py::list& points_sampled, const py::list& points_sampled_value, int dim, int num_sampled,
           LogLikelihoodTypes objective_type, const py::list& hyperparameters, const py::list& derivatives,
           int num_derivatives, const py::list& noise_variance) -> double {
          if (objective_type != LogLikelihoodTypes::kLogMarginalLikelihood) {
            PyErr_SetString(g_exc_base, "ERROR: invalid objective mode choice. Setting log likelihood to -DBL_MAX.");
            throw py::error_already_set();
          }
          const double alpha = hyperparameters[0].cast<double>();
          const auto lengths = to_vec(hyperparameters[1].cast<py::list>(), dim);
          const auto d = training_data(points_sampled, points_sampled_value, dim, num_sampled, derivatives,
                                       num_derivatives, &noise_variance);
          double value = 0.0;
          int info = 0;
          // the reference's Python boundary hard-wires MaternNu2p5 here as well (:57)
          check(cmoe_log_marginal_likelihood(CMOE_KERNEL_MATERN_NU_2P5, alpha, lengths.data(), d.X.data(), d.y.data(),
                                             d.noise.data(), d.derivs.data(), num_derivatives, dim, num_sampled, 0,
                                             &value, &info), info);
          return value;
        });
  // compute_hyperparameter_grad_log_likelihood(... same arguments ...)   gpp_python_model_selection.cpp:89-140
  m.def("compute_hyperparameter_grad_log_likelihood",
        [](const py::list& points_sampled, const py::list& points_sampled_value, int dim, int num_sampled,
           LogLikelihoodTypes objective_type, const py::list& hyperparameters, const py::list& derivatives,
           int num_derivatives, const py::list& noise_variance) -> py::list {
          if (objective_type != LogLikelihoodTypes::kLogMarginalLikelihood) {
            PyErr_SetString(g_exc_base, "ERROR: invalid objective mode choice. Setting all gradients to DBL_MAX.");
            throw py::error_already_set();
          }
          const double alpha = hyperparameters[0].cast<double>();
          const auto lengths = to_vec(hyperparameters[1].cast<py::list>(), dim);
          const auto d = training_data(points_sampled, points_sampled_value, dim, num_sampled, derivatives,
                                       num_derivatives, &noise_variance);
          std::vector<double> grad(static_cast<size_t>(dim) + 2 + num_derivatives);
          int info = 0;
          check(cmoe_grad_log_marginal_likelihood(CMOE_KERNEL_MATERN_NU_2P5, alpha, lengths.data(), d.X.data(),
                                                  d.y.data(), d.noise.data(), d.derivs.data(), num_derivatives, dim,
                                                  num_sampled, 0, grad.data(), &info), info);
          return to_list(grad);
        });
  // evaluate_log_likelihood_at_hyperparameter_list(hyperparameter_list, points_sampled, points_sampled_value, dim,
  //     num_sampled, objective_mode, hyperparameters, noise_variance, derivatives, num_derivatives, num_multistarts,
  //     max_num_threads, status)                                    gpp_python_model_selection.cpp:281-341, 520-556
  // One device call for the whole list (cmoe_log_marginal_likelihood_list); `max_num_threads` is accepted and ignored
  // (the sets run in parallel on the GPU).  Each set is (alpha, lengths..., noise by observation type).
  m.def("evaluate_log_likelihood_at_hyperparameter_list",
        [](const py::list& hyperparameter_list, const py::list& points_sampled, const py::list& points_sampled_value,
           int dim, int num_sampled, LogLikelihoodTypes objective_mode, const py::list& hyperparameters,
           const py::list& noise_variance, const py::list& derivatives, int num_derivatives, int num_multistarts,
           int /*max_num_threads*/, py::dict status) -> py::list {
          // the reference's order: input lists, covariance constructor, list copy, objective mode, then the driver
          const auto d = training_data(points_sampled, points_sampled_value, dim, num_sampled, derivatives,
                                       num_derivatives, &noise_variance);
          covariance_hyperparameters(hyperparameters, dim);
          const size_t nh = static_cast<size_t>(dim) + 2 + num_derivatives;
          const auto hypers = to_vec(hyperparameter_list, nh * std::max(num_multistarts, 0));
          if (objective_mode != LogLikelihoodTypes::kLogMarginalLikelihood) {  // leave-one-out is commented out (:323-333)
            status["evaluate_invalid_log_likelihood_at_hyperparameter_list"] = false;
            PyErr_SetString(g_exc_base, "ERROR: invalid objective mode choice. Setting all results to -DBL_MAX.");
            throw py::error_already_set();
          }
          if (num_multistarts < 1) {  // gpp_model_selection.hpp:1285-1287
            PyErr_SetString(g_exc_bounds, "num_multistarts must be > 1");
            throw py::error_already_set();
          }
          std::vector<double> values(num_multistarts);
          int info = 0;
          // MaternNu2p5 hard-wired, as the reference's boundary does (:297)
          check(cmoe_log_marginal_likelihood_list(CMOE_KERNEL_MATERN_NU_2P5, hypers.data(), num_multistarts,
                                                  d.X.data(), d.y.data(), d.derivs.data(), num_derivatives, dim,
                                                  num_sampled, 0, values.data(), &info),
                info);
          // found_flag of MultistartOptimize: some value beat the initial -inf with a strict < (gpp_optimization.hpp:1511)
          const bool found = std::any_of(values.begin(), values.end(),
                                         [](double v) { return -std::numeric_limits<double>::infinity() < v; });
          status["evaluate_log_marginal_likelihood_at_hyperparameter_list"] = found;
          return to_list(values);
        });
  // multistart_hyperparameter_optimization(optimizer_parameters, hyperparameter_domain, points_sampled,
  //     points_sampled_value, dim, num_sampled, hyperparameters, noise_variance, derivatives, num_derivatives,
  //     max_num_threads, randomness_source, status)                              gpp_python_model_selection.cpp:219-279
  // restarted_hyperparameter_optimization(optimizer_parameters, hyperparameter_domain, points_sampled,
  //     points_sampled_value, dim, num_sampled, hyperparameters, noise_variance, derivatives, num_derivatives,
  //     status)                                                                  gpp_python_model_selection.cpp:343-376
  // A call that matches neither signature reaches the catch-all overload and raises the library's own exception.
  m.def("multistart_hyperparameter_optimization", &multistart_hyperparameter_optimization);
  m.def("restarted_hyperparameter_optimization", &restarted_hyperparameter_optimization);
  for (const char* name : {"multistart_hyperparameter_optimization", "restarted_hyperparameter_optimization"}) {
    const std::string n(name);
    m.def(name, [n](const py::args&, const py::kwargs&) -> py::object {
      raise_exc(g_exc_base, (n + ": the arguments match no signature of the reference's function").c_str());
    });
  }
  // sample_hyperparameters_mcmc(points_sampled, points_sampled_value, dim, num_sampled, derivatives, num_derivatives,
  //     initial_positions, num_walkers, num_steps, noisy, use_default_prior, seed, first_step)
  // Not in the reference module: the emcee chain of GaussianProcessLogLikelihoodMCMC.train (log_likelihood_mcmc.py:
  // 170-239) in one device call (cmoe_hyperparameter_mcmc, DESIGN.md K12).  Walkers are log-scale
  // [log alpha, log lengths..., log noise...]; returns (positions, log_probabilities) as flat lists.
  m.def("sample_hyperparameters_mcmc",
        [](const py::list& points_sampled, const py::list& points_sampled_value, int dim, int num_sampled,
           const py::list& derivatives, int num_derivatives, const py::list& initial_positions, int num_walkers,
           int num_steps, bool noisy, bool use_default_prior, uint64_t seed, uint64_t first_step) -> py::tuple {
          const auto d =
              training_data(points_sampled, points_sampled_value, dim, num_sampled, derivatives, num_derivatives);
          const size_t nh = static_cast<size_t>(dim) + 2 + num_derivatives;
          const auto p0 = to_vec(initial_positions, nh * std::max(num_walkers, 0));
          std::vector<double> pos(p0.size()), lnp(std::max(num_walkers, 0));
          int info = 0;
          // MaternNu2p5 hard-wired, as compute_log_likelihood's boundary does
          check(cmoe_hyperparameter_mcmc(CMOE_KERNEL_MATERN_NU_2P5,
                                         use_default_prior ? CMOE_HYPER_PRIOR_DEFAULT : CMOE_HYPER_PRIOR_NONE,
                                         noisy ? 1 : 0, p0.data(), num_walkers, num_steps, seed, first_step, nullptr,
                                         d.X.data(), d.y.data(), d.derivs.data(), num_derivatives, dim, num_sampled, 0,
                                         pos.data(), lnp.data(), &info),
                info);
          return py::make_tuple(to_list(pos), to_list(lnp));
        },
        py::arg("points_sampled"), py::arg("points_sampled_value"), py::arg("dim"), py::arg("num_sampled"),
        py::arg("derivatives"), py::arg("num_derivatives"), py::arg("initial_positions"), py::arg("num_walkers"),
        py::arg("num_steps"), py::arg("noisy"), py::arg("use_default_prior"), py::arg("seed"),
        py::arg("first_step") = 0);
  // hyperparameter_map_optimization(points_sampled, points_sampled_value, dim, num_sampled, derivatives,
  //     num_derivatives, initial_positions, num_starts, noisy, use_default_prior, gtol, max_iterations)
  // Not in the reference module: GaussianProcessLogLikelihoodMCMC.optimize (log_likelihood_mcmc.py:241-275), BFGS on
  // -compute_log_likelihood from every start in one device call (cmoe_hyperparameter_map, DESIGN.md K19), with the
  // analytic gradient.  Starts are log-scale [log alpha, log lengths..., log noise...]; max_iterations = 0 is scipy's
  // 200 nh.  Returns (positions, values, status) as flat lists; values are the negative log-likelihood.
  m.def("hyperparameter_map_optimization",
        [](const py::list& points_sampled, const py::list& points_sampled_value, int dim, int num_sampled,
           const py::list& derivatives, int num_derivatives, const py::list& initial_positions, int num_starts,
           bool noisy, bool use_default_prior, double gtol, int max_iterations) -> py::tuple {
          const auto d =
              training_data(points_sampled, points_sampled_value, dim, num_sampled, derivatives, num_derivatives);
          const size_t nh = static_cast<size_t>(dim) + 2 + num_derivatives, S = std::max(num_starts, 0);
          const auto p0 = to_vec(initial_positions, nh * S);
          std::vector<double> pos(p0.size()), grads(p0.size()), vals(S);
          std::vector<int> iters(S), evals(S), status(S);
          const cmoe_map_opts opts{gtol, max_iterations};
          int info = 0;
          // MaternNu2p5 hard-wired, as compute_log_likelihood's boundary does
          check(cmoe_hyperparameter_map(CMOE_KERNEL_MATERN_NU_2P5,
                                        use_default_prior ? CMOE_HYPER_PRIOR_DEFAULT : CMOE_HYPER_PRIOR_NONE,
                                        noisy ? 1 : 0, p0.data(), num_starts, &opts, d.X.data(), d.y.data(),
                                        d.derivs.data(), num_derivatives, dim, num_sampled, 0, pos.data(), vals.data(),
                                        grads.data(), iters.data(), evals.data(), status.data(), &info),
                info);
          py::list st;
          for (int v : status) st.append(v);
          return py::make_tuple(to_list(pos), to_list(vals), st);
        },
        py::arg("points_sampled"), py::arg("points_sampled_value"), py::arg("dim"), py::arg("num_sampled"),
        py::arg("derivatives"), py::arg("num_derivatives"), py::arg("initial_positions"), py::arg("num_starts"),
        py::arg("noisy"), py::arg("use_default_prior"), py::arg("gtol") = 1.0e-5, py::arg("max_iterations") = 0);
  // lower_confidence_bound_optimization(gaussian_process, candidate_pts, num_candidates, num_to_sample)
  // Not in the reference module: the body of lower_confidence_bound.py:52-80 in one device call (cmoe_lcb_select,
  // DESIGN.md K13).  `gaussian_process` is a GaussianProcess or a wrapper holding one as `_gaussian_process`;
  // candidate_pts is the flat [num_candidates][dim] list.  Returns the num_to_sample * dim coordinates as a flat list.
  // The GP is left unchanged (the reference leaves its fantasy points in it).
  m.def("lower_confidence_bound_optimization",
        [](const py::object& gaussian_process, const py::list& candidate_pts, int num_candidates,
           int num_to_sample) -> py::list {
          py::object o = gaussian_process;
          if (!py::isinstance<GaussianProcess>(o) && py::hasattr(o, "_gaussian_process")) o = o.attr("_gaussian_process");
          const GaussianProcess& gp = o.cast<const GaussianProcess&>();
          const int dim = gp.dim();
          const auto P = to_vec(candidate_pts, static_cast<size_t>(std::max(num_candidates, 0)) * dim);
          std::vector<int> sel(std::max(num_to_sample, 0));
          int info = 0;
          check(cmoe_lcb_select(gp.h, P.data(), num_candidates, num_to_sample, sel.data(), nullptr, nullptr, nullptr,
                                &info),
                info);
          std::vector<double> out(sel.size() * dim);
          for (size_t i = 0; i < sel.size(); ++i)
            std::copy(P.begin() + static_cast<size_t>(sel[i]) * dim, P.begin() + static_cast<size_t>(sel[i] + 1) * dim,
                      out.begin() + i * dim);
          return to_list(out);
        },
        py::arg("gaussian_process"), py::arg("candidate_pts"), py::arg("num_candidates"), py::arg("num_to_sample"));
  // sample_from_global_optima(gaussian_process, num_features, domain_bounds, grid, num_grid, num_points)
  // Not in the reference module: random_features.sample_from_global_optima (random_features.py:171-175) in one device
  // call (cmoe_gp_sample_rff_optima, DESIGN.md K14).  `gaussian_process` is a GaussianProcess or a wrapper holding one
  // as `_gaussian_process`; domain_bounds is the flat [dim][2] list, grid the flat [num_grid][dim] list.  Uses the GP's
  // (seed, next draw), one draw per point, as sample_global_optima does.  Returns the num_points * dim coordinates as
  // a flat list.  The GP is not modified.
  m.def("sample_from_global_optima",
        [](const py::object& gaussian_process, int num_features, const py::list& domain_bounds, const py::list& grid,
           int num_grid, int num_points) -> py::list {
          py::object o = gaussian_process;
          if (!py::isinstance<GaussianProcess>(o) && py::hasattr(o, "_gaussian_process")) o = o.attr("_gaussian_process");
          GaussianProcess& gp = o.cast<GaussianProcess&>();
          const int dim = gp.dim();
          const auto B = to_vec(domain_bounds, 2 * static_cast<size_t>(dim));
          const auto Gr = to_vec(grid, static_cast<size_t>(std::max(num_grid, 0)) * dim);
          std::vector<double> out(static_cast<size_t>(std::max(num_points, 0)) * dim), vals(std::max(num_points, 0));
          int info = 0;
          check(cmoe_gp_sample_rff_optima(gp.h, num_features, num_points, B.data(), Gr.data(), num_grid, gp.seed_,
                                          gp.next_draw_, nullptr, out.data(), vals.data(), nullptr, nullptr, nullptr,
                                          &info),
                info);
          gp.next_draw_ += static_cast<uint64_t>(num_points);
          return to_list(out);
        },
        py::arg("gaussian_process"), py::arg("num_features"), py::arg("domain_bounds"), py::arg("grid"),
        py::arg("num_grid"), py::arg("num_points"));
  // sample_from_global_optima_kernel_matched: as sample_from_global_optima, with frequencies drawn from the GP's own
  // kernel (CMOE_RFF_SPECTRAL_KERNEL: the Student-t mixture for Matern-5/2; a SquareExponential GP gives the same
  // points as sample_from_global_optima).
  m.def("sample_from_global_optima_kernel_matched",
        [](const py::object& gaussian_process, int num_features, const py::list& domain_bounds, const py::list& grid,
           int num_grid, int num_points) -> py::list {
          GaussianProcess& gp = unwrap_gp(gaussian_process);
          const int dim = gp.dim();
          const auto B = to_vec(domain_bounds, 2 * static_cast<size_t>(dim));
          const auto Gr = to_vec(grid, static_cast<size_t>(std::max(num_grid, 0)) * dim);
          std::vector<double> out(static_cast<size_t>(std::max(num_points, 0)) * dim), vals(std::max(num_points, 0));
          const cmoe_rff_opts opts{CMOE_RFF_SPECTRAL_KERNEL, nullptr};
          int info = 0;
          check(cmoe_gp_sample_rff_optima_ex(gp.h, num_features, num_points, B.data(), Gr.data(), num_grid, gp.seed_,
                                             gp.next_draw_, nullptr, &opts, out.data(), vals.data(), nullptr, nullptr,
                                             nullptr, &info),
                info);
          gp.next_draw_ += static_cast<uint64_t>(num_points);
          return to_list(out);
        },
        py::arg("gaussian_process"), py::arg("num_features"), py::arg("domain_bounds"), py::arg("grid"),
        py::arg("num_grid"), py::arg("num_points"));
  // sample_gp_with_random_features(gaussian_process, num_features, kernel_matched=False)
  // random_features.sample_gp_with_random_features (random_features.py:29-133) through cmoe_gp_sample_rff_functions:
  // one draw of the GP's (seed, next draw).  Returns a RandomFeatureSample, callable as the reference's
  // wrapper(x, gradient) and evaluated on the device (cmoe_rff_evaluate).
  py::class_<RandomFeatureSample>(m, "RandomFeatureSample")
      .def("__call__", &RandomFeatureSample::call, py::arg("x"), py::arg("gradient") = false)
      .def_property_readonly("omega", [](const RandomFeatureSample& s) { return s.array(s.omega, {s.F, s.dim}); })
      .def_property_readonly("b", [](const RandomFeatureSample& s) { return s.array(s.b, {s.F}); })
      .def_property_readonly("theta", [](const RandomFeatureSample& s) { return s.array(s.theta, {s.F}); })
      .def_readonly("c", &RandomFeatureSample::c);
  m.def("sample_gp_with_random_features",
        [](const py::object& gaussian_process, int num_features, bool kernel_matched) {
          GaussianProcess& gp = unwrap_gp(gaussian_process);
          RandomFeatureSample r;
          r.dim = gp.dim();
          r.F = num_features;
          r.device = cmoe_gp_device(gp.h);
          const size_t F = static_cast<size_t>(std::max(num_features, 0));
          r.omega.resize(F * r.dim);
          r.b.resize(F);
          r.theta.resize(F);
          const cmoe_rff_opts opts{kernel_matched ? CMOE_RFF_SPECTRAL_KERNEL : CMOE_RFF_SPECTRAL_REFERENCE, nullptr};
          int info = 0;
          check(cmoe_gp_sample_rff_functions(gp.h, num_features, 1, gp.seed_, gp.next_draw_, nullptr, &opts,
                                             r.omega.data(), r.b.data(), r.theta.data(), &info),
                info);
          gp.next_draw_ += 1;
          r.c = std::sqrt(2.0 * gp.alpha_ / num_features);
          return r;
        },
        py::arg("gaussian_process"), py::arg("num_features"), py::arg("kernel_matched") = false);
  // heuristic_expected_improvement_optimization(optimizer_parameters, gaussian_process, domain_bounds,
  //     estimation_policy, num_to_sample, best_so_far, max_num_threads, randomness_source, status)
  //                                                            gpp_python_expected_improvement.cpp:602-659 (DESIGN.md K20)
  py::class_<ObjectiveEstimationPolicyInterface>(m, "ObjectiveEstimationPolicyInterface");
  py::class_<ConstantLiarEstimationPolicy, ObjectiveEstimationPolicyInterface>(m, "ConstantLiarEstimationPolicy")
      .def(py::init<double, double>(), py::arg("lie_value"), py::arg("lie_noise_variance"));
  py::class_<KrigingBelieverEstimationPolicy, ObjectiveEstimationPolicyInterface>(m, "KrigingBelieverEstimationPolicy")
      .def(py::init<double, double>(), py::arg("std_deviation_coef"), py::arg("kriging_noise_variance"));
  m.def("heuristic_expected_improvement_optimization", &heuristic_expected_improvement_optimization);
  // a call that matches no signature raises the library's own exception
  m.def("heuristic_expected_improvement_optimization", [](const py::args&, const py::kwargs&) -> py::object {
    raise_exc(g_exc_base,
              "heuristic_expected_improvement_optimization: the arguments match no signature of the reference's "
              "function");
  });
  m.def("run_cpp_tests", []() -> int { not_on_path("run_cpp_tests"); });
  m.def("device_count", []() { return cmoe_device_count(); });
  m.def("version", []() { return std::string(cmoe_version()); });
}

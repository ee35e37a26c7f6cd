// extern "C" entry points that run the reference's own hyper-parameter optimisers.  Used only by
// make_hyper_opt_golden.py, which compiles this file against the reference headers and links it to
// oracle/_ref/libmoe_ref.so; the product never sees it.
#include <omp.h>

#include <vector>

#include "gpp_covariance.hpp"
#include "gpp_domain.hpp"
#include "gpp_model_selection.hpp"
#include "gpp_optimization.hpp"
#include "gpp_optimizer_parameters.hpp"
#include "gpp_random.hpp"

using namespace optimal_learning;  // NOLINT

namespace {

std::vector<ClosedInterval> intervals(const double* bounds, int nh) {
  std::vector<ClosedInterval> d(nh);
  for (int i = 0; i < nh; ++i) d[i] = {bounds[2 * i], bounds[2 * i + 1]};
  return d;
}

GradientDescentParameters gd_of(const double* gd) {
  return GradientDescentParameters(static_cast<int>(gd[0]), static_cast<int>(gd[1]), static_cast<int>(gd[2]),
                                   static_cast<int>(gd[3]), gd[4], gd[5], gd[6], gd[7]);
}

}  // namespace

extern "C" {

// num_calls consecutive calls on ONE explicitly seeded generator, each set up as the Python boundary does
// (gpp_python_model_selection.cpp:150-279): MaternNu2p5(alpha, lengths), LogMarginalLikelihoodEvaluator, log10 domain
// [nh][2], one thread.  optimizer 0: LatinHypercubeSearchHyperparameterOptimization with num_random_samples = gd[0];
// 1: MultistartGradientDescentHyperparameterOptimization.  gd[8] = GradientDescentParameters' constructor arguments.
// best[num_calls][nh], found[num_calls]; starts[num_calls][n][nh] = the (linear-space) starts each call drew, from a
// second generator with the same seed and the same sequence of draws.
void href_multistart(int optimizer, double alpha, const double* lengths, const double* noise, const double* X,
                     const double* y, const int* derivs, int g, int dim, int N, const double* log_domain,
                     const double* gd, unsigned seed, int num_calls, double* best, int* found, double* starts) {
  const int nh = dim + 2 + g, n = static_cast<int>(gd[0]);
  MaternNu2p5 cov(dim, alpha, lengths);
  LogMarginalLikelihoodEvaluator ev(X, y, derivs, g, dim, N);
  std::vector<double> nz(noise, noise + 1 + g);
  const std::vector<ClosedInterval> dom = intervals(log_domain, nh);
  UniformRandomGenerator gen(seed), gen_starts(seed);
  for (int c = 0; c < num_calls; ++c) {
    bool f = false;
    if (optimizer == 0) {
      ThreadSchedule sched(1, omp_sched_guided);
      LatinHypercubeSearchHyperparameterOptimization(ev, cov, nz, dom.data(), sched, n, &f, &gen,
                                                     best + static_cast<size_t>(c) * nh);
    } else {
      ThreadSchedule sched(1, omp_sched_dynamic);
      MultistartGradientDescentHyperparameterOptimization(ev, cov, nz, gd_of(gd), dom.data(), sched, &f, &gen,
                                                          best + static_cast<size_t>(c) * nh);
    }
    found[c] = f ? 1 : 0;
    std::vector<ClosedInterval> d2 = dom;
    std::vector<double> s(static_cast<size_t>(n) * nh);
    ConvertFromLogToLinearDomainAndBuildInitialGuesses(nh, n, &gen_starts, &d2, &s);
    std::copy(s.begin(), s.end(), starts + static_cast<size_t>(c) * n * nh);
  }
}

// RestartedGradientDescentHyperparameterOptimizationTensor from the set (alpha, lengths, noise) on the log10 domain,
// as restarted_hyperparameter_optimization sets it up (:343-376); out[nh] starts zeroed, as the wrapper's vector does.
void href_restarted(double alpha, const double* lengths, const double* noise, const double* X, const double* y,
                    const int* derivs, int g, int dim, int N, const double* log_domain, const double* gd, double* out) {
  const int nh = dim + 2 + g;
  MaternNu2p5 cov(dim, alpha, lengths);
  LogMarginalLikelihoodEvaluator ev(X, y, derivs, g, dim, N);
  std::vector<double> nz(noise, noise + 1 + g);
  const std::vector<ClosedInterval> dom = intervals(log_domain, nh);
  std::fill(out, out + nh, 0.0);
  RestartedGradientDescentHyperparameterOptimizationTensor(ev, cov, nz, gd_of(gd), dom.data(), out);
}

}  // extern "C"

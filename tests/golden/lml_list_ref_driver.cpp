// extern "C" entry point that runs the reference's own EvaluateLogLikelihoodAtPointList.  Used only by
// make_lml_list_golden.py, which compiles this file against the reference headers and links it to
// oracle/_ref/libmoe_ref.so; the product never sees it.
#include <omp.h>

#include <vector>

#include "gpp_covariance.hpp"
#include "gpp_domain.hpp"
#include "gpp_model_selection.hpp"
#include "gpp_optimization.hpp"

using namespace optimal_learning;  // NOLINT

extern "C" {

// EvaluateLogLikelihoodAtPointList (gpp_model_selection.hpp:1274-1308), set up as its Python boundary does
// (gpp_python_model_selection.cpp:281-341): MaternNu2p5 built from (alpha, lengths), LogMarginalLikelihoodEvaluator, a
// dummy domain, one thread.  hypers[num_sets][2 + dim + g]; values[num_sets] in list order; returns found_flag.
int lref_log_likelihood_at_hyperparameter_list(double alpha, const double* lengths, const double* noise,
                                               const double* hypers, int num_sets, const double* X, const double* y,
                                               const int* derivs, int g, int dim, int N, double* values) {
  MaternNu2p5 cov(dim, alpha, lengths);
  LogMarginalLikelihoodEvaluator ev(X, y, derivs, g, dim, N);
  std::vector<double> nz(noise, noise + 1 + g);
  std::vector<double> best(static_cast<size_t>(dim) + 2 + g);
  TensorProductDomain dummy_domain(nullptr, 0);
  ThreadSchedule sched(1, omp_sched_guided);
  bool found = false;
  EvaluateLogLikelihoodAtPointList(ev, cov, nz, dummy_domain, sched, hypers, num_sets, &found, values, best.data());
  return found ? 1 : 0;
}

}  // extern "C"

// posterior_mean_optimization: minimise the GP posterior mean from one start point with the reference's line-search
// gradient descent (the recommendation step of the BayesOpt loop).
//
// Replaces ComputeOptimalPosteriorMean with num_starts = 1 on the un-fantasised GP
// (gpp_knowledge_gradient_optimization.cpp:420-472; PosteriorMeanEvaluator :334-359; line search
// gpp_optimization.hpp:708-828, 1242-1283; LimitUpdate gpp_domain.cpp:64-104); Python boundary
// posterior_mean_optimization (gpp_python_knowledge_gradient.cpp:306-350).
//
// The problem is inherently sequential (one trajectory), so it runs as ONE warp: lanes split the n rows of
// k(x, X) . K^-1 y, shuffle-reduce value and gradient, and every lane carries the (uniform) optimiser state.
//
// The ensemble forms (cmoe_posterior_mean_mcmc, cmoe_posterior_mean_mcmc_optimization) serve the recommendation step
// of the MCMC loop: screening many points, then the Python fixed-step gradient descent on the averaged mean from many
// starts at once (one CTA per start); they share the row arithmetic (pm_rows) with pm_opt_kernel.
#include <algorithm>
#include <cmath>
#include <limits>

#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {
namespace {

struct PmOptParams {
  int N, ps, max_steps, max_restarts;
  double mean, mrc, tol;
  double lo[CMOE_MAX_DIM], hi[CMOE_MAX_DIM];
};

__device__ __forceinline__ double limit_step_pm(double step, double x, double lo, double hi, double mrc) {
  double dist = fmin(x - lo, hi - x);
  if (fabs(step) > mrc * dist) step = copysign(mrc * dist, step);
  const double next = x + step;
  if (next < lo || next > hi) {
    if (next < lo) {
      dist = lo - x;
      step = (x + step * 0.5 < lo) ? dist * 0.5 : step * 0.5;
    } else {
      dist = hi - x;
      step = (x + step * 0.5 > hi) ? dist * 0.5 : step * 0.5;
    }
  }
  return step;
}

// One thread's share of k(x, X) . beta (and, if g != null, of its gradient on the first ps coordinates) for one GP
// (spec, N sampled points X, beta = K^-1 (y - mean)): the rows row0, row0 + stride, ... added in ascending order.
__device__ __forceinline__ void pm_rows(const KernelSpec& spec, int N, int ps, const double* __restrict__ X,
                                        const double* __restrict__ beta, const double* xq, int row0, int stride,
                                        double& val, double* g) {
  const int dim = spec.dim, b1 = 1 + spec.g, n = N * b1;
  for (int row = row0; row < n; row += stride) {
    const int j = row / b1, ty = (row % b1) ? spec.derivs[row % b1 - 1] : -1;
    const double* xj = X + static_cast<size_t>(j) * dim;
    const KParts kp = kernel_parts(spec, weighted_sqdist(spec, xj, xq));
    val += cov_entry(spec, kp, xj, xq, ty, -1) * beta[row];
    if (g) {
      const KParts kq = kernel_parts(spec, weighted_sqdist(spec, xq, xj));
      for (int d = 0; d < ps; ++d) g[d] += grad_cov_entry(spec, kq, xq, xj, -1, ty, d) * beta[row];
    }
  }
}

// f(x) = -mu(x), grad f = -dmu/dx on the free coordinates; all lanes return the same values
__device__ double pm_eval(const KernelSpec& spec, const PmOptParams& prm, const double* __restrict__ X,
                          const double* __restrict__ beta, const double* xq, double* grad /* [dim] or null */) {
  const int dim = spec.dim, lane = threadIdx.x & 31;
  double val = 0.0;
  double g[CMOE_MAX_DIM];
  for (int d = 0; d < dim; ++d) g[d] = 0.0;
  pm_rows(spec, prm.N, prm.ps, X, beta, xq, lane, 32, val, grad ? g : nullptr);
  val = warp_sum(val);
  if (grad)
    for (int d = 0; d < dim; ++d) grad[d] = (d < prm.ps) ? -warp_sum(g[d]) : 0.0;
  return -(prm.mean + val);
}

__global__ void __launch_bounds__(32) pm_opt_kernel(const __grid_constant__ KernelSpec spec,
                                                    const __grid_constant__ PmOptParams prm,
                                                    const double* __restrict__ X, const double* __restrict__ beta,
                                                    const double* __restrict__ alpha0, const double* __restrict__ x0,
                                                    double* __restrict__ out) {
  const int dim = spec.dim, ps = prm.ps;
  double x[CMOE_MAX_DIM], gb[CMOE_MAX_DIM], xt[CMOE_MAX_DIM], step[CMOE_MAX_DIM], run0[CMOE_MAX_DIM];
  for (int d = 0; d < dim; ++d) x[d] = x0[d];
  double fb = pm_eval(spec, prm, X, beta, x, gb);
  if (prm.max_restarts > 0) {
    const double step_tol = prm.max_steps > 0 ? prm.tol / static_cast<double>(prm.max_steps) : 0.0;
    for (int r = 0; r < prm.max_restarts; ++r) {
      for (int d = 0; d < dim; ++d) run0[d] = x[d];
      for (int i = 0; i < prm.max_steps; ++i) {
        double alpha = alpha0[i];
        double nrm = 0.0;
        for (int d = 0; d < ps; ++d) nrm += gb[d] * gb[d];
        int search = 0;
        double obj = 0.0;
        while (search < 30) {
          for (int d = 0; d < dim; ++d) xt[d] = x[d] + ((d < ps) ? alpha * gb[d] : 0.0);
          obj = pm_eval(spec, prm, X, beta, xt, nullptr);
          if (obj - fb > 0.5 * alpha * nrm) break;
          alpha *= 0.5;
          search += 1;
        }
        for (int d = 0; d < dim; ++d)
          step[d] = (d < ps) ? limit_step_pm(alpha * gb[d], x[d], prm.lo[d], prm.hi[d], prm.mrc) : 0.0;
        for (int d = 0; d < dim; ++d) xt[d] = x[d] + step[d];
        obj = pm_eval(spec, prm, X, beta, xt, nullptr);
        if (obj <= fb || search == 30) break;
        double ns = 0.0;
        for (int d = 0; d < dim; ++d) {
          x[d] += step[d];
          ns += step[d] * step[d];
        }
        fb = pm_eval(spec, prm, X, beta, x, gb);
        if (sqrt(ns) < step_tol) break;
      }
      double nd = 0.0;
      for (int d = 0; d < ps; ++d) nd += (run0[d] - x[d]) * (run0[d] - x[d]);
      if (sqrt(nd) <= prm.tol) break;
    }
  }
  if (threadIdx.x == 0) {
    for (int d = 0; d < ps; ++d) out[d] = x[d];
    out[ps] = fb;
  }
}

// --------------------------------------------------------------------------------------------------------------
// Ensemble posterior mean f(x) = -(1/M) sum_m mu_m(x) (PosteriorMeanMCMC, cpp_wrappers/knowledge_gradient_mcmc.py:25-157)
// and the Python GradientDescentOptimizer on it (python_version/optimization.py:392-528): fixed-step descent
// alpha_k = pre_mult k^-gamma with TensorProductDomain.compute_update_restricted_to_domain (python_version/domain.py:
// 158-202), then the Polyak-Ruppert average.  One CTA per start runs the whole trajectory; inside it, warps take
// (member, row slice) units, so a single start spreads its M * N rows over the whole CTA.
// --------------------------------------------------------------------------------------------------------------
struct PmMember {
  KernelSpec spec;
  const double* X;     // [N][dim]
  const double* beta;  // [N (1 + g)]  K^-1 (y - mean)
  double mean;
  int N;
};

struct PmMcmcParams {
  int M, S, ps, dim, steps;
  int avg_first, avg_count;  // x_k for k in [avg_first, avg_first + avg_count) are averaged
  double mrc;
  double lo[CMOE_MAX_DIM], hi[CMOE_MAX_DIM];
};

constexpr int kPmMcmcThreads = 256;

// Row sums of every (member, slice) unit at the CTA's point xq [dim]: red[u][0] = sum of k(xq, X_j) beta_j,
// red[u][1 + d] = the same for d/dx_d (if grad).  Unit u = m S + s is member m's rows s*32 + lane, stride 32 S, on one
// warp, lanes combined by the fixed xor butterfly; the assignment depends only on (M, S), not on the start.
__device__ void ens_partials(const PmMember* mem, const PmMcmcParams& prm, const double* xq, bool grad, double* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5, w1 = 1 + prm.ps;
  for (int u = warp; u < prm.M * prm.S; u += nw) {
    const PmMember& mb = mem[u / prm.S];
    double val = 0.0;
    double g[CMOE_MAX_DIM];
    for (int d = 0; d < prm.ps; ++d) g[d] = 0.0;
    pm_rows(mb.spec, mb.N, prm.ps, mb.X, mb.beta, xq, (u % prm.S) * 32 + lane, prm.S * 32, val, grad ? g : nullptr);
    val = warp_sum(val);
    if (lane == 0) red[u * w1] = val;
    if (grad) {
      for (int d = 0; d < prm.ps; ++d) {
        const double t = warp_sum(g[d]);
        if (lane == 0) red[u * w1 + 1 + d] = t;
      }
    }
  }
}

// Component c (0: value, 1 + d: d/dx_d) of f from the unit sums: slices in ascending order per member, members in
// ascending order, then the division by M, which is PosteriorMeanMCMC's order (sum of -mu_m, then old_div).
__device__ double ens_combine(const PmMember* mem, const PmMcmcParams& prm, const double* red, int c) {
  const int w1 = 1 + prm.ps;
  double acc = 0.0;
  for (int m = 0; m < prm.M; ++m) {
    double t = red[(m * prm.S) * w1 + c];
    for (int s = 1; s < prm.S; ++s) t = __dadd_rn(t, red[(m * prm.S + s) * w1 + c]);
    if (c == 0) t = __dadd_rn(mem[m].mean, t);
    acc = __dadd_rn(acc, -t);  // 0.0 + (-t) first, as the Python sum starts from 0
  }
  return __ddiv_rn(acc, static_cast<double>(prm.M));
}

// grid = starts; out[start][ps + 1] = (averaged point, f there).  Dynamic shared memory: the M member descriptors,
// the unit sums [M S][1 + ps], the current point [dim].
__global__ void __launch_bounds__(kPmMcmcThreads) pm_mcmc_opt_kernel(const __grid_constant__ PmMcmcParams prm,
                                                                     const PmMember* __restrict__ members,
                                                                     const double* __restrict__ alpha,
                                                                     const double* __restrict__ starts,
                                                                     double* __restrict__ out) {
  extern __shared__ unsigned long long pm_smem[];
  const int tid = threadIdx.x, ps = prm.ps;
  const int words = prm.M * static_cast<int>(sizeof(PmMember) / sizeof(unsigned long long));
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(members);
  for (int i = tid; i < words; i += blockDim.x) pm_smem[i] = src[i];
  const PmMember* mem = reinterpret_cast<const PmMember*>(pm_smem);
  double* red = reinterpret_cast<double*>(pm_smem + words);
  double* x = red + prm.M * prm.S * (1 + ps);
  const size_t st = blockIdx.x;
  for (int d = tid; d < prm.dim; d += blockDim.x) x[d] = (d < ps) ? starts[st * ps + d] : 1.0;  // fidelity = 1
  __syncthreads();
  double sum = 0.0;  // thread d < ps: Polyak-Ruppert sum of coordinate d, ascending k
  for (int k = 1; k <= prm.steps; ++k) {
    ens_partials(mem, prm, x, true, red);
    __syncthreads();
    if (tid < ps) {
      const double xd = x[tid];
      // explicitly rounded, so that nothing is contracted into an FMA: numpy's arithmetic, operation for operation
      double step = __dmul_rn(ens_combine(mem, prm, red, 1 + tid), alpha[k - 1]);
      const double lim = __dmul_rn(prm.mrc, fmin(__dsub_rn(xd, prm.lo[tid]), __dsub_rn(prm.hi[tid], xd)));
      if (fabs(step) > lim) step = copysign(lim, step);
      const double xn = __dadd_rn(step, xd);
      if (k == prm.avg_first) sum = xn;
      else if (k > prm.avg_first) sum = __dadd_rn(sum, xn);
      x[tid] = xn;
    }
    __syncthreads();
  }
  if (tid < ps) x[tid] = __ddiv_rn(sum, static_cast<double>(prm.avg_count));
  __syncthreads();
  ens_partials(mem, prm, x, false, red);
  __syncthreads();
  if (tid == 0) out[st * (ps + 1) + ps] = ens_combine(mem, prm, red, 0);
  if (tid < ps) out[st * (ps + 1) + tid] = x[tid];
}

// values [P] = (sum_m -mu[m][i]) / M; grads [P][ps] likewise from gmu [M][P][dim] (if not null).  Members in ascending
// order, as PosteriorMeanMCMC adds them.  One thread per (point, component).
__global__ void __launch_bounds__(256) pm_mcmc_combine_kernel(int M, size_t P, int dim, int ps,
                                                              const double* __restrict__ mu,
                                                              const double* __restrict__ gmu,
                                                              double* __restrict__ values, double* __restrict__ grads) {
  const int per = gmu ? 1 + ps : 1;
  const size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (o >= P * per) return;
  const size_t i = o / per;
  const int c = static_cast<int>(o % per);
  double acc = 0.0;
  for (int m = 0; m < M; ++m) {
    const size_t mi = static_cast<size_t>(m) * P + i;
    const double v = (c == 0) ? mu[mi] : gmu[mi * dim + c - 1];
    acc = __dadd_rn(acc, -v);
  }
  acc = __ddiv_rn(acc, static_cast<double>(M));
  if (c == 0) {
    values[i] = acc;
  } else {
    grads[i * ps + c - 1] = acc;
  }
}

// the members' fits ran on their own streams; the ensemble calls work on member 0's
void join_member_streams(const cmoe_gp* const* gps, int num_gp) {
  for (int m = 1; m < num_gp; ++m)
    if (gps[m]->stream != gps[0]->stream) CMOE_CUDA(cudaStreamSynchronize(gps[m]->stream));
}

}  // namespace
}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_posterior_mean_optimization(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* params,
                                                const double* domain_bounds, const double* initial_guess,
                                                double* best_point, double* best_value, int* found_flag) {
  return guarded(nullptr, [&] {
    const KernelSpec& spec = gp->spec;
    const int dim = spec.dim, ps = dim - num_fidelity;
    CMOE_REQUIRE(num_fidelity >= 0 && ps >= 1, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    CMOE_REQUIRE(params->max_num_steps <= 1 << 20, CMOE_ERR_BOUNDS, "max_num_steps too large");
    for (int d = 0; d < ps; ++d)
      CMOE_REQUIRE(domain_bounds[2 * d] <= domain_bounds[2 * d + 1], CMOE_ERR_BOUNDS, "Tensor product region is EMPTY.");
    require_device(gp->device);
    if (found_flag) *found_flag = 0;
    if (params->max_num_restarts <= 0) return;  // the reference returns without touching its outputs (:424-426)
    cudaStream_t s = gp->stream;
    PmOptParams prm{};
    prm.N = gp->N;
    prm.ps = ps;
    prm.max_steps = params->max_num_steps;
    prm.max_restarts = params->max_num_restarts;
    prm.mean = gp->mean;
    prm.mrc = params->max_relative_change;
    prm.tol = params->tolerance;
    for (int d = 0; d < CMOE_MAX_DIM; ++d) {
      prm.lo[d] = (d < ps) ? domain_bounds[2 * d] : -1e300;
      prm.hi[d] = (d < ps) ? domain_bounds[2 * d + 1] : 1e300;
    }
    std::vector<double> a0(std::max(1, params->max_num_steps)), x0(dim, 1.0), res(ps + 1);
    for (int i = 0; i < params->max_num_steps; ++i)
      a0[i] = params->pre_mult * std::pow(static_cast<double>(i + 1), -params->gamma);
    for (int d = 0; d < ps; ++d) x0[d] = initial_guess[d];
    DevBuf<double> dA0, dX0, dOut(ps + 1);
    dA0.upload(a0.data(), a0.size(), s);
    dX0.upload(x0.data(), x0.size(), s);
    pm_opt_kernel<<<1, 32, 0, s>>>(spec, prm, gp->dX.p, gp->dKinvY.p, dA0.p, dX0.p, dOut.p);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    dOut.download(res.data(), ps + 1, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    for (int d = 0; d < ps; ++d) best_point[d] = res[d];
    if (best_value) *best_value = res[ps];
    if (found_flag) *found_flag = 1;
  });
}

extern "C" int cmoe_posterior_mean_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const double* points,
                                        int num_points, double* values, double* grads, double* member_values,
                                        int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_points >= 1, CMOE_ERR_BOUNDS, "num_points must be >= 1");
    CMOE_REQUIRE(num_fidelity >= 0, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    check_ensemble(gps, num_gp);
    const int dim = gps[0]->spec.dim, ps = dim - num_fidelity;
    CMOE_REQUIRE(ps >= 1, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    require_device(gps[0]->device);
    join_member_streams(gps, num_gp);
    cudaStream_t s = gps[0]->stream;
    const size_t P = num_points, M = num_gp;
    // fidelity coordinates pinned to 1.0, as compute_posterior_mean_of_points pads them
    std::vector<double> full(P * dim, 1.0);
    for (size_t i = 0; i < P; ++i)
      for (int d = 0; d < ps; ++d) full[i * dim + d] = points[i * ps + d];
    DevBuf<double> dP, dmu(M * P), dgmu(grads ? M * P * dim : 0), dval(P), dgrad(grads ? P * ps : 0);
    DevBuf<int> dd(1);
    dP.upload(full.data(), full.size(), s);
    for (int m = 0; m < num_gp; ++m)
      posterior_mean_points(*gps[m], dP.p, P, dd.p, 0, dmu.p + m * P, grads ? dgmu.p + m * P * dim : nullptr, s);
    const size_t outs = P * (grads ? 1 + ps : 1);
    pm_mcmc_combine_kernel<<<static_cast<unsigned>((outs + 255) / 256), 256, 0, s>>>(
        num_gp, P, dim, ps, dmu.p, grads ? dgmu.p : nullptr, dval.p, grads ? dgrad.p : nullptr);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    dval.download(values, P, s);
    if (grads) dgrad.download(grads, P * ps, s);
    if (member_values) dmu.download(member_values, M * P, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    if (member_values)
      for (size_t k = 0; k < M * P; ++k) member_values[k] = -member_values[k];
  });
}

extern "C" int cmoe_posterior_mean_mcmc_optimization(const cmoe_gp* const* gps, int num_gp, int num_fidelity,
                                                     const cmoe_gd_params* params, const double* domain_bounds,
                                                     const double* starts, int num_starts, double* points_out,
                                                     double* values_out, double* best_point, double* best_value,
                                                     int* info) {
  return guarded(info, [&] {
    // every check comes before any device work; those that need no GP handle come first
    CMOE_REQUIRE(params != nullptr && domain_bounds != nullptr && starts != nullptr, CMOE_ERR_INVALID_VALUE,
                 "params, domain_bounds and starts must not be NULL");
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_starts must be >= 1");
    // the Python optimiser averages an empty range (NaN) with max_num_steps < 1
    CMOE_REQUIRE(params->max_num_steps >= 1 && params->max_num_steps <= 1 << 20, CMOE_ERR_BOUNDS,
                 "max_num_steps must be in [1, 2^20]");
    CMOE_REQUIRE(num_fidelity >= 0, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    check_ensemble(gps, num_gp);
    const int dim = gps[0]->spec.dim, ps = dim - num_fidelity;
    CMOE_REQUIRE(ps >= 1, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    for (int d = 0; d < ps; ++d)
      CMOE_REQUIRE(domain_bounds[2 * d] <= domain_bounds[2 * d + 1], CMOE_ERR_BOUNDS, "Tensor product region is EMPTY.");
    require_device(gps[0]->device);
    join_member_streams(gps, num_gp);
    cudaStream_t s = gps[0]->stream;

    PmMcmcParams prm{};
    prm.M = num_gp;
    prm.ps = ps;
    prm.dim = dim;
    prm.steps = params->max_num_steps;
    prm.mrc = params->max_relative_change;
    // _get_averaging_range (optimization.py:415-442): < 0 or > steps -> all steps, 0 -> the last step only
    int nav = params->num_steps_averaged;
    if (nav < 0 || nav > prm.steps) {
      nav = prm.steps;
    } else if (nav == 0) {
      nav = 1;
    }
    prm.avg_first = prm.steps - nav + 1;
    prm.avg_count = nav;
    for (int d = 0; d < CMOE_MAX_DIM; ++d) {
      prm.lo[d] = (d < ps) ? domain_bounds[2 * d] : 0.0;
      prm.hi[d] = (d < ps) ? domain_bounds[2 * d + 1] : 0.0;
    }
    // row slices per member: enough units to occupy every warp of the CTA, none shorter than one row per lane
    int max_rows = 0;
    std::vector<PmMember> mem(num_gp);
    for (int m = 0; m < num_gp; ++m) {
      mem[m] = PmMember{gps[m]->spec, gps[m]->dX.p, gps[m]->dKinvY.p, gps[m]->mean, gps[m]->N};
      max_rows = std::max(max_rows, gps[m]->n);
    }
    constexpr int kWarps = kPmMcmcThreads / 32;
    prm.S = std::max(1, std::min((kWarps + num_gp - 1) / num_gp, (max_rows + 31) / 32));
    const size_t smem = num_gp * sizeof(PmMember) +
                        (static_cast<size_t>(num_gp) * prm.S * (1 + ps) + dim) * sizeof(double);
    int dev_smem = 0;
    CMOE_CUDA(cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, gps[0]->device));
    CMOE_REQUIRE(smem <= static_cast<size_t>(dev_smem), CMOE_ERR_BOUNDS, "ensemble too large for one CTA");
    if (smem > 48 * 1024)
      CMOE_CUDA(cudaFuncSetAttribute(pm_mcmc_opt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(smem)));

    // alpha_k = pre_mult k^-gamma on the host, as numpy.power computes it
    std::vector<double> a(prm.steps);
    for (int k = 1; k <= prm.steps; ++k) a[k - 1] = params->pre_mult * std::pow(static_cast<double>(k), -params->gamma);
    const size_t ns = num_starts;
    DevBuf<PmMember> dMem;
    DevBuf<double> dA, dStarts, dOut(ns * (ps + 1));
    dMem.upload(mem.data(), mem.size(), s);
    dA.upload(a.data(), a.size(), s);
    dStarts.upload(starts, ns * ps, s);
    pm_mcmc_opt_kernel<<<static_cast<unsigned>(ns), kPmMcmcThreads, smem, s>>>(prm, dMem.p, dA.p, dStarts.p, dOut.p);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    std::vector<double> res(ns * (ps + 1));
    dOut.download(res.data(), res.size(), s);
    CMOE_CUDA(cudaStreamSynchronize(s));

    // MultistartOptimizer.optimize (optimization.py:565-610): best -inf, point = starts[0], strict > in start order
    double bv = -std::numeric_limits<double>::infinity();
    const double* bp = starts;
    for (size_t i = 0; i < ns; ++i) {
      const double* r = res.data() + i * (ps + 1);
      if (points_out) std::copy(r, r + ps, points_out + i * ps);
      if (values_out) values_out[i] = r[ps];
      if (r[ps] > bv) {
        bv = r[ps];
        bp = r;
      }
    }
    if (best_point) std::copy(bp, bp + ps, best_point);
    if (best_value) *best_value = bv;
  });
}

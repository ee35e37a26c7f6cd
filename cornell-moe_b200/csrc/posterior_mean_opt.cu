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
//
// cmoe_posterior_mean_optima_mcmc is the discretisation step of the MCMC q-KG loop: the same line search
// (pm_descend) for every member of an ensemble at once, one CTA per member, after a screen over (member, point).
#include <algorithm>
#include <cmath>
#include <limits>

#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {
namespace {

// the line-search gradient descent's parameters (cmoe_gd_params) and box; coordinates >= ps (fidelity) do not move
struct PmDescent {
  int ps, max_steps, max_restarts;
  double mrc, tol;
  double lo[CMOE_MAX_DIM], hi[CMOE_MAX_DIM];
};

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
__device__ double pm_eval(const KernelSpec& spec, int N, int ps, double mean, const double* __restrict__ X,
                          const double* __restrict__ beta, const double* xq, double* grad /* [dim] or null */) {
  const int dim = spec.dim, lane = threadIdx.x & 31;
  double val = 0.0;
  double g[CMOE_MAX_DIM];
  for (int d = 0; d < dim; ++d) g[d] = 0.0;
  pm_rows(spec, N, ps, X, beta, xq, lane, 32, val, grad ? g : nullptr);
  val = warp_sum(val);
  if (grad)
    for (int d = 0; d < dim; ++d) grad[d] = (d < ps) ? -warp_sum(g[d]) : 0.0;
  return -(mean + val);
}

// The reference's restarted line-search gradient descent on f from x [dim] (moved in place); returns f at the end
// point.  eval(xq, grad or null) = f(xq) must return the same bits in every thread that calls this, so that every
// decision below is uniform over those threads and each of them carries the same optimiser state.
template <class Eval>
__device__ __forceinline__ double pm_descend(const PmDescent& prm, int dim, const double* __restrict__ alpha0, double* x,
                                             Eval&& eval) {
  const int ps = prm.ps;
  double gb[CMOE_MAX_DIM], xt[CMOE_MAX_DIM], step[CMOE_MAX_DIM], run0[CMOE_MAX_DIM];
  double fb = eval(x, gb);
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
          obj = eval(xt, nullptr);
          if (obj - fb > 0.5 * alpha * nrm) break;
          alpha *= 0.5;
          search += 1;
        }
        for (int d = 0; d < dim; ++d)
          step[d] = (d < ps) ? limit_step(alpha * gb[d], x[d], prm.lo[d], prm.hi[d], prm.mrc) : 0.0;
        for (int d = 0; d < dim; ++d) xt[d] = x[d] + step[d];
        obj = eval(xt, nullptr);
        if (obj <= fb || search == 30) break;
        double ns = 0.0;
        for (int d = 0; d < dim; ++d) {
          x[d] += step[d];
          ns += step[d] * step[d];
        }
        fb = eval(x, gb);
        if (sqrt(ns) < step_tol) break;
      }
      double nd = 0.0;
      for (int d = 0; d < ps; ++d) nd += (run0[d] - x[d]) * (run0[d] - x[d]);
      if (sqrt(nd) <= prm.tol) break;
    }
  }
  return fb;
}

__global__ void __launch_bounds__(32) pm_opt_kernel(const __grid_constant__ KernelSpec spec,
                                                    const __grid_constant__ PmDescent prm, int N, double mean,
                                                    const double* __restrict__ X, const double* __restrict__ beta,
                                                    const double* __restrict__ alpha0, const double* __restrict__ x0,
                                                    double* __restrict__ out) {
  const int dim = spec.dim, ps = prm.ps;
  double x[CMOE_MAX_DIM];
  for (int d = 0; d < dim; ++d) x[d] = x0[d];
  const double fb = pm_descend(prm, dim, alpha0, x, [&](const double* xq, double* grad) {
    return pm_eval(spec, N, ps, mean, X, beta, xq, grad);
  });
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

// --------------------------------------------------------------------------------------------------------------
// Per-member posterior-mean optima (cmoe_posterior_mean_optima_mcmc): for every member on its own, screen a list of
// points by mu_m, descend from the argmin with the line search above, fall back to the start if the descent ended
// higher, and take the least mu_m over the member's discretisation set [shared points ; optimum]
// (examples/main.py:172-197, knowledge_gradient_mcmc.py:386-393).
//   pm_members_screen_kernel   one CTA per (member, screen index) of a chunk
//   pm_members_argmin_kernel   one CTA per member: the chunk's least value and lowest index, merged into the running one
//   pm_members_opt_kernel      one CTA per member: descent, fallback, baseline
// Per member the three kernels share one row of `state`, kPmStateHead + 2 ps doubles:
//   [0] least screened mu  [1] its index in the member's screen list  [2] mu at the optimum  [3] best_so_far
//   [4] 1 if the start was kept  [5, 5 + ps) the start x0  [5 + ps, 5 + 2 ps) the optimum
// --------------------------------------------------------------------------------------------------------------
constexpr int kPmScreenParts = 128;    // partial sums per screened value: post_mean_only_kernel's thread count
constexpr int kPmOptimaThreads = 256;  // pm_members_argmin_kernel, pm_members_opt_kernel
constexpr int kPmMaxSlices = kPmOptimaThreads / 32;
constexpr int kPmStateHead = 5;
constexpr size_t kPmOptimaWorkspaceBytes = size_t(64) << 20;  // one screen chunk: its points and its values

// row slices (warps) of a member's descent: a function of its rows n = N (1 + g) only, none shorter than two rows a lane
__device__ __forceinline__ int pm_member_slices(int n) { return max(1, min(kPmMaxSlices, n / 64)); }

__device__ __forceinline__ void load_member(PmMember* dst, const PmMember* __restrict__ src) {
  const unsigned long long* in = reinterpret_cast<const unsigned long long*>(src);
  unsigned long long* out = reinterpret_cast<unsigned long long*>(dst);
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(PmMember) / sizeof(unsigned long long)); i += blockDim.x)
    out[i] = in[i];
}

// mu(x) of one member with the arithmetic of posterior_mean_points (post_mean_only_kernel, value only), so that a value
// screened here and one returned by cmoe_posterior_mean_mcmc or cmoe_gp_posterior are the same bits: thread
// p < kPmScreenParts adds the sampled points p, p + kPmScreenParts, ... in ascending order, thread 0 adds the partial
// sums in ascending order.  Called by the whole CTA (>= kPmScreenParts threads); x [dim] and red [kPmScreenParts] are
// shared memory; the result is valid in thread 0.
__device__ __forceinline__ double pm_screen_mean(const PmMember& mb, const double* x, double* red) {
  const int tid = threadIdx.x, dim = mb.spec.dim, b1 = 1 + mb.spec.g;
  if (tid < kPmScreenParts) {
    double acc = 0.0;
    for (int j = tid; j < mb.N; j += kPmScreenParts) {
      const double* xj = mb.X + static_cast<size_t>(j) * dim;
      const KParts kp = kernel_parts(mb.spec, weighted_sqdist(mb.spec, x, xj));
      for (int cc = 0; cc < b1; ++cc) {
        const int a2 = cc ? mb.spec.derivs[cc - 1] : -1;
        acc = fma(cov_entry(mb.spec, kp, x, xj, -1, a2), mb.beta[static_cast<size_t>(j) * b1 + cc], acc);
      }
    }
    red[tid] = acc;
  }
  __syncthreads();
  double t = 0.0;
  if (tid == 0)
    for (int q = 0; q < kPmScreenParts; ++q) t += red[q];
  __syncthreads();
  return mb.mean + t;
}

// Screen indices [i0, i0 + len) of every member's list: the given points (shared by the members, or one list per
// member), then the member's own sampled points, read from its X.  grid.x = num_gp * len; V [num_gp][len].  pts holds
// the given points of this chunk only, [1 or num_gp][num_given][ps], num_given = those of the chunk's indices below
// num_points.
__global__ void __launch_bounds__(kPmScreenParts) pm_members_screen_kernel(const PmMember* __restrict__ members, int ps,
                                                                           const double* __restrict__ pts,
                                                                           int per_member, int num_points,
                                                                           int include_sampled, int i0, int len,
                                                                           int num_given, double* __restrict__ V) {
  __shared__ PmMember mb;
  __shared__ double x[CMOE_MAX_DIM];
  __shared__ double red[kPmScreenParts];
  const int m = blockIdx.x / len, i = blockIdx.x % len, gi = i0 + i;
  load_member(&mb, members + m);
  __syncthreads();
  if (gi >= num_points + (include_sampled ? mb.N : 0)) return;
  const double* src = (gi < num_points) ? pts + (static_cast<size_t>(per_member ? m : 0) * num_given + i) * ps
                                        : mb.X + static_cast<size_t>(gi - num_points) * mb.spec.dim;
  for (int d = threadIdx.x; d < mb.spec.dim; d += blockDim.x) x[d] = (d < ps) ? src[d] : 1.0;  // fidelity = 1
  __syncthreads();
  const double mu = pm_screen_mean(mb, x, red);
  if (threadIdx.x == 0) V[static_cast<size_t>(m) * len + i] = mu;
}

// grid.x = num_gp.  Each thread scans its indices of the chunk, then block_best combines the threads; the chunk's winner
// replaces the running one only if it is strictly smaller, so the result is np.argmin's (first occurrence) however the
// screen is chunked.  The winner's coordinates become the member's start.
__global__ void __launch_bounds__(kPmOptimaThreads) pm_members_argmin_kernel(const PmMember* __restrict__ members,
                                                                             int ps, const double* __restrict__ pts,
                                                                             int per_member, int num_points,
                                                                             int include_sampled, int i0, int len,
                                                                             int num_given,
                                                                             const double* __restrict__ V,
                                                                             double* __restrict__ state) {
  __shared__ double sv[kPmOptimaThreads / 32];
  __shared__ int si[kPmOptimaThreads / 32];
  const int m = blockIdx.x, tid = threadIdx.x;
  const PmMember& mb = members[m];
  const int cnt = min(len, num_points + (include_sampled ? mb.N : 0) - i0);
  if (cnt <= 0) return;
  const double* Vm = V + static_cast<size_t>(m) * len;
  double bv = Vm[0];  // a chunk whose values are all NaN still names a point
  int bi = 0;
  for (int i = tid; i < cnt; i += kPmOptimaThreads)
    if (beats<false>(Vm[i], i, bv, bi)) {
      bv = Vm[i];
      bi = i;
    }
  block_best<false>(bv, bi, sv, si);
  double* row = state + static_cast<size_t>(m) * (kPmStateHead + 2 * ps);
  const bool take = i0 == 0 || bv < row[0];
  __syncthreads();  // every thread has read the running minimum before thread 0 replaces it
  if (!take) return;
  const int gi = i0 + bi;
  const double* src = (gi < num_points) ? pts + (static_cast<size_t>(per_member ? m : 0) * num_given + bi) * ps
                                        : mb.X + static_cast<size_t>(gi - num_points) * mb.spec.dim;
  if (tid < ps) row[kPmStateHead + tid] = src[tid];
  if (tid == 0) {
    row[0] = bv;
    row[1] = static_cast<double>(gi);
  }
}

// f(x) = -mu_m(x) and its gradient for the whole CTA: warp s < S takes the rows s * 32 + lane, stride 32 S (pm_rows),
// lanes combined by the xor butterfly, slices added in ascending order.  Every thread returns the same bits; with S = 1
// they are pm_eval's.  red [kPmMaxSlices][1 + ps] is shared memory.  Not inlined: the line search calls it from four
// places, and one copy of the row loop keeps the kernel's code small and its registers unspilled.
__device__ __noinline__ double pm_member_eval(const PmMember& mb, int ps, int S, const double* xq, double* grad,
                                                 double* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, dim = mb.spec.dim, w1 = 1 + ps;
  if (warp < S) {
    double val = 0.0;
    double g[CMOE_MAX_DIM];
    for (int d = 0; d < ps; ++d) g[d] = 0.0;
    pm_rows(mb.spec, mb.N, ps, mb.X, mb.beta, xq, warp * 32 + lane, S * 32, val, grad ? g : nullptr);
    val = warp_sum(val);
    if (lane == 0) red[warp * w1] = val;
    if (grad)
      for (int d = 0; d < ps; ++d) {
        const double t = warp_sum(g[d]);
        if (lane == 0) red[warp * w1 + 1 + d] = t;
      }
  }
  __syncthreads();
  double val = red[0];
  for (int s = 1; s < S; ++s) val = __dadd_rn(val, red[s * w1]);
  if (grad)
    for (int d = 0; d < dim; ++d) {
      double t = 0.0;
      if (d < ps) {
        t = red[1 + d];
        for (int s = 1; s < S; ++s) t = __dadd_rn(t, red[s * w1 + 1 + d]);
      }
      grad[d] = (d < ps) ? -t : 0.0;
    }
  __syncthreads();
  return -(mb.mean + val);
}

// grid.x = num_gp.  Descent from the member's start with every thread carrying the optimiser state (pm_descend), the
// fallback of main.py:191-193, then mu_m over [shared_pts ; optimum] in the screen's arithmetic, which is what
// cmoe_gp_posterior returns at those points.
__global__ void __launch_bounds__(kPmOptimaThreads) pm_members_opt_kernel(const __grid_constant__ PmDescent prm,
                                                                          const PmMember* __restrict__ members,
                                                                          const double* __restrict__ alpha0,
                                                                          const double* __restrict__ shared_pts,
                                                                          int num_shared, double* __restrict__ state) {
  __shared__ PmMember mb;
  __shared__ double red[kPmMaxSlices * (1 + CMOE_MAX_DIM)];
  __shared__ double sred[kPmScreenParts];
  __shared__ double xs[CMOE_MAX_DIM];
  const int tid = threadIdx.x, ps = prm.ps;
  load_member(&mb, members + blockIdx.x);
  __syncthreads();
  const int dim = mb.spec.dim;
  double* row = state + static_cast<size_t>(blockIdx.x) * (kPmStateHead + 2 * ps);
  const double screen_min = row[0];
  double x[CMOE_MAX_DIM];
  for (int d = 0; d < dim; ++d) x[d] = (d < ps) ? row[kPmStateHead + d] : 1.0;  // fidelity = 1
  bool kept = true;  // max_num_restarts <= 0: the reference's descent returns without moving
  double mu_opt = screen_min;
  if (prm.max_restarts > 0) {
    const int S = pm_member_slices(mb.N * (1 + mb.spec.g));
    const double fb = pm_descend(prm, dim, alpha0, x, [&](const double* xq, double* grad) {
      return pm_member_eval(mb, ps, S, xq, grad, red);
    });
    kept = -fb > screen_min;
    if (!kept) mu_opt = -fb;
  }
  if (kept)
    for (int d = 0; d < ps; ++d) x[d] = row[kPmStateHead + d];
  double best = 0.0;
  for (int j = 0; j <= num_shared; ++j) {
    for (int d = 0; d < dim; ++d)
      if (tid == d) xs[d] = (d >= ps) ? 1.0 : (j < num_shared) ? shared_pts[static_cast<size_t>(j) * ps + d] : x[d];
    __syncthreads();
    const double mu = pm_screen_mean(mb, xs, sred);
    best = (j == 0 || mu < best) ? mu : best;
  }
  if (tid == 0) {
    row[2] = mu_opt;
    row[3] = best;
    row[4] = kept ? 1.0 : 0.0;
    for (int d = 0; d < ps; ++d) row[kPmStateHead + ps + d] = x[d];
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
    PmDescent prm{};
    prm.ps = ps;
    prm.max_steps = params->max_num_steps;
    prm.max_restarts = params->max_num_restarts;
    prm.mrc = params->max_relative_change;
    prm.tol = params->tolerance;
    for (int d = 0; d < CMOE_MAX_DIM; ++d) {
      prm.lo[d] = (d < ps) ? domain_bounds[2 * d] : -1e300;
      prm.hi[d] = (d < ps) ? domain_bounds[2 * d + 1] : 1e300;
    }
    std::vector<double> a0(std::max(1, params->max_num_steps)), x0(dim, 1.0), res(ps + 1);
    for (int i = 0; i < params->max_num_steps; ++i)
      a0[i] = gd_step_size(params->pre_mult, params->gamma, i);
    for (int d = 0; d < ps; ++d) x0[d] = initial_guess[d];
    DevBuf<double> dA0, dX0, dOut(ps + 1);
    dA0.upload(a0.data(), a0.size(), s);
    dX0.upload(x0.data(), x0.size(), s);
    pm_opt_kernel<<<1, 32, 0, s>>>(spec, prm, gp->N, gp->mean, gp->dX.p, gp->dKinvY.p, dA0.p, dX0.p, dOut.p);
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
    for (int i = 0; i < prm.steps; ++i) a[i] = gd_step_size(params->pre_mult, params->gamma, i);
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

extern "C" int cmoe_posterior_mean_optima_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity,
                                               const cmoe_gd_params* params, const double* domain_bounds,
                                               const double* points, int num_points, int points_per_member,
                                               int include_sampled, const double* shared_discrete, int num_shared,
                                               double* optima, double* optimum_means, int* start_index,
                                               int* kept_start, double* screen_min, double* discrete_pts,
                                               double* best_so_far, int* info) {
  return guarded(info, [&] {
    // every check comes before any device work; those that need no GP handle come first
    CMOE_REQUIRE(params != nullptr && domain_bounds != nullptr && points != nullptr && optima != nullptr,
                 CMOE_ERR_INVALID_VALUE, "params, domain_bounds, points and optima must not be NULL");
    CMOE_REQUIRE(shared_discrete != nullptr || num_shared <= 0, CMOE_ERR_INVALID_VALUE,
                 "shared_discrete must not be NULL when num_shared > 0");
    CMOE_REQUIRE(num_points >= 1, CMOE_ERR_BOUNDS, "num_points must be >= 1");
    CMOE_REQUIRE(num_shared >= 0, CMOE_ERR_BOUNDS, "num_shared must be >= 0");
    CMOE_REQUIRE(params->max_num_steps <= 1 << 20, CMOE_ERR_BOUNDS, "max_num_steps too large");
    CMOE_REQUIRE(num_fidelity >= 0, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    check_ensemble(gps, num_gp);
    const int dim = gps[0]->spec.dim, ps = dim - num_fidelity;
    CMOE_REQUIRE(ps >= 1, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    for (int d = 0; d < ps; ++d)
      CMOE_REQUIRE(domain_bounds[2 * d] <= domain_bounds[2 * d + 1], CMOE_ERR_BOUNDS, "Tensor product region is EMPTY.");
    const size_t M = num_gp, P = num_points, lists = points_per_member ? M : 1, steps = std::max(0, params->max_num_steps);
    for (size_t k = 0; k < lists * P * ps; ++k)
      CMOE_REQUIRE(std::isfinite(points[k]), CMOE_ERR_INVALID_VALUE, "screen points must be finite");
    for (size_t k = 0; k < static_cast<size_t>(num_shared) * ps; ++k)
      CMOE_REQUIRE(std::isfinite(shared_discrete[k]), CMOE_ERR_INVALID_VALUE, "shared_discrete must be finite");
    int max_N = 0;
    for (int m = 0; m < num_gp; ++m) max_N = std::max(max_N, gps[m]->N);
    const size_t total = P + (include_sampled ? max_N : 0);  // the longest member's screen list
    CMOE_REQUIRE(total <= static_cast<size_t>(std::numeric_limits<int>::max()), CMOE_ERR_BOUNDS,
                 "num_points + num_sampled must fit an int");
    require_device(gps[0]->device);
    join_member_streams(gps, num_gp);
    cudaStream_t s = gps[0]->stream;

    PmDescent prm{};
    prm.ps = ps;
    prm.max_steps = params->max_num_steps;
    prm.max_restarts = params->max_num_restarts;
    prm.mrc = params->max_relative_change;
    prm.tol = params->tolerance;
    for (int d = 0; d < CMOE_MAX_DIM; ++d) {
      prm.lo[d] = (d < ps) ? domain_bounds[2 * d] : -1e300;
      prm.hi[d] = (d < ps) ? domain_bounds[2 * d + 1] : 1e300;
    }
    // screen indices per chunk: the chunk's given points and its values fit kPmOptimaWorkspaceBytes
    const size_t chunk =
        std::max<size_t>(1, std::min(total, kPmOptimaWorkspaceBytes / (sizeof(double) * (M + lists * ps))));
    // one staging buffer, one upload: member table | step sizes | shared discrete points | the chunk's given points
    const size_t o_alpha = M * sizeof(PmMember) / sizeof(double), o_shared = o_alpha + steps,
                 o_pts = o_shared + static_cast<size_t>(num_shared) * ps, given_max = std::min(chunk, P);
    std::vector<double> stage(o_pts + lists * given_max * ps);
    static_assert(sizeof(PmMember) % sizeof(double) == 0, "the member table is staged as doubles");
    for (int m = 0; m < num_gp; ++m) {
      const PmMember mb{gps[m]->spec, gps[m]->dX.p, gps[m]->dKinvY.p, gps[m]->mean, gps[m]->N};
      std::memcpy(stage.data() + m * (sizeof(PmMember) / sizeof(double)), &mb, sizeof(PmMember));
    }
    for (size_t i = 0; i < steps; ++i)
      stage[o_alpha + i] = gd_step_size(params->pre_mult, params->gamma, i);
    std::copy(shared_discrete, shared_discrete + static_cast<size_t>(num_shared) * ps, stage.begin() + o_shared);
    const size_t W = kPmStateHead + 2 * ps;
    DevBuf<double> dIn(stage.size()), dV(M * chunk), dState(M * W);
    const PmMember* dMem = reinterpret_cast<const PmMember*>(dIn.p);
    for (size_t i0 = 0; i0 < total; i0 += chunk) {
      const size_t len = std::min(chunk, total - i0), given = i0 < P ? std::min(len, P - i0) : 0;
      for (size_t l = 0; l < lists; ++l)
        std::copy(points + (l * P + i0) * ps, points + (l * P + i0 + given) * ps, stage.begin() + o_pts + l * given * ps);
      const size_t first = i0 == 0 ? 0 : o_pts, count = o_pts + lists * given * ps - first;
      if (count) CMOE_CUDA(cudaMemcpyAsync(dIn.p + first, stage.data() + first, count * sizeof(double),
                                           cudaMemcpyHostToDevice, s));
      pm_members_screen_kernel<<<static_cast<unsigned>(M * len), kPmScreenParts, 0, s>>>(
          dMem, ps, dIn.p + o_pts, points_per_member != 0, num_points, include_sampled != 0, static_cast<int>(i0),
          static_cast<int>(len), static_cast<int>(given), dV.p);
      pm_members_argmin_kernel<<<num_gp, kPmOptimaThreads, 0, s>>>(
          dMem, ps, dIn.p + o_pts, points_per_member != 0, num_points, include_sampled != 0, static_cast<int>(i0),
          static_cast<int>(len), static_cast<int>(given), dV.p, dState.p);
      count_launch(2);
      CMOE_CUDA(cudaGetLastError());
    }
    pm_members_opt_kernel<<<num_gp, kPmOptimaThreads, 0, s>>>(prm, dMem, dIn.p + o_alpha, dIn.p + o_shared, num_shared,
                                                              dState.p);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    std::vector<double> res(M * W);
    dState.download(res.data(), res.size(), s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    for (size_t m = 0; m < M; ++m) {
      const double* r = res.data() + m * W;
      const double* opt = r + kPmStateHead + ps;
      std::copy(opt, opt + ps, optima + m * ps);
      if (screen_min) screen_min[m] = r[0];
      if (start_index) start_index[m] = static_cast<int>(r[1]);
      if (optimum_means) optimum_means[m] = r[2];
      if (best_so_far) best_so_far[m] = r[3];
      if (kept_start) kept_start[m] = static_cast<int>(r[4]);
      if (discrete_pts) {
        double* dp = discrete_pts + m * (static_cast<size_t>(num_shared) + 1) * ps;
        std::copy(stage.begin() + o_shared, stage.begin() + o_pts, dp);
        std::copy(opt, opt + ps, dp + static_cast<size_t>(num_shared) * ps);
      }
    }
  });
}

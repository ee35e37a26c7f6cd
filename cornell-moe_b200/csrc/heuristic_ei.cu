// Heuristic batch EI in one device call (DESIGN.md K20): Constant Liar and Kriging Believer.
//
// Replaces (reference): ComputeHeuristicPointsToSample (gpp_python_expected_improvement.cpp:602-659) with the
// estimation policies (:445-486) and, per round, ComputeOptimalPointsToSample for q = 1 (gpp_math.cpp:2369-2429):
//
//   for r in 0 .. q-1:
//     x_r = arg max 1-EI over the start block r (screen, top 20, restarted gradient descent, strict `<` from -1)
//     y_r = policy estimate at x_r on the current GP;  GP <- GP + (x_r, y_r, noise)
//
// Every round works on a private copy of the caller's GP (clone_gp_to_device); per round:
//   screen            analytic_ei on the copy (cmoe_ei_analytic's values), one synchronise; top 20 on the host
//   hei_descent_kernel one CTA per kept start runs its whole restarted descent (gradient_descent_batch's rules); an
//                     evaluation builds k(X, x) on the fly, v = L^-1 k and w = L^-T v by in-CTA blocked solves against
//                     the copy's factor, then the closed-form EI and its gradient
//   hei_select_kernel  the strict-`<` winner and its EI; Kriging Believer's mu and sigma^2 there from cmoe_gp_posterior
//   append_points      the winner with the estimate and the policy's noise (O(N^2) bordered factor)
// so the host synchronises a fixed number of times per round, whatever the step count.
#include <cmath>

#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {

namespace {

constexpr int kHeiThreads = 256;
constexpr int kHeiWarps = kHeiThreads / 32;
constexpr int kHeiOut = 1;  // per start after its coordinates: its EI

// The optimiser's and the GP copy's constants, identical for every CTA.
struct HeiParams {
  KernelSpec spec;
  const double* X;     // [N][dim] training points of the round's copy
  const double* beta;  // [N] K^-1 (y - mean)
  const double* L;     // [N][N] column-major lower Cholesky factor
  int N;
  double mean, best, kxx;  // prior mean, best_so_far, k(x, x)
  int max_steps, max_restarts;
  double mrc, tol, step_tol;
  double lo[CMOE_MAX_DIM], hi[CMOE_MAX_DIM];
};

struct HeiShared {
  double x[CMOE_MAX_DIM];    // the evaluation point
  double x0[CMOE_MAX_DIM];   // the point a restart began from
  double g[CMOE_MAX_DIM];    // EI gradient
  double tile[32][33];       // diagonal block of L: tile[r][c] = L(i0 + r, i0 + c)
  double inv[32];            // 1 / L(i0 + c, i0 + c)
  double part[kHeiWarps][33];
  double red[2 * kHeiThreads];
  int stop;
};

// tile <- the lower triangle of L's diagonal block at i0 (nb rows), inv <- the reciprocals of its diagonal
__device__ __forceinline__ void load_diag_block(const double* __restrict__ L, int n, int i0, int nb, HeiShared& sh) {
  for (int e = threadIdx.x; e < 32 * 32; e += kHeiThreads) {
    const int c = e >> 5, r = e & 31;
    if (r < nb && c <= r) {
      const double v = L[static_cast<size_t>(i0 + c) * n + i0 + r];
      sh.tile[r][c] = v;
      if (r == c) sh.inv[c] = 1.0 / v;
    }
  }
}

// vec <- L^-1 vec (shared, n entries), left-looking by 32-row blocks: every warp adds the products of the columns
// j = warp (mod 8) below the block for its lane's row (coalesced down a column), then warp 0 combines the eight partials
// in warp order and solves the diagonal block by lane-parallel column sweeps.
__device__ void forward_solve(const double* __restrict__ L, int n, double* vec, HeiShared& sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int nb = min(32, n - i0);
    load_diag_block(L, n, i0, nb, sh);
    double a = 0.0;
    if (lane < nb)
      for (int j = warp; j < i0; j += kHeiWarps) a = fma(L[static_cast<size_t>(j) * n + i0 + lane], vec[j], a);
    sh.part[warp][lane] = a;
    __syncthreads();
    if (warp == 0) {
      double b = 0.0, res = 0.0;
      if (lane < nb) {
        b = vec[i0 + lane];
        for (int w = 0; w < kHeiWarps; ++w) b -= sh.part[w][lane];
      }
      for (int c = 0; c < nb; ++c) {
        const double xc = __shfl_sync(0xffffffffu, b, c) * sh.inv[c];
        if (lane == c) res = xc;
        else if (lane > c && lane < nb) b = fma(-sh.tile[lane][c], xc, b);
      }
      if (lane < nb) vec[i0 + lane] = res;
    }
    __syncthreads();
  }
}

// vec <- L^-T vec, blocks from the bottom: row i of L^T is column i of L, so each of a block's rows is one coalesced dot
// product over the rows below the block (warp per row, butterfly sum), then warp 0 solves the diagonal block.
__device__ void back_solve(const double* __restrict__ L, int n, double* vec, HeiShared& sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i0 = ((n - 1) / 32) * 32; i0 >= 0; i0 -= 32) {
    const int nb = min(32, n - i0);
    load_diag_block(L, n, i0, nb, sh);
    for (int r = warp; r < nb; r += kHeiWarps) {
      const double* Lr = L + static_cast<size_t>(i0 + r) * n;
      double a = 0.0;
      for (int j = i0 + nb + lane; j < n; j += 32) a = fma(Lr[j], vec[j], a);
      a = warp_sum(a);
      if (lane == 0) sh.part[0][r] = a;
    }
    __syncthreads();
    if (warp == 0) {
      double b = (lane < nb) ? vec[i0 + lane] - sh.part[0][lane] : 0.0, res = 0.0;
      for (int c = nb - 1; c >= 0; --c) {
        const double xc = __shfl_sync(0xffffffffu, b, c) * sh.inv[c];
        if (lane == c) res = xc;
        else if (lane < c) b = fma(-sh.tile[c][lane], xc, b);
      }
      if (lane < nb) vec[i0 + lane] = res;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ double norm_pdf(double z) { return exp(-0.5 * z * z) * 0.39894228040143267793994605993438; }
__device__ __forceinline__ double norm_cdf(double z) { return 0.5 * erfc(-z * 0.70710678118654752440084436210485); }

// 1-EI at sh.x (and, with grad, its gradient into sh.g) on the round's GP, for the whole CTA; every thread returns the
// same bits, and mu, var receive the posterior mean and the f-variance k(x,x) - |L^-1 k|^2.  vec and kb are shared
// scratch of N doubles each.  The EI arithmetic is analytic_ei's (gpp_math.cpp:2196-2253).
__device__ __forceinline__ double hei_eval(const HeiParams& p, HeiShared& sh, double* vec, double* kb, bool grad,
                                        double& mu, double& var) {
  const int tid = threadIdx.x, dim = p.spec.dim, N = p.N;
  double acc = 0.0;
  for (int j = tid; j < N; j += kHeiThreads) {
    const KParts kp = kernel_parts(p.spec, weighted_sqdist(p.spec, sh.x, p.X + static_cast<size_t>(j) * dim));
    vec[j] = kp.A;
    kb[j] = kp.B;
    acc = fma(kp.A, p.beta[j], acc);
  }
  mu = p.mean + block_sum(acc, sh.red);  // its barriers also publish vec and kb
  forward_solve(p.L, N, vec, sh);
  acc = 0.0;
  for (int j = tid; j < N; j += kHeiThreads) acc = fma(vec[j], vec[j], acc);
  var = p.kxx - block_sum(acc, sh.red);
  const double kMinVarEI = 2.2250738585072014e-308;                          // numeric_limits<double>::min()
  const double kMinVarGradEI = 150.0 * 2.220446049250313e-16 * 2.220446049250313e-16;  // 150 eps^2
  const double t = p.best - mu;
  double ei;
  {
    const double sigma = sqrt(fmax(kMinVarEI, var));
    ei = fmax(0.0, t * norm_cdf(t / sigma) + sigma * norm_pdf(t / sigma));
  }
  if (!grad) return ei;
  back_solve(p.L, N, vec, sh);
  // component i of grad mu and of (dk/dx)^T w: thread (i, part) sums the rows part, part + parts, ... in ascending order
  const int parts = kHeiThreads / dim, i = tid % dim, part = tid / dim;
  double am = 0.0, aw = 0.0;
  if (part < parts) {
    const double xi = sh.x[i], li = p.spec.lsq[i];
    for (int j = part; j < N; j += parts) {
      const double dk = (p.X[static_cast<size_t>(j) * dim + i] - xi) / li * kb[j];
      am = fma(dk, p.beta[j], am);
      aw = fma(dk, vec[j], aw);
    }
  }
  sh.red[tid] = am;
  sh.red[kHeiThreads + tid] = aw;
  __syncthreads();
  if (tid < dim) {
    double sm = 0.0, sw = 0.0;
    for (int q = 0; q < parts; ++q) {
      sm += sh.red[q * dim + tid];
      sw += sh.red[kHeiThreads + q * dim + tid];
    }
    const double v = fmax(kMinVarGradEI, var), sigma = sqrt(v);
    const double C = t / sigma, pdf_C = norm_pdf(C), cdf_C = norm_cdf(C);
    const double gm = sm, gchol = 0.5 * (-2.0 * sw) / sigma;
    const double d_C = (-sigma * gm - gchol * t) / v;
    const double d_A = -gm * cdf_C + t * pdf_C * d_C;
    const double d_B = gchol * pdf_C + sigma * (-C) * pdf_C * d_C;
    sh.g[tid] = d_A + d_B;
  }
  __syncthreads();
  return ei;
}

// grid.x = kept starts (starts [k][dim]).  One start's restarted descent with gradient_descent_batch's rules
// (multistart.cu): steps a[i] = pre_mult (i + 1)^-gamma, limit_step per coordinate, a run ends when a step is shorter
// than tol / max_steps, a restart is skipped once a run moved no more than tol; then a value-only evaluation at the end
// point.  Thread 0 takes each step (in coordinate order, rounded as the host rounds), the CTA evaluates.
// res [k][dim + 1]: end point, EI.
__global__ void __launch_bounds__(kHeiThreads, 1) hei_descent_kernel(const __grid_constant__ HeiParams p,
                                                                  const double* __restrict__ starts,
                                                                  const double* __restrict__ steps,
                                                                  double* __restrict__ res) {
  extern __shared__ double hei_smem[];
  __shared__ HeiShared sh;
  double* vec = hei_smem;
  double* kb = hei_smem + p.N;
  const int tid = threadIdx.x, dim = p.spec.dim;
  if (tid < dim) sh.x[tid] = starts[static_cast<size_t>(blockIdx.x) * dim + tid];
  __syncthreads();
  double mu, var;
  bool converged = false;
  for (int r = 0; r < p.max_restarts && !converged; ++r) {
    if (tid < dim) sh.x0[tid] = sh.x[tid];
    for (int i = 0; i < p.max_steps; ++i) {
      hei_eval(p, sh, vec, kb, true, mu, var);
      if (tid == 0) {
        double ns2 = 0.0;
        for (int d = 0; d < dim; ++d) {
          const double step = limit_step(steps[i] * sh.g[d], sh.x[d], p.lo[d], p.hi[d], p.mrc);
          sh.x[d] += step;
          ns2 = __dadd_rn(ns2, __dmul_rn(step, step));
        }
        sh.stop = sqrt(ns2) < p.step_tol;
      }
      __syncthreads();
      if (sh.stop) break;
    }
    __syncthreads();
    if (tid == 0) {
      double nd = 0.0;
      for (int d = 0; d < dim; ++d) {
        const double df = sh.x0[d] - sh.x[d];
        nd = __dadd_rn(nd, __dmul_rn(df, df));
      }
      sh.stop = sqrt(nd) <= p.tol;
    }
    __syncthreads();
    converged = sh.stop;
    __syncthreads();
  }
  const double ei = hei_eval(p, sh, vec, kb, false, mu, var);
  if (tid == 0) {
    double* out = res + static_cast<size_t>(blockIdx.x) * (dim + kHeiOut);
    for (int d = 0; d < dim; ++d) out[d] = sh.x[d];
    out[dim] = ei;
  }
}

// The round's winner among `count` candidates (cand [count][dim + 1], EI at dim): best -1, strict `<` in candidate
// order, `first` when none wins (multistart_common's OptimizationIOContainer).  out [dim + 2]: the point, its EI (or
// -1), found.  One thread: count is at most the number of starts.
__global__ void hei_select_kernel(int dim, const double* __restrict__ cand, int count, const double* __restrict__ first,
                                  double* __restrict__ out) {
  const int stride = dim + kHeiOut;
  double best = -1.0;
  int bi = -1;
  for (int c = 0; c < count; ++c) {
    const double v = cand[static_cast<size_t>(c) * stride + dim];
    if (best < v) {
      best = v;
      bi = c;
    }
  }
  const double* x = (bi >= 0) ? cand + static_cast<size_t>(bi) * stride : first;
  for (int d = 0; d < dim; ++d) out[d] = x[d];
  out[dim] = best;
  out[dim + 1] = (bi >= 0) ? 1.0 : 0.0;
}

struct GpDeleter {
  void operator()(cmoe_gp* gp) const { cmoe_gp_destroy(gp); }
};

}  // namespace

}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_heuristic_ei(const cmoe_gp* gp, const cmoe_estimation_policy* policy, const cmoe_gd_params* gd,
                                 const double* domain_bounds, const double* starts, int num_starts, int q,
                                 double best_so_far, double* points, double* fantasy_values, double* ei_values,
                                 int* found, int* info) {
  return guarded(info, [&] {
    // every check comes before any device work; those that need no GP handle come first
    CMOE_REQUIRE(q >= 1, CMOE_ERR_BOUNDS, "num_to_sample must be >= 1");
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be >= 1");
    CMOE_REQUIRE(!gd || gd->max_num_steps <= 1 << 20, CMOE_ERR_BOUNDS, "max_num_steps too large");
    CMOE_REQUIRE(policy != nullptr, CMOE_ERR_INVALID_VALUE, "policy must not be NULL");
    CMOE_REQUIRE(policy->policy == CMOE_ESTIMATION_CONSTANT_LIAR || policy->policy == CMOE_ESTIMATION_KRIGING_BELIEVER,
                 CMOE_ERR_INVALID_VALUE, "unknown estimation policy");
    CMOE_REQUIRE(std::isfinite(policy->value), CMOE_ERR_INVALID_VALUE,
                 "the lie value / std_deviation_coef must be finite");
    CMOE_REQUIRE(policy->noise_variance >= 0.0, CMOE_ERR_INVALID_VALUE, "the policy's noise_variance must be >= 0");
    CMOE_REQUIRE(gp != nullptr && domain_bounds != nullptr && starts != nullptr && points != nullptr,
                 CMOE_ERR_INVALID_VALUE, "gp, domain_bounds, starts and points must not be NULL");
    CMOE_REQUIRE(gp->spec.g == 0, CMOE_ERR_BOUNDS,
                 "heuristic EI: an estimation policy gives function values only, so a GP with derivative observations "
                 "has no fantasy rows");
    const int dim = gp->spec.dim;
    validate_bounds(domain_bounds, dim);
    require_device(gp->device);
    const long long rows = static_cast<long long>(gp->N) + q - 1;  // the largest copy the descent sees
    int smem_max = 0;
    CMOE_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, gp->device));
    const size_t smem_static = sizeof(HeiShared) + 64;
    CMOE_REQUIRE(rows * 2 * sizeof(double) + smem_static <= static_cast<size_t>(smem_max), CMOE_ERR_BOUNDS,
                 "heuristic EI: num_sampled + num_to_sample - 1 exceeds the rows one CTA holds in shared memory");
    CMOE_CUDA(cudaFuncSetAttribute(hei_descent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   smem_max - static_cast<int>(smem_static)));

    std::unique_ptr<cmoe_gp, GpDeleter> w(clone_gp_to_device(gp, gp->device));
    cudaStream_t s = w->stream;
    HeiParams prm{};
    prm.spec = gp->spec;
    prm.best = best_so_far;
    for (int d = 0; d < CMOE_MAX_DIM; ++d) {
      prm.lo[d] = d < dim ? domain_bounds[2 * d] : 0.0;
      prm.hi[d] = d < dim ? domain_bounds[2 * d + 1] : 0.0;
    }
    const int k = std::min(kTopK, num_starts);
    DevBuf<double> dSteps, dKept(static_cast<size_t>(k) * dim), dRes, dOut(dim + 2);
    if (gd) {
      prm.max_steps = gd->max_num_steps;
      prm.max_restarts = gd->max_num_restarts;
      prm.mrc = gd->max_relative_change;
      prm.tol = gd->tolerance;
      prm.step_tol = gd->tolerance / static_cast<double>(gd->max_num_steps);  // as gradient_descent_batch
      std::vector<double> a(std::max(1, gd->max_num_steps));
      for (int i = 0; i < gd->max_num_steps; ++i) a[i] = gd_step_size(gd->pre_mult, gd->gamma, i);
      dSteps.upload(a.data(), a.size(), s);
      dRes.alloc(static_cast<size_t>(k) * (dim + kHeiOut));
    } else {
      dRes.alloc(static_cast<size_t>(num_starts) * (dim + kHeiOut));
    }
    const double noise[1] = {policy->noise_variance};
    std::vector<double> vals(num_starts), host(dRes.count), out(dim + 2);
    for (int r = 0; r < q; ++r) {
      const double* S = starts + static_cast<size_t>(r) * num_starts * dim;
      analytic_ei(w.get(), S, num_starts, best_so_far, vals.data(), nullptr);  // the screen
      prm.X = w->dX.p;
      prm.beta = w->dKinvY.p;
      prm.L = w->dK.p;
      prm.N = w->N;
      prm.mean = w->mean;
      prm.kxx = w->spec.alpha;  // k(x, x) of both kernels
      const size_t smem = static_cast<size_t>(w->N) * 2 * sizeof(double);
      if (gd) {
        const std::vector<int> top = top_k_indices(vals.data(), num_starts);
        for (int i = 0; i < k; ++i)
          std::copy(S + static_cast<size_t>(top[i]) * dim, S + static_cast<size_t>(top[i] + 1) * dim,
                    host.begin() + static_cast<size_t>(i) * dim);
        CMOE_CUDA(cudaMemcpyAsync(dKept.p, host.data(), static_cast<size_t>(k) * dim * sizeof(double),
                                  cudaMemcpyHostToDevice, s));
        hei_descent_kernel<<<k, kHeiThreads, smem, s>>>(prm, dKept.p, dSteps.p, dRes.p);
        hei_select_kernel<<<1, 1, 0, s>>>(dim, dRes.p, k, dKept.p, dOut.p);
        count_launch(2);
      } else {
        // kNull: the candidates are the screened starts themselves
        const size_t stride = dim + kHeiOut;
        for (int c = 0; c < num_starts; ++c) {
          std::copy(S + static_cast<size_t>(c) * dim, S + static_cast<size_t>(c + 1) * dim, host.begin() + c * stride);
          host[c * stride + dim] = vals[c];
        }
        dRes.upload(host.data(), num_starts * stride, s);
        hei_select_kernel<<<1, 1, 0, s>>>(dim, dRes.p, num_starts, dRes.p, dOut.p);
        count_launch();
      }
      CMOE_CUDA(cudaGetLastError());
      dOut.download(out.data(), out.size(), s);
      CMOE_CUDA(cudaStreamSynchronize(s));
      // Kriging Believer: mu and the f-variance at the winner as cmoe_gp_posterior returns them on the round's GP
      double y = policy->value;
      if (policy->policy == CMOE_ESTIMATION_KRIGING_BELIEVER) {
        double mu = 0.0, var = 0.0;
        int pinfo = 0;
        const int rc = cmoe_gp_posterior(w.get(), out.data(), 1, 1, nullptr, 0, &mu, nullptr, &var, nullptr, nullptr,
                                         nullptr, &pinfo);
        if (rc != CMOE_OK) throw Error(rc, cmoe_last_error(), pinfo);
        y = mu + policy->value * std::sqrt(std::fmax(var, 0.0));
      }
      std::copy(out.begin(), out.begin() + dim, points + static_cast<size_t>(r) * dim);
      if (ei_values) ei_values[r] = out[dim];
      if (fantasy_values) fantasy_values[r] = y;
      if (found) found[r] = out[dim + 1] != 0.0;
      append_points(w.get(), out.data(), &y, 1, noise);
    }
  });
}

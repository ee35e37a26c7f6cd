// Batched GP-posterior set-up: for nc point sets at once, K* -> K^-1 K* -> mean, variance, q*q Cholesky and the
// gradients of mean / variance / Cholesky factor.  One CTA (or a small CTA grid) per point set; the N-sized
// contractions stream K* and K^-1 K* (L2-resident) and re-evaluate the kernel gradient on the fly instead of
// materialising the reference's grad_K_star tensor.
//
// Replaces (reference, moe/optimal_learning/cpp/gpp_math.cpp):
//   FillPointsToSampleState                      :600-653
//   ComputeMeanOfPoints / ComputeGradMeanOfPoints :662-678 / :721-726
//   ComputeVarianceOfPoints                       :924-970
//   ComputeGradVarianceOfPointsPerPoint           :1267-1358
//   ComputeGradCholeskyVarianceOfPointsPerPoint   :1389-1458 (Smith 1995)
// and the q*q ComputeCholeskyFactorL calls of the EI / KG states (gpp_math.cpp:2064,
// gpp_knowledge_gradient_optimization.cpp:310).
#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {

namespace {

constexpr double kPivotTol = 1.0e-16;
constexpr double kMinimumStdDev = 2.220446049250313e-16;  // gpp_math.hpp:291

__device__ __forceinline__ int row_type(int local, const int* derivs) { return local ? derivs[local - 1] : -1; }

// --------------------------------------------------------------------------------------------------------------
// mean, variance, Cholesky of (variance + diagonal term) for one point set per CTA
//   diag_mode 0: nothing added; 1: +1e-6 (EI, gpp_math.cpp:2000-2002); 2: +noise[type] (KG, ...optimization.cpp:304-309)
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) post_var_kernel(const __grid_constant__ KernelSpec spec, int n, double mean,
                                                       const double* __restrict__ beta,
                                                       const double* __restrict__ noise,
                                                       const double* __restrict__ P, int num,
                                                       const int* __restrict__ dPs, int gs,
                                                       const double* __restrict__ Ks, const double* __restrict__ B,
                                                       int diag_mode, double* __restrict__ mu,
                                                       double* __restrict__ var, double* __restrict__ chol,
                                                       int* __restrict__ fail) {
  extern __shared__ double sm[];
  const int c = blockIdx.x, bs = 1 + gs, Q = num * bs, dim = spec.dim;
  double* V = sm;                  // [Q][Q+1]
  double* Ps = sm + Q * (Q + 1);   // [num][dim]
  __shared__ int failed;
  const int tid = threadIdx.x;
  for (int e = tid; e < num * dim; e += blockDim.x) Ps[e] = P[static_cast<size_t>(c) * num * dim + e];
  if (tid == 0) failed = 0;
  __syncthreads();
  const double* Kc = Ks + static_cast<size_t>(c) * Q * n;
  const double* Bc = B + static_cast<size_t>(c) * Q * n;
  for (int a = tid; a < Q; a += blockDim.x) {
    const double* ka = Kc + static_cast<size_t>(a) * n;
    double t = 0.0;
    for (int j = 0; j < n; ++j) t += ka[j] * beta[j];
    mu[static_cast<size_t>(c) * Q + a] = ((a % bs == 0) ? mean : 0.0) + t;
  }
  for (int o = tid; o < Q * Q; o += blockDim.x) {
    const int a = o % Q, b = o / Q;
    // Var(a, b) = K(Xs_a, Xs_b) - (K^-1 K*)_a^T K*_b    (precomputed branch, gpp_math.cpp:962-968)
    const double* ba = Bc + static_cast<size_t>(a) * n;
    const double* kb = Kc + static_cast<size_t>(b) * n;
    double t = 0.0;
    for (int j = 0; j < n; ++j) t += ba[j] * kb[j];
    const int pa = a / bs, pb = b / bs;
    const double* p1 = Ps + pa * dim;
    const double* p2 = Ps + pb * dim;
    const KParts kp = kernel_parts(spec, weighted_sqdist(spec, p1, p2));
    const double v = cov_entry(spec, kp, p1, p2, row_type(a % bs, dPs), row_type(b % bs, dPs)) - t;
    V[a * (Q + 1) + b] = v;
    if (var) var[static_cast<size_t>(c) * Q * Q + o] = v;
  }
  __syncthreads();
  if (chol == nullptr) return;
  if (diag_mode != 0) {
    for (int a = tid; a < Q; a += blockDim.x) V[a * (Q + 1) + a] += (diag_mode == 1) ? 1.0e-6 : noise[a % bs];
    __syncthreads();
  }
  // unblocked right-looking Cholesky (gpp_linear_algebra.cpp:109-148) on the lower triangle
  for (int j = 0; j < Q; ++j) {
    if (tid == 0) {
      const double piv = V[j * (Q + 1) + j];
      if (piv > kPivotTol) {
        V[j * (Q + 1) + j] = sqrt(piv);
      } else {
        failed = j + 1;
      }
    }
    __syncthreads();
    if (failed) break;
    const double ljj = V[j * (Q + 1) + j];
    for (int i = j + 1 + tid; i < Q; i += blockDim.x) V[i * (Q + 1) + j] /= ljj;
    __syncthreads();
    const int m = Q - j - 1;
    for (int e = tid; e < m * m; e += blockDim.x) {
      const int cc = j + 1 + e / m, i = j + 1 + e % m;
      if (i >= cc) V[i * (Q + 1) + cc] = V[i * (Q + 1) + cc] - V[i * (Q + 1) + j] * V[cc * (Q + 1) + j];
    }
    __syncthreads();
  }
  if (tid == 0) fail[c] = failed;
  for (int o = tid; o < Q * Q; o += blockDim.x) {
    const int a = o % Q, b = o / Q;  // column-major out: element (a, b)
    chol[static_cast<size_t>(c) * Q * Q + o] = (a >= b) ? V[a * (Q + 1) + b] : 0.0;  // ZeroUpperTriangle
  }
}

// --------------------------------------------------------------------------------------------------------------
// E[delta, b, col] = sum_rows dK*[delta, row, col] * (K^-1 K*)[row, b]  and  grad_mu[delta, col] = sum_rows dK* beta
// grid (nc, nd*bs); the kernel gradient d cov(P_i type m, X_j type cc)/d P_i is re-evaluated on the fly.
// --------------------------------------------------------------------------------------------------------------
constexpr int kChunk = 128;

__global__ void __launch_bounds__(kChunk) post_gradE_kernel(const __grid_constant__ KernelSpec spec, int N,
                                                            const double* __restrict__ X,
                                                            const double* __restrict__ beta,
                                                            const double* __restrict__ P, int num,
                                                            const int* __restrict__ dPs, int gs, int nd,
                                                            const double* __restrict__ B, double* __restrict__ E,
                                                            double* __restrict__ gmu) {
  extern __shared__ double sm[];
  const int c = blockIdx.x, col = blockIdx.y, bs = 1 + gs, Q = num * bs, dim = spec.dim, b1 = 1 + spec.g;
  const int n = N * b1;
  const int i = col / bs, a1 = row_type(col % bs, dPs);
  double* Pi = sm;                                  // [dim]
  double* Xc = sm + dim;                            // [kChunk][dim]
  KParts* kps = reinterpret_cast<KParts*>(Xc + kChunk * dim);  // [kChunk]
  const int tid = threadIdx.x;
  for (int e = tid; e < dim; e += blockDim.x) Pi[e] = P[(static_cast<size_t>(c) * num + i) * dim + e];
  const int nout = dim * (Q + 1);
  const double* Bc = B + static_cast<size_t>(c) * Q * n;
  for (int o0 = 0; o0 < nout; o0 += blockDim.x) {
    const int o = o0 + tid;
    const int delta = o % dim, b = o / dim;  // b == Q -> grad mean
    const double* vec = (b < Q) ? (Bc + static_cast<size_t>(b) * n) : beta;
    double acc = 0.0;
    for (int j0 = 0; j0 < N; j0 += kChunk) {
      __syncthreads();
      const int jj = j0 + tid;
      if (jj < N) {
        for (int e = 0; e < dim; ++e) Xc[tid * dim + e] = X[static_cast<size_t>(jj) * dim + e];
        kps[tid] = kernel_parts(spec, weighted_sqdist(spec, Pi, Xc + tid * dim));
      }
      __syncthreads();
      if (o < nout) {
        const int cnt = min(kChunk, N - j0);
        for (int t = 0; t < cnt; ++t) {
          for (int cc = 0; cc < b1; ++cc) {
            const double gval =
                grad_cov_entry(spec, kps[t], Pi, Xc + t * dim, a1, row_type(cc, spec.derivs), delta);
            acc += gval * vec[(j0 + t) * b1 + cc];
          }
        }
      }
    }
    if (o < nout) {
      if (b < Q) {
        E[((static_cast<size_t>(c) * nd * bs + col) * Q + b) * dim + delta] = acc;
      } else {
        gmu[(static_cast<size_t>(c) * nd * bs + col) * dim + delta] = acc;
      }
    }
  }
}

// --------------------------------------------------------------------------------------------------------------
// Mean (and its gradient) of ANY number of points without forming K^-1 K*: one CTA per point,
//   mu(x, type a) = [a == value] mean + sum_j sum_cc cov(x type a, X_j type cc) beta_(j,cc)
// (GaussianProcess::ComputeMeanOfPoints / ComputeGradMeanOfPoints, gpp_math.cpp:600-653; the points are independent, so
// the (q+p)(1+g) <= 96 bound of the variance kernels does not apply — this is the screening call the front end makes
// with 1e3-1e4 points).  Threads = (output, slice of the training points); slices are combined in a fixed order.
// --------------------------------------------------------------------------------------------------------------
constexpr int kMeanThreads = 128;

__global__ void __launch_bounds__(kMeanThreads) post_mean_only_kernel(const __grid_constant__ KernelSpec spec, int N,
                                                                      double mean, const double* __restrict__ X,
                                                                      const double* __restrict__ beta,
                                                                      const double* __restrict__ P,
                                                                      const int* __restrict__ dPs, int gs,
                                                                      double* __restrict__ mu,
                                                                      double* __restrict__ gmu) {
  __shared__ double Pi[CMOE_MAX_DIM];
  __shared__ double red[kMeanThreads];
  const int pt = blockIdx.x, bs = 1 + gs, dim = spec.dim, b1 = 1 + spec.g;
  const int per = gmu ? 1 + dim : 1;       // outputs per row type: value [+ dim gradient components]
  const int nout = bs * per;
  const int tid = threadIdx.x;
  for (int e = tid; e < dim; e += blockDim.x) Pi[e] = P[static_cast<size_t>(pt) * dim + e];
  __syncthreads();
  for (int o0 = 0; o0 < nout; o0 += kMeanThreads) {
    const int group = min(nout - o0, kMeanThreads);  // outputs handled in this pass
    const int nparts = kMeanThreads / group;
    const int o = o0 + tid % group, part = tid / group;
    double acc = 0.0;
    if (part < nparts) {
      const int a1 = row_type((o / per), dPs), comp = o % per;
      for (int j = part; j < N; j += nparts) {
        const double* xj = X + static_cast<size_t>(j) * dim;
        const KParts kp = kernel_parts(spec, weighted_sqdist(spec, Pi, xj));
        for (int cc = 0; cc < b1; ++cc) {
          const int a2 = row_type(cc, spec.derivs);
          const double v = (comp == 0) ? cov_entry(spec, kp, Pi, xj, a1, a2)
                                       : grad_cov_entry(spec, kp, Pi, xj, a1, a2, comp - 1);
          acc = fma(v, beta[static_cast<size_t>(j) * b1 + cc], acc);
        }
      }
    }
    red[tid] = acc;
    __syncthreads();
    if (part == 0 && tid < group) {
      double t = 0.0;
      for (int q = 0; q < nparts; ++q) t += red[q * group + tid];
      const int row = o / per, comp = o % per;
      if (comp == 0) {
        mu[static_cast<size_t>(pt) * bs + row] = ((row == 0) ? mean : 0.0) + t;
      } else {
        gmu[(static_cast<size_t>(pt) * bs + row) * dim + comp - 1] = t;
      }
    }
    __syncthreads();
  }
}

// --------------------------------------------------------------------------------------------------------------
// grad variance wrt point p (reference layout gv[delta + row*dim + col*dim*Q]); grid (nc, nd)
// With F(delta; colp, other) = -E[delta, other, colp] + d cov(P_p type(colp), P_other type(other)) / d P_p,delta :
//   row in p, col not in p (and the mirror): F ;  both in p: F(col,row) + F(row,col) ;  neither: 0.
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) post_gradvar_kernel(const __grid_constant__ KernelSpec spec,
                                                           const double* __restrict__ P, int num,
                                                           const int* __restrict__ dPs, int gs, int nd,
                                                           const double* __restrict__ E, double* __restrict__ gvar) {
  const int c = blockIdx.x, p = blockIdx.y, bs = 1 + gs, Q = num * bs, dim = spec.dim;
  const double* Pc = P + static_cast<size_t>(c) * num * dim;
  const double* Ec = E + static_cast<size_t>(c) * nd * bs * Q * dim;
  double* out = gvar + (static_cast<size_t>(c) * nd + p) * Q * Q * dim;
  const double* pp = Pc + p * dim;
  for (int o = threadIdx.x; o < Q * Q * dim; o += blockDim.x) {
    const int delta = o % dim, row = (o / dim) % Q, col = o / (dim * Q);
    const int jr = row / bs, jc = col / bs;
    double v = 0.0;
    if (jr == p || jc == p) {
      // F(delta; colp, other)
      auto F = [&](int colp, int other) {
        const double* po = Pc + (other / bs) * dim;
        const KParts kp = kernel_parts(spec, weighted_sqdist(spec, pp, po));
        const double lead = grad_cov_entry(spec, kp, pp, po, row_type(colp % bs, dPs), row_type(other % bs, dPs), delta);
        return lead - Ec[(static_cast<size_t>(colp) * Q + other) * dim + delta];
      };
      if (jr == p && jc == p) {
        v = F(col, row) + F(row, col);
      } else if (jc == p) {
        v = F(col, row);
      } else {
        v = F(row, col);
      }
    }
    out[o] = v;
  }
}

// --------------------------------------------------------------------------------------------------------------
// Smith's forward differentiation of the Cholesky factorisation, in place on a copy of grad-variance.
// On exit G(m, k, j) (stored at [j*Q*dim + k*dim + m], j >= k) = d L_{jk} / d P_p,m.   grid (nc, nd)
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) post_smith_kernel(int Q, int dim, int nd, const double* __restrict__ chol,
                                                         const double* __restrict__ gvar, double* __restrict__ gchol,
                                                         const int* __restrict__ fail) {
  const int c = blockIdx.x, p = blockIdx.y;
  if (fail[c] != 0) return;
  const double* Lc = chol + static_cast<size_t>(c) * Q * Q;
  const size_t off = (static_cast<size_t>(c) * nd + p) * Q * Q * dim;
  const double* gv = gvar + off;
  double* G = gchol + off;
  const int tid = threadIdx.x, nt = blockDim.x;
#define L_(i, j) Lc[(j) * Q + (i)]
#define G_(m, i, j) G[(static_cast<size_t>(j) * Q + (i)) * dim + (m)]
  // copy, zeroing the lower block triangle (row slot > col slot), gpp_math.cpp:1402-1411
  for (int o = tid; o < Q * Q * dim; o += nt) {
    const int rowslot = (o / dim) % Q, colslot = o / (dim * Q);
    G[o] = (rowslot > colslot) ? 0.0 : gv[o];
  }
  __syncthreads();
  for (int k = 0; k < Q; ++k) {
    const double lkk = L_(k, k);
    if (lkk > kMinimumStdDev) {
      for (int m = tid; m < dim; m += nt) G_(m, k, k) = 0.5 * G_(m, k, k) / lkk;
      __syncthreads();
      for (int e = tid; e < (Q - k - 1) * dim; e += nt) {
        const int j = k + 1 + e / dim, m = e % dim;
        G_(m, k, j) = (G_(m, k, j) - L_(j, k) * G_(m, k, k)) / lkk;
      }
      __syncthreads();
      const int w = Q - k - 1;
      for (int e = tid; e < w * w * dim; e += nt) {
        const int m = e % dim, jj = (e / dim) % w, ii = e / (dim * w);
        const int j = k + 1 + jj, i = k + 1 + ii;
        if (i >= j) G_(m, j, i) = G_(m, j, i) - G_(m, k, i) * L_(j, k) - L_(i, k) * G_(m, k, j);
      }
      __syncthreads();
    }
  }
#undef L_
#undef G_
}

}  // namespace

void PosteriorBatch::configure(const cmoe_gp& gp, int nc_in, int num_in, const int* dPs_host, int gs_in, int nd_in,
                               cudaStream_t s) {
  nc = nc_in;
  num = num_in;
  gs = gs_in;
  nd = nd_in;
  Q = num * (1 + gs);
  n = gp.n;
  dim = gp.spec.dim;
  CMOE_REQUIRE(Q >= 1 && Q <= kMaxQ, CMOE_ERR_BOUNDS, "(q+p)*(1+num_derivatives) must be in [1, 96]");
  P.ensure(static_cast<size_t>(nc) * num * dim);
  dPs.ensure(gs > 0 ? gs : 1);
  if (gs > 0) dPs.upload(dPs_host, gs, s);
  Ks.ensure(static_cast<size_t>(n) * nc * Q);
  B.ensure(static_cast<size_t>(n) * nc * Q);
  mu.ensure(static_cast<size_t>(nc) * Q);
  var.ensure(static_cast<size_t>(nc) * Q * Q);
  chol.ensure(static_cast<size_t>(nc) * Q * Q);
  fail.ensure(nc);
  if (nd > 0) {
    const size_t bs = 1 + gs;
    gmu.ensure(static_cast<size_t>(nc) * nd * bs * dim);
    E.ensure(static_cast<size_t>(nc) * nd * bs * Q * dim);
    gvar.ensure(static_cast<size_t>(nc) * nd * Q * Q * dim);
    gchol.ensure(static_cast<size_t>(nc) * nd * Q * Q * dim);
  }
}

void PosteriorBatch::run(const cmoe_gp& gp, int diag_mode, bool want_chol, bool want_grad_chol, cudaStream_t s) {
  const KernelSpec& spec = gp.spec;
  // K* for all sets at once, then K^-1 K* with two blocked triangular sweeps over n x (nc*Q)
  build_mix_covariance(spec, gp.dX.p, gp.N, P.p, nc * num, dPs.p, gs, Ks.p, s);
  const size_t cnt = static_cast<size_t>(n) * nc * Q;
  CMOE_CUDA(cudaMemcpyAsync(B.p, Ks.p, cnt * sizeof(double), cudaMemcpyDeviceToDevice, s));
  potrs_lower(gp.dK.p, n, B.p, n, nc * Q, s);
  const size_t smem = (static_cast<size_t>(Q) * (Q + 1) + static_cast<size_t>(num) * dim) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(post_var_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
  post_var_kernel<<<nc, 256, smem, s>>>(spec, n, gp.mean, gp.dKinvY.p, gp.dnoise.p, P.p, num, dPs.p, gs, Ks.p, B.p,
                                        diag_mode, mu.p, var.p, want_chol ? chol.p : nullptr, fail.p);
  count_launch();
  if (nd > 0) {
    const int bs = 1 + gs;
    const size_t smemE = (static_cast<size_t>(dim) + static_cast<size_t>(kChunk) * dim) * sizeof(double) +
                         kChunk * sizeof(KParts);
    CMOE_CUDA(cudaFuncSetAttribute(post_gradE_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    post_gradE_kernel<<<dim3(nc, nd * bs), kChunk, smemE, s>>>(spec, gp.N, gp.dX.p, gp.dKinvY.p, P.p, num, dPs.p, gs,
                                                              nd, B.p, E.p, gmu.p);
    post_gradvar_kernel<<<dim3(nc, nd), 256, 0, s>>>(spec, P.p, num, dPs.p, gs, nd, E.p, gvar.p);
    count_launch(2);
    if (want_grad_chol) {
      post_smith_kernel<<<dim3(nc, nd), 128, 0, s>>>(Q, dim, nd, chol.p, gvar.p, gchol.p, fail.p);
      count_launch();
    }
  }
  CMOE_CUDA(cudaGetLastError());
}

void posterior_mean_points(const cmoe_gp& gp, const double* P, size_t npts, const int* dPs, int gs, double* mu,
                           double* gmu, cudaStream_t s) {
  if (npts == 0) return;
  post_mean_only_kernel<<<static_cast<unsigned>(npts), kMeanThreads, 0, s>>>(gp.spec, gp.N, gp.mean, gp.dX.p,
                                                                             gp.dKinvY.p, P, dPs, gs, mu, gmu);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

int PosteriorBatch::first_failure(cudaStream_t s, int* which_set) {
  std::vector<int> h(nc);
  fail.download(h.data(), nc, s);
  CMOE_CUDA(cudaStreamSynchronize(s));
  for (int c = 0; c < nc; ++c)
    if (h[c] != 0) {
      if (which_set) *which_set = c;
      return h[c];
    }
  return 0;
}

}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_gp_posterior(const cmoe_gp* gp, const double* sets, int num_sets, int num_pts, const int* derivs_s,
                                 int g_s, double* mean, double* grad_mean, double* var, double* chol_var,
                                 double* grad_var, double* grad_chol, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_sets >= 1 && num_pts >= 1, CMOE_ERR_BOUNDS, "num_sets and num_pts must be >= 1");
    CMOE_REQUIRE(g_s >= 0 && g_s <= gp->spec.dim, CMOE_ERR_BOUNDS, "g_s out of range");
    for (int k = 0; k < g_s; ++k)
      CMOE_REQUIRE(derivs_s[k] >= 0 && derivs_s[k] < gp->spec.dim, CMOE_ERR_BOUNDS, "derivative index out of range");
    require_device(gp->device);
    cudaStream_t s = gp->stream;
    const bool need_grad = grad_mean || grad_var || grad_chol;
    const bool need_chol = chol_var || grad_chol;
    if (!var && !chol_var && !grad_var && !grad_chol) {
      // mean / grad mean only: every point is independent — any number of points, no K^-1 K*
      const size_t npts = static_cast<size_t>(num_sets) * num_pts, bs = 1 + g_s, dim = gp->spec.dim;
      DevBuf<double> dP(npts * dim), dmu(npts * bs), dgmu(grad_mean ? npts * bs * dim : 0);
      DevBuf<int> dd(g_s > 0 ? g_s : 1);
      dP.upload(sets, npts * dim, s);
      if (g_s > 0) dd.upload(derivs_s, g_s, s);
      posterior_mean_points(*gp, dP.p, npts, dd.p, g_s, dmu.p, grad_mean ? dgmu.p : nullptr, s);
      if (mean) dmu.download(mean, npts * bs, s);
      if (grad_mean) dgmu.download(grad_mean, npts * bs * dim, s);
      CMOE_CUDA(cudaStreamSynchronize(s));
      return;
    }
    PosteriorBatch pb;
    pb.configure(*gp, num_sets, num_pts, derivs_s, g_s, need_grad ? num_pts : 0, s);
    pb.P.upload(sets, static_cast<size_t>(num_sets) * num_pts * gp->spec.dim, s);
    pb.run(*gp, 0, need_chol, grad_chol != nullptr, s);
    const size_t Q = pb.Q, dim = gp->spec.dim, ns = num_sets;
    if (need_chol) {
      const int f = pb.first_failure(s, nullptr);
      if (f != 0)
        throw Error(CMOE_ERR_SINGULAR,
                    "GP-Variance matrix singular. Check for duplicate points_to_sample or points_to_sample duplicating "
                    "points_sampled with 0 noise.",
                    f);
    }
    if (mean) pb.mu.download(mean, ns * Q, s);
    if (var) pb.var.download(var, ns * Q * Q, s);
    if (chol_var) pb.chol.download(chol_var, ns * Q * Q, s);
    if (grad_mean) pb.gmu.download(grad_mean, ns * Q * dim, s);
    if (grad_var) pb.gvar.download(grad_var, ns * num_pts * Q * Q * dim, s);
    if (grad_chol) pb.gchol.download(grad_chol, ns * num_pts * Q * Q * dim, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
  });
}

// q-KG value and envelope-theorem gradient for unions of up to CMOE_MAX_KG_LARGE_ROWS rows (DESIGN.md K17).
//
// The estimator and the draws of cmoe_kg_eval (kg.cu) without its 32-row bound: the fantasised posterior of sample s is
// a GP mean over the N training points followed by the U union points, with their derivative rows,
//     mu+_s(x) = m + sum_r w_s,r k(x, row_r),   w_s = [beta - B c_s ; c_s],   c_s = L_U^-T z_s,  B = K^-1 K*,
// so the union's weights are a per-sample column, not registers, and Q only sizes dense products.  Per chunk of
// candidates (union = candidate's q points + the p pending points, U = q + p points, Q = U (1 + g) rows):
//   posterior     the K8 stages (posterior_cov_large) with the noise by observation type on the diagonal, the batched
//                 Cholesky L_U, and B = L^-T V
//   discrete set  Cov_n(Xu rows, A) for A = [union ; discrete points], W = L_U^-1 Cov_n, mu_n(A); the scan mu_A + W^T Z
//                 is a DMMA product, each sample's start is its first strict arg-min
//   weights       C = L_U^-T Z (blocked solve), beta 1^T - B C (DMMA) and C, in the ~ convention of the general path
//   inner optim.  kg_mc_large_kernel: kg_mc_body's general path reading the precomputed weight columns
//   value         kg_value_kernel
//   gradient      R = sum_s k(rows, x*_s) c_s^T (DMMA over the samples), T' = R_U - B^T R_X, K^-1 R_X, G1 (kg.cu's
//                 kernels, generic in Q); the dependence through L_U goes through the Cholesky adjoint of K16 with
//                 Lbar = tril(T' L_U^-T) / num_mc, and kgl_grad_kernel contracts 2 Sigmabar and B 2 Sigmabar with dK.
// The normals Z [num_mc][Q] are written once per call: every candidate uses the same draws.  Every stage treats the
// candidates of a chunk independently and reduces in a fixed order, so a candidate's result does not depend on the
// batch or the chunking.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <memory>

#include "kg_mc.cuh"

namespace cmoe {

namespace {

__device__ __forceinline__ int rtype(int local, const int* derivs) { return local ? derivs[local - 1] : -1; }

// ~ convention of the weight columns: derivative rows divided by l_t (t = derivs[m - 1])
__device__ __forceinline__ double row_scale(const KernelSpec& spec, int m) {
  return m ? spec.inv_len[spec.derivs[m - 1]] : 1.0;
}

// Z [num_mc][Q]: sample s draws pair s >> 1 (Philox call k gives normals 2k, 2k + 1, or row s >> 1 of the table); odd
// samples are the antithetic negation (kg_prep_kernel's draws)
__global__ void __launch_bounds__(256) kgl_normals_kernel(int Q, int num_mc, uint64_t seed,
                                                          const double* __restrict__ table, double* __restrict__ Z) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<size_t>(Q) * num_mc) return;
  const int s = static_cast<int>(e / Q), a = static_cast<int>(e % Q), pair = s >> 1;
  const double sign = (s & 1) ? -1.0 : 1.0;
  double z;
  if (table != nullptr) {
    z = table[static_cast<size_t>(pair) * Q + a];
  } else {
    double n0, n1;
    philox_normal_pair(seed, static_cast<uint64_t>(pair), a >> 1, n0, n1);
    z = (a & 1) ? n1 : n0;
  }
  Z[e] = sign * z;
}

// One CTA per candidate: the union P [U][dim] (raw), the MC kernel's point operands for the N training then U union
// points (Xt [N+U][DIMP] scaled and centred, Pk [N+U][2] = (e_j, 0), as kg_pack_kernel forms them) and the discretisation
// set's union part (Afull [U][dim] raw, fidelity coordinates pinned to 1) and all of A [M][DIMP] (centred).  `stale`
// (q points or NULL): the reference drivers' discretisation set keeps the q points its state was built with
// (kg_pack_kernel); they stand in for the candidate's in A's union part only, the fantasy union is always the current one.
__global__ void __launch_bounds__(256) kgl_pack_kernel(const __grid_constant__ KernelSpec spec,
                                                       const __grid_constant__ Centre ctr, int N, int U, int q, int ps,
                                                       int num_pts, int DIMP, const double* __restrict__ X,
                                                       const double* __restrict__ cand, const double* __restrict__ Xp,
                                                       const double* __restrict__ D,
                                                       const double* __restrict__ stale, double* __restrict__ P,
                                                       double* __restrict__ Xt, double* __restrict__ Pk,
                                                       double* __restrict__ Afull, double* __restrict__ A) {
  const int c = blockIdx.x, tid = threadIdx.x, dim = spec.dim, Np = N + U, M = U + num_pts;
  const bool se = spec.kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL;
  const double lna = log(spec.alpha);
  auto union_pt = [&](int u) {
    return u < q ? cand + (static_cast<size_t>(c) * q + u) * dim : Xp + static_cast<size_t>(u - q) * dim;
  };
  for (int e = tid; e < U * dim; e += blockDim.x) P[static_cast<size_t>(c) * U * dim + e] = union_pt(e / dim)[e % dim];
  double* xt = Xt + static_cast<size_t>(c) * Np * DIMP;
  double* pk = Pk + static_cast<size_t>(c) * Np * 2;
  for (int j = tid; j < Np; j += blockDim.x) {
    const double* pt = j < N ? X + static_cast<size_t>(j) * dim : union_pt(j - N);
    double nrm = 0.0;
    for (int d = 0; d < DIMP; ++d) {
      const double v = (d < dim) ? (pt[d] - ctr.c[d]) * spec.inv_len[d] : 0.0;
      xt[static_cast<size_t>(j) * DIMP + d] = v;
      nrm = fma(v, v, nrm);
    }
    pk[2 * j] = se ? (lna - 0.5 * nrm) : nrm;
    pk[2 * j + 1] = 0.0;
  }
  double* Ac = A + static_cast<size_t>(c) * M * DIMP;
  double* Af = Afull + static_cast<size_t>(c) * U * dim;
  for (int e = tid; e < M * DIMP; e += blockDim.x) {
    const int j = e / DIMP, d = e % DIMP;
    double v = 0.0;
    if (d < ps) {
      v = (j < U) ? ((stale != nullptr && j < q) ? stale[j * dim + d] : union_pt(j)[d])
                  : D[static_cast<size_t>(j - U) * dim + d];
    } else if (d < dim) {
      v = 1.0;
    }
    Ac[e] = (d < dim) ? v - ctr.c[d] : 0.0;
    if (j < U && d < dim) Af[j * dim + d] = v;
  }
}

// Var + noise[type] on the diagonal (pb.run's diag_mode 2)
__global__ void kgl_noise_kernel(int nb, int Q, int bs, const double* __restrict__ noise, double* __restrict__ A) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<size_t>(nb) * Q) return;
  const size_t c = e / Q;
  const int a = static_cast<int>(e % Q);
  A[c * Q * Q + static_cast<size_t>(a) * Q + a] += noise[a % bs];
}

// best_posterior = min(best_so_far, min_j mu_j) over the union's value rows, first strict minimiser (kg_discrete_kernel)
__global__ void kgl_best_kernel(int nb, int U, int bs, double best_so_far, const double* __restrict__ mu,
                                double* __restrict__ best_post, int* __restrict__ winner) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nb) return;
  double bp = best_so_far;
  int w = -1;
  for (int j = 0; j < U; ++j) {
    const double m = mu[static_cast<size_t>(c) * U * bs + j * bs];
    if (m < bp) {
      bp = m;
      w = j;
    }
  }
  best_post[c] = bp;
  winner[c] = w;
}

// Cov_n(Xu row a, A_j) = k(Xu row a, A_j) - (B^T K(X, A))_aj  ->  Wd [c][j][a] (column j of length Q, for the solve),
// in place: Wd holds the DMMA product B^T K(X, A) on entry.  The a = -1 slice of the threads forms mu_n(A_j).
// KAu = K(X rows, A union part) [n][nb U], KD = K(X rows, D).
__global__ void __launch_bounds__(256) kgl_disc_cov_kernel(const __grid_constant__ KernelSpec spec, int n, int U,
                                                           int num_pts, double mean, const double* __restrict__ beta,
                                                           const double* __restrict__ P,
                                                           const double* __restrict__ Afull,
                                                           const double* __restrict__ D,
                                                           const double* __restrict__ KAu,
                                                           const double* __restrict__ KD, double* __restrict__ Wd,
                                                           double* __restrict__ muA) {
  const int c = blockIdx.y, dim = spec.dim, bs = 1 + spec.g, Q = U * bs, M = U + num_pts;
  const size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (o >= static_cast<size_t>(M) * (Q + 1)) return;
  const int j = static_cast<int>(o / (Q + 1)), a = static_cast<int>(o % (Q + 1)) - 1;
  const double* kcol = (j < U) ? (KAu + (static_cast<size_t>(c) * U + j) * n) : (KD + static_cast<size_t>(j - U) * n);
  if (a < 0) {
    double m = 0.0;
    for (int r = 0; r < n; ++r) m += kcol[r] * beta[r];
    muA[static_cast<size_t>(c) * M + j] = m + mean;
    return;
  }
  const double* aj = (j < U) ? (Afull + (static_cast<size_t>(c) * U + j) * dim) : (D + static_cast<size_t>(j - U) * dim);
  const double* pa = P + (static_cast<size_t>(c) * U + a / bs) * dim;
  const KParts kp = kernel_parts(spec, weighted_sqdist(spec, pa, aj));
  double* w = Wd + (static_cast<size_t>(c) * M + j) * Q + a;
  *w = cov_entry(spec, kp, pa, aj, rtype(a % bs, spec.derivs), -1) - *w;
}

// out = in^T for nb column-major rows x cols matrices (out: cols x rows)
__global__ void __launch_bounds__(256) kgl_transpose_kernel(int rows, int cols, const double* __restrict__ in,
                                                            double* __restrict__ out) {
  const size_t off = static_cast<size_t>(blockIdx.y) * rows * cols;
  const size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (o >= static_cast<size_t>(rows) * cols) return;
  const size_t r = o % cols, cc = o / cols;  // out (r, cc) = in (cc, r)
  out[off + o] = in[off + r * rows + cc];
}

// each sample's start: first strict arg-min over j of mu_A[j] + S[s][j], S = W^T Z [num_mc][M]
__global__ void __launch_bounds__(256) kgl_argmin_kernel(int M, int num_mc, const double* __restrict__ muA,
                                                         const double* __restrict__ S, int* __restrict__ start) {
  const int c = blockIdx.y, s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= num_mc) return;
  const double* mc_ = muA + static_cast<size_t>(c) * M;
  const double* sv = S + (static_cast<size_t>(c) * num_mc + s) * M;
  int arg = 0;
  double best = 0.0;
  for (int j = 0; j < M; ++j) {
    const double v = mc_[j] + sv[j];
    if (j == 0 || best > v) {
      best = v;
      arg = j;
    }
  }
  start[static_cast<size_t>(c) * num_mc + s] = arg;
}

// weight columns [num_mc][R], R = n + Q:  rows r < n hold B C (gemm_nn) on entry -> (beta_r - (B C)_r) ~;  rows n + a
// <- c_a ~
__global__ void __launch_bounds__(256) kgl_weights_kernel(const __grid_constant__ KernelSpec spec, int n, int Q,
                                                          int num_mc, const double* __restrict__ beta,
                                                          const double* __restrict__ C, double* __restrict__ Wts) {
  const int c = blockIdx.y, bs = 1 + spec.g, R = n + Q;
  const size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (o >= static_cast<size_t>(R) * num_mc) return;
  const int s = static_cast<int>(o / R), r = static_cast<int>(o % R);
  double* w = Wts + static_cast<size_t>(c) * num_mc * R + o;
  if (r < n) {
    *w = (beta[r] - *w) * row_scale(spec, r % bs);
  } else {
    const int a = r - n;
    *w = C[(static_cast<size_t>(c) * num_mc + s) * Q + a] * row_scale(spec, a % bs);
  }
}

// Kx [num_mc][R]: k(row r, x*_s) for the training rows then the union rows (x*_s back in raw coordinates)
__global__ void __launch_bounds__(256) kgl_kx_kernel(const __grid_constant__ KernelSpec spec,
                                                     const __grid_constant__ Centre ctr, int N, int U, int num_mc,
                                                     int DIMP, const double* __restrict__ X,
                                                     const double* __restrict__ P, const double* __restrict__ outX,
                                                     double* __restrict__ Kx) {
  const int c = blockIdx.y, dim = spec.dim, bs = 1 + spec.g, R = (N + U) * bs;
  const size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (o >= static_cast<size_t>(R) * num_mc) return;
  const int s = static_cast<int>(o / R), r = static_cast<int>(o % R), j = r / bs, m = r % bs;
  const double* xs = outX + (static_cast<size_t>(c) * num_mc + s) * DIMP;
  double x[CMOE_MAX_DIM];
  for (int d = 0; d < dim; ++d) x[d] = fma(xs[d], 1.0 / spec.inv_len[d], ctr.c[d]);
  const double* pt = j < N ? X + static_cast<size_t>(j) * dim : P + (static_cast<size_t>(c) * U + j - N) * dim;
  const KParts kp = kernel_parts(spec, weighted_sqdist(spec, pt, x));
  Kx[static_cast<size_t>(c) * num_mc * R + o] = cov_entry(spec, kp, pt, x, rtype(m, spec.derivs), -1);
}

// Lbar (column-major, lower) = tril(T' L^-T) / num_mc from X = L^-1 T'^T (column-major), i.e. Lbar(j, i) = X(i, j)
__global__ void __launch_bounds__(256) kgl_lbar_kernel(int Q, int num_mc, const double* __restrict__ Xs,
                                                       double* __restrict__ Lbar) {
  const size_t off = static_cast<size_t>(blockIdx.y) * Q * Q;
  const size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (o >= static_cast<size_t>(Q) * Q) return;
  const int j = static_cast<int>(o % Q), i = static_cast<int>(o / Q);
  Lbar[off + o] = (i <= j) ? Xs[off + static_cast<size_t>(j) * Q + i] / static_cast<double>(num_mc) : 0.0;
}

// Gradient of candidate point p < q, grid (q, candidates).  Threads = (component delta, slice of the N + U points);
// slices are combined in a fixed order.
//   grad = ( -G1 + sum_r dK*(p, r) (K^-1 R)_r ) / num_mc + tr(Sigmabar dSigma_U) + [p == winner] dmu_p
// with T = 2 Sigmabar (column-major Q x Q) and R2 = B T[:, rows of the q points] (n x q (1+g), ld n):
//   tr(Sigmabar dSigma_U) = sum_m [ sum_(b not in p) T(p m, b) dK(p m, b) - sum_r dK(p m, x_r) R2(r, p m) ].
constexpr int kGradThreads = 128;
__global__ void __launch_bounds__(kGradThreads) kgl_grad_kernel(const __grid_constant__ KernelSpec spec, int N, int U,
                                                                int q, int num_mc, const double* __restrict__ X,
                                                                const double* __restrict__ beta,
                                                                const double* __restrict__ P,
                                                                const double* __restrict__ KinvR,
                                                                const double* __restrict__ T,
                                                                const double* __restrict__ R2,
                                                                const double* __restrict__ G1,
                                                                const int* __restrict__ winner,
                                                                double* __restrict__ grad) {
  __shared__ double Pp[CMOE_MAX_DIM];
  __shared__ double red[kGradThreads];
  const int p = blockIdx.x, c = blockIdx.y, dim = spec.dim, bs = 1 + spec.g, n = N * bs, Q = U * bs, R = n + Q;
  const int tid = threadIdx.x;
  const double* Pc = P + static_cast<size_t>(c) * U * dim;
  for (int e = tid; e < dim; e += blockDim.x) Pp[e] = Pc[static_cast<size_t>(p) * dim + e];
  __syncthreads();
  const int nparts = kGradThreads / dim, delta = tid % dim, part = tid / dim;
  const bool win = winner[c] == p;
  const double inv_mc = 1.0 / static_cast<double>(num_mc);
  const double* Kc = KinvR + static_cast<size_t>(c) * Q * R;
  const double* R2c = R2 + static_cast<size_t>(c) * q * bs * n;
  const double* Tc = T + static_cast<size_t>(c) * Q * Q;
  double acc = 0.0;
  if (part < nparts) {
    for (int t = part; t < N + U; t += nparts) {
      if (t < N) {
        const double* xj = X + static_cast<size_t>(t) * dim;
        const KParts kp = kernel_parts(spec, weighted_sqdist(spec, Pp, xj));
        for (int m = 0; m < bs; ++m) {
          const int a = p * bs + m;
          for (int cc = 0; cc < bs; ++cc) {
            const int r = t * bs + cc;
            double coef = Kc[static_cast<size_t>(a) * R + r] * inv_mc - R2c[static_cast<size_t>(a) * n + r];
            if (m == 0 && win) coef += beta[r];
            const double g = grad_cov_entry(spec, kp, Pp, xj, rtype(m, spec.derivs), rtype(cc, spec.derivs), delta);
            acc = fma(g, coef, acc);
          }
        }
      } else if (t - N != p) {
        const int u = t - N;
        const double* pu = Pc + static_cast<size_t>(u) * dim;
        const KParts kp = kernel_parts(spec, weighted_sqdist(spec, Pp, pu));
        for (int m = 0; m < bs; ++m)
          for (int m2 = 0; m2 < bs; ++m2) {
            const double g = grad_cov_entry(spec, kp, Pp, pu, rtype(m, spec.derivs), rtype(m2, spec.derivs), delta);
            acc = fma(g, Tc[static_cast<size_t>(u * bs + m2) * Q + p * bs + m], acc);
          }
      }
    }
  }
  red[tid] = acc;
  __syncthreads();
  if (tid < dim) {
    double t = 0.0;
    for (int pp = 0; pp < nparts; ++pp) t += red[pp * dim + tid];
    t -= G1[(static_cast<size_t>(c) * q + p) * dim + tid] * inv_mc;
    grad[(static_cast<size_t>(c) * q + p) * dim + tid] = t;
  }
}

}  // namespace

// Device workspace of cmoe_kg_eval_large beyond the K8 buffers of SampleWork, kept on the handle (cmoe_gp::kg_large_ws)
// and grown on demand.
struct KgLargeWork {
  DevBuf<double> Z, D, KD, alpha0, Xt, Pk, Afull, A, KAu, Bt, Wd, WdT, muA, S, C, Wts, outVal, outX, outH, best, kg;
  DevBuf<double> aw, stale;
  DevBuf<double> Kx, Ct, Rm, Tp, T1, T2, R2, G1, grad;
  DevBuf<int> start, winner, work;
  DevBuf<unsigned long long> stats;
};

namespace {

KgLargeWork& kg_large_work(const cmoe_gp& gp) {
  if (!gp.kg_large_ws) gp.kg_large_ws = std::make_shared<KgLargeWork>();
  return *static_cast<KgLargeWork*>(gp.kg_large_ws.get());
}

// Argument checks that need no handle (the size bounds of cmoe_kg_eval_large)
// samples of one call: the sample axis of the scan product is grid.y of gemm_nn (64 samples per CTA row, <= 65535)
constexpr long long kMaxKgLargeSamples = 65535LL * 64;
// inner-optimiser scratch (kg_mc_large_kernel's per-lane weight columns), counted in the 2 GiB budget
constexpr size_t kKgLargeScratchBytes = size_t(256) << 20;

void check_sizes(int num_candidates, int q, int p, int num_mc) {
  CMOE_REQUIRE(num_candidates >= 1, CMOE_ERR_BOUNDS, "num_candidates must be >= 1");
  CMOE_REQUIRE(q >= 1 && p >= 0 && num_mc >= 1, CMOE_ERR_BOUNDS, "q >= 1, p >= 0, num_mc >= 1 required");
  CMOE_REQUIRE(static_cast<long long>(q) + p <= CMOE_MAX_KG_LARGE_ROWS, CMOE_ERR_BOUNDS,
               "(q+p)*(1+num_derivatives) must be <= 1024");
  CMOE_REQUIRE(num_mc <= kMaxKgLargeSamples, CMOE_ERR_BOUNDS, "num_mc must be <= 4194240");
}

}  // namespace

void kg_large_eval(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds,
                   const double* discrete_pts, int num_pts, const double* candidates, int num_candidates, int q,
                   const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                   const double* normals_table, const double* stale_union, double* kg, double* grad_kg,
                   cmoe_kg_stats* stats) {
    check_sizes(num_candidates, q, p, num_mc);
    CMOE_REQUIRE(gp != nullptr, CMOE_ERR_INVALID_VALUE, "gp is NULL");
    const KernelSpec& spec = gp->spec;
    const int dim = spec.dim, g = spec.g, bs = 1 + g, U = q + p;
    CMOE_REQUIRE(static_cast<long long>(U) * bs <= CMOE_MAX_KG_LARGE_ROWS, CMOE_ERR_BOUNDS,
                 "(q+p)*(1+num_derivatives) must be <= 1024");
    CMOE_REQUIRE(num_pts >= 0, CMOE_ERR_BOUNDS, "bad sizes");
    CMOE_REQUIRE(num_fidelity >= 0 && num_fidelity < dim, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    CMOE_REQUIRE(g <= kMaxGWide, CMOE_ERR_BOUNDS, "at most 31 derivative observations per point in the q-KG kernel");
    if (g > kMaxG) {
      for (int a = 0; a < g; ++a)
        for (int b = 0; b < a; ++b)
          CMOE_REQUIRE(spec.derivs[a] != spec.derivs[b], CMOE_ERR_BOUNDS,
                       "a partial derivative is observed twice per point (q-KG with more than 8 derivative observations)");
    }
    CMOE_REQUIRE(inner->max_num_steps <= 4096, CMOE_ERR_BOUNDS, "inner max_num_steps must be <= 4096");
    const int ps = dim - num_fidelity;
    for (int d = 0; d < ps; ++d)
      CMOE_REQUIRE(inner_bounds[2 * d] <= inner_bounds[2 * d + 1], CMOE_ERR_BOUNDS, "Tensor product region is EMPTY.");
    const KgLargeEntry* entry = find_kg_large_entry(spec.kernel, dim, g);
    CMOE_REQUIRE(entry != nullptr, CMOE_ERR_BOUNDS, "dim exceeds the largest compiled q-KG kernel (32 dims)");
    const int DIMP = entry->dim, N = gp->N, n = gp->n, Q = U * bs, Np = N + U, R = Np * bs, M = U + num_pts;
    const int qb = q * bs;
    const bool want_grad = grad_kg != nullptr;
    const size_t QQ = static_cast<size_t>(Q) * Q, mc = static_cast<size_t>(num_mc);
    // device workspace of one candidate (doubles; ints counted as doubles)
    const size_t nb64 = static_cast<size_t>((Q + NB - 1) / NB) * NB * NB;
    size_t per = static_cast<size_t>(U) * dim * 2 + static_cast<size_t>(n) * Q + QQ + Q + nb64 + 1 +
                 static_cast<size_t>(Np) * (DIMP + 2) + static_cast<size_t>(M) * (DIMP + 1) +
                 static_cast<size_t>(n) * U + 2 * static_cast<size_t>(Q) * M + mc * (M + Q + R + DIMP + 3) + 4;
    if (want_grad) per += mc * (R + Q) + static_cast<size_t>(R) * Q + 3 * QQ + static_cast<size_t>(n) * qb +
                          2 * static_cast<size_t>(q) * dim;
    per += static_cast<size_t>(n) * Q;  // B^T for the discretisation product
    const size_t per_bytes = per * sizeof(double);
    // per call: the draws Z and the inner optimiser's scratch; the chunks get the rest of the 2 GiB
    const size_t fixed = mc * Q * sizeof(double) + kKgLargeScratchBytes;
    const size_t budget = kSampleWorkspaceBytes > fixed ? kSampleWorkspaceBytes - fixed : 0;
    if (per_bytes > budget) {
      char msg[320];
      snprintf(msg, sizeof(msg),
               "one candidate's q-KG workspace (%zu bytes: Q = %d rows, N + U = %d points, num_mc = %d) does not fit "
               "the %zu bytes left of 2 GiB beside the call's normals and scratch",
               per_bytes, Q, Np, num_mc, budget);
      throw Error(CMOE_ERR_BOUNDS, msg);
    }
    require_device(gp->device);
    cudaStream_t s = gp->stream;
    const Centre ctr = centre_of(*gp);
    const int chunk = static_cast<int>(chunk_items(num_candidates, budget, per_bytes, kMaxChunkSets));
    SampleWork& w = sample_work(*gp);
    KgLargeWork& k = kg_large_work(*gp);
    // per call: the draws, the discrete points (fidelity coordinates 1), K(X, D), the step sizes
    k.Z.ensure(mc * Q);
    DevBuf<double> dtable;
    if (normals_table) dtable.upload(normals_table, ((mc + 1) / 2) * Q, s);
    kgl_normals_kernel<<<static_cast<unsigned>((mc * Q + 255) / 256), 256, 0, s>>>(
        Q, num_mc, seed, normals_table ? dtable.p : nullptr, k.Z.p);
    count_launch();
    std::vector<double> hD(static_cast<size_t>(std::max(1, num_pts)) * dim, 1.0);
    for (int j = 0; j < num_pts; ++j)
      for (int d = 0; d < ps; ++d) hD[static_cast<size_t>(j) * dim + d] = discrete_pts[static_cast<size_t>(j) * ps + d];
    k.D.upload(hD.data(), hD.size(), s);
    k.KD.ensure(static_cast<size_t>(n) * std::max(1, num_pts));
    if (num_pts > 0) build_mix_covariance(spec, gp->dX.p, N, k.D.p, num_pts, nullptr, 0, k.KD.p, s);
    std::vector<double> a0(std::max(1, inner->max_num_steps));
    for (int i = 0; i < inner->max_num_steps; ++i) a0[i] = gd_step_size(inner->pre_mult, inner->gamma, i);
    k.alpha0.upload(a0.data(), a0.size(), s);
    std::vector<int> hderivs(std::max(1, g), 0);
    for (int a = 0; a < g; ++a) hderivs[a] = spec.derivs[a];
    w.dPs.upload(hderivs.data(), hderivs.size(), s);
    DevBuf<double> dcand, dXp;
    dcand.upload(candidates, static_cast<size_t>(num_candidates) * q * dim, s);
    if (p) dXp.upload(points_being_sampled, static_cast<size_t>(p) * dim, s);
    if (stale_union) k.stale.upload(stale_union, static_cast<size_t>(q) * dim, s);
    // chunk workspace
    w.P.ensure(static_cast<size_t>(chunk) * U * dim);
    w.V.ensure(static_cast<size_t>(chunk) * Q * n);
    w.A.ensure(static_cast<size_t>(chunk) * QQ);
    w.mu.ensure(static_cast<size_t>(chunk) * Q);
    w.fail.ensure(chunk);
    k.Xt.ensure(static_cast<size_t>(chunk) * Np * DIMP);
    k.Pk.ensure(static_cast<size_t>(chunk) * Np * 2);
    k.Afull.ensure(static_cast<size_t>(chunk) * U * dim);
    k.A.ensure(static_cast<size_t>(chunk) * M * DIMP);
    k.KAu.ensure(static_cast<size_t>(chunk) * n * U);
    k.Bt.ensure(static_cast<size_t>(chunk) * n * Q);
    k.Wd.ensure(static_cast<size_t>(chunk) * Q * M);
    k.WdT.ensure(static_cast<size_t>(chunk) * Q * M);
    k.muA.ensure(static_cast<size_t>(chunk) * M);
    k.S.ensure(static_cast<size_t>(chunk) * mc * M);
    k.C.ensure(static_cast<size_t>(chunk) * mc * Q);
    k.Wts.ensure(static_cast<size_t>(chunk) * mc * R);
    k.outVal.ensure(static_cast<size_t>(chunk) * mc);
    k.outX.ensure(static_cast<size_t>(chunk) * mc * DIMP);
    k.outH.ensure(static_cast<size_t>(chunk) * mc);
    k.best.ensure(chunk);
    k.kg.ensure(chunk);
    k.start.ensure(static_cast<size_t>(chunk) * mc);
    k.winner.ensure(chunk);
    k.work.ensure(1);
    k.stats.ensure(4);
    if (want_grad) {
      k.Kx.ensure(static_cast<size_t>(chunk) * mc * R);
      k.Ct.ensure(static_cast<size_t>(chunk) * mc * Q);
      k.Rm.ensure(static_cast<size_t>(chunk) * R * Q);
      k.Tp.ensure(static_cast<size_t>(chunk) * QQ);
      k.T1.ensure(static_cast<size_t>(chunk) * QQ);
      k.T2.ensure(static_cast<size_t>(chunk) * QQ);
      k.R2.ensure(static_cast<size_t>(chunk) * n * qb);
      k.G1.ensure(static_cast<size_t>(chunk) * q * dim);
      k.grad.ensure(static_cast<size_t>(chunk) * q * dim);
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    {
      // one scratch column set (R rows x kMcThreads lanes) per resident CTA, at most 3 per SM and
      // kKgLargeScratchBytes in total
      const size_t slot = static_cast<size_t>(R) * kMcThreads;
      const size_t slots = std::max<size_t>(1, std::min<size_t>(3 * static_cast<size_t>(sms),
                                                                kKgLargeScratchBytes / (slot * sizeof(double))));
      k.aw.ensure(slot * slots);
    }
    const int aw_slots = static_cast<int>(k.aw.count / (static_cast<size_t>(R) * kMcThreads));
    CMOE_CUDA(cudaMemsetAsync(k.stats.p, 0, 4 * sizeof(unsigned long long), s));

    KgMcParams m{};
    m.N = Np;
    m.U = 0;
    m.ps = ps;
    m.dim = dim;
    m.M = M;
    m.num_mc = num_mc;
    m.use_smem = 0;
    m.g = g;
    m.Q = 0;
    m.pk_stride = 2;
    for (int a = 0; a < CMOE_MAX_DIM; ++a) {
      m.derivs[a] = (a < g) ? spec.derivs[a] : 0;
      m.drow[a] = 0;
    }
    for (int a = 0; a < g; ++a) m.drow[spec.derivs[a]] = 1 + a;
    m.max_steps = inner->max_num_steps;
    m.max_restarts = inner->max_num_restarts;
    m.mean = gp->mean;
    m.mrc = inner->max_relative_change;
    m.tol = inner->tolerance;
    m.step_tol = inner->max_num_steps > 0 ? inner->tolerance / static_cast<double>(inner->max_num_steps) : 0.0;
    m.alpha = spec.alpha;
    m.alpha0 = k.alpha0.p;
    for (int d = 0; d < CMOE_MAX_DIM; ++d) {
      m.lo[d] = -1.0e300;
      m.hi[d] = 1.0e300;
      m.inv_len[d] = (d < dim) ? spec.inv_len[d] : 0.0;
    }
    for (int d = 0; d < ps; ++d) {  // the frame of A
      m.lo[d] = inner_bounds[2 * d] - gp->centre[d];
      m.hi[d] = inner_bounds[2 * d + 1] - gp->centre[d];
    }
    m.stats = k.stats.p;
    m.aw = k.aw.p;
    m.aw_slots = aw_slots;
    m.work = k.work.p;
    m.stage_ops = 0;

    std::vector<int> hfail(chunk);
    for (int c0 = 0; c0 < num_candidates; c0 += chunk) {
      const int nb = std::min(chunk, num_candidates - c0);
      kgl_pack_kernel<<<nb, 256, 0, s>>>(spec, ctr, N, U, q, ps, num_pts, DIMP, gp->dX.p,
                                         dcand.p + static_cast<size_t>(c0) * q * dim, dXp.p, k.D.p,
                                         stale_union ? k.stale.p : nullptr, w.P.p, k.Xt.p,
                                         k.Pk.p, k.Afull.p, k.A.p);
      count_launch();
      // posterior of the union: V = L^-1 K*, mu, Var + noise[type], L_U, B = L^-T V
      posterior_cov_large(*gp, w, nb, U, g, 0.0, s);
      kgl_noise_kernel<<<static_cast<unsigned>((static_cast<size_t>(nb) * Q + 255) / 256), 256, 0, s>>>(
          nb, Q, bs, gp->dnoise.p, w.A.p);
      count_launch();
      CMOE_CUDA(cudaMemsetAsync(w.fail.p, 0, nb * sizeof(int), s));
      potrf_batched(w.A.p, Q, nb, w.fail.p, w.stage, s);
      w.fail.download(hfail.data(), nb, s);
      CMOE_CUDA(cudaStreamSynchronize(s));
      for (int c = 0; c < nb; ++c)
        if (hfail[c] != 0)
          throw Error(CMOE_ERR_SINGULAR,
                      "GP-Variance matrix singular. Check for duplicate points_to_sample/being_sampled or "
                      "points_to_sample/being_sampled duplicating points_sampled with 0 noise.",
                      hfail[c]);
      zero_upper(nb, Q, w.A.p, s);
      trsm_lower_blocked(gp->dK.p, n, w.V.p, n, nb * Q, true, s);
      kgl_best_kernel<<<(nb + 127) / 128, 128, 0, s>>>(nb, U, bs, best_so_far, w.mu.p, k.best.p, k.winner.p);
      count_launch();
      // discretisation set: W = L_U^-1 Cov_n(Xu rows, A), mu_n(A); starts = first strict arg-min of mu_A + W^T z
      build_mix_covariance(spec, gp->dX.p, N, k.Afull.p, nb * U, nullptr, 0, k.KAu.p, s);
      // B^T K(X, A) on DMMA: B^T [Q][n] per candidate, then the union part and the shared discrete part of A
      kgl_transpose_kernel<<<dim3(static_cast<unsigned>((static_cast<size_t>(n) * Q + 255) / 256), nb), 256, 0, s>>>(
          n, Q, w.V.p, k.Bt.p);
      count_launch();
      gemm_nn(Q, U, n, k.Bt.p, Q, static_cast<size_t>(Q) * n, k.KAu.p, n, static_cast<size_t>(n) * U, k.Wd.p, Q,
              static_cast<size_t>(Q) * M, nb, s);
      if (num_pts > 0)
        gemm_nn(Q, num_pts, n, k.Bt.p, Q, static_cast<size_t>(Q) * n, k.KD.p, n, 0, k.Wd.p + static_cast<size_t>(U) * Q,
                Q, static_cast<size_t>(Q) * M, nb, s);
      const size_t nwd = static_cast<size_t>(M) * (Q + 1);
      kgl_disc_cov_kernel<<<dim3(static_cast<unsigned>((nwd + 255) / 256), nb), 256, 0, s>>>(
          spec, n, U, num_pts, gp->mean, gp->dKinvY.p, w.P.p, k.Afull.p, k.D.p, k.KAu.p, k.KD.p, k.Wd.p, k.muA.p);
      count_launch();
      for (int c = 0; c < nb; ++c)
        trsm_lower_blocked(w.A.p + c * QQ, Q, k.Wd.p + static_cast<size_t>(c) * Q * M, Q, M, false, s);
      kgl_transpose_kernel<<<dim3(static_cast<unsigned>((static_cast<size_t>(Q) * M + 255) / 256), nb), 256, 0, s>>>(
          Q, M, k.Wd.p, k.WdT.p);
      count_launch();
      gemm_nn(M, num_mc, Q, k.WdT.p, M, static_cast<size_t>(M) * Q, k.Z.p, Q, 0, k.S.p, M, mc * M, nb, s);
      kgl_argmin_kernel<<<dim3((num_mc + 255) / 256, nb), 256, 0, s>>>(M, num_mc, k.muA.p, k.S.p, k.start.p);
      count_launch();
      // C = L_U^-T Z and the weight columns
      for (int c = 0; c < nb; ++c) {
        double* Cc = k.C.p + static_cast<size_t>(c) * mc * Q;
        CMOE_CUDA(cudaMemcpyAsync(Cc, k.Z.p, mc * Q * sizeof(double), cudaMemcpyDeviceToDevice, s));
        trsm_lower_blocked(w.A.p + c * QQ, Q, Cc, Q, num_mc, true, s);
      }
      gemm_nn(n, num_mc, Q, w.V.p, n, static_cast<size_t>(n) * Q, k.C.p, Q, mc * Q, k.Wts.p, R, mc * R, nb, s);
      kgl_weights_kernel<<<dim3(static_cast<unsigned>((mc * R + 255) / 256), nb), 256, 0, s>>>(spec, n, Q, num_mc,
                                                                                            gp->dKinvY.p, k.C.p,
                                                                                            k.Wts.p);
      count_launch();
      // inner optimisation of every sample
      KgMcParams prm = m;
      {
        // samples per work item: aim for >= ~8 waves of 3 CTAs per SM over the chunk, 2 to 16 samples per lane
        const long long target = 8LL * sms * 3;
        long long sc = (static_cast<long long>(nb) * num_mc + target - 1) / target;
        sc = std::max<long long>(2 * kMcThreads, std::min<long long>(sc, 16 * kMcThreads));
        sc = (sc + kMcThreads - 1) / kMcThreads * kMcThreads;
        prm.chunk = static_cast<int>(std::min<long long>(sc, (num_mc + kMcThreads - 1) / kMcThreads * kMcThreads));
      }
      prm.chunks = (num_mc + prm.chunk - 1) / prm.chunk;
      prm.work_total = prm.chunks * nb;
      prm.Xt = k.Xt.p;
      prm.Pk = k.Pk.p;
      prm.A = k.A.p;
      prm.recC = k.C.p;  // not read by the large-union build
      prm.recStart = k.start.p;
      prm.Wt = k.Wts.p;
      prm.outVal = k.outVal.p;
      prm.outX = k.outX.p;
      prm.outH = k.outH.p;
      CMOE_CUDA(cudaMemsetAsync(k.work.p, 0, sizeof(int), s));
      entry->mc(prm, s);
      count_launch();
      CMOE_CUDA(cudaGetLastError());
      if (inner->max_num_restarts <= 0) kg_fill_points(spec, ctr, nb * num_mc, DIMP, k.outX.p, k.outH.p, s);
      kg_value(nb, num_mc, k.outVal.p, k.best.p, w.fail.p, k.kg.p, s);
      k.kg.download(kg + c0, nb, s);
      if (want_grad) {
        // R = Kx C^T over the samples, [Q][R] (column a of length R = n + Q)
        kgl_kx_kernel<<<dim3(static_cast<unsigned>((mc * R + 255) / 256), nb), 256, 0, s>>>(
            spec, ctr, N, U, num_mc, DIMP, gp->dX.p, w.P.p, k.outX.p, k.Kx.p);
        kgl_transpose_kernel<<<dim3(static_cast<unsigned>((mc * Q + 255) / 256), nb), 256, 0, s>>>(Q, num_mc, k.C.p,
                                                                                                 k.Ct.p);
        count_launch(2);
        gemm_nn(R, Q, num_mc, k.Kx.p, R, mc * R, k.Ct.p, num_mc, mc * Q, k.Rm.p, R, static_cast<size_t>(R) * Q, nb, s);
        kg_tprime(nb, n, Q, Q, k.Rm.p, w.V.p, k.Tp.p, s);
        potrs_lower(gp->dK.p, n, k.Rm.p, R, nb * Q, s);
        kg_g1(spec, ctr, nb, U, q, Q, DIMP, num_mc, w.P.p, k.C.p, k.outX.p, k.G1.p, s);
        // Lbar = tril(T' L_U^-T) / num_mc, then 2 Sigmabar through the Cholesky adjoint, and R2 = B 2 Sigmabar
        for (int c = 0; c < nb; ++c) trsm_lower_blocked(w.A.p + c * QQ, Q, k.Tp.p + c * QQ, Q, Q, false, s);
        kgl_lbar_kernel<<<dim3(static_cast<unsigned>((QQ + 255) / 256), nb), 256, 0, s>>>(Q, num_mc, k.Tp.p, k.T1.p);
        count_launch();
        cholesky_adjoint(w.A.p, Q, nb, k.T1.p, k.T2.p, s);
        gemm_nn(n, qb, Q, w.V.p, n, static_cast<size_t>(n) * Q, k.T1.p, Q, QQ, k.R2.p, n, static_cast<size_t>(n) * qb,
                nb, s);
        kgl_grad_kernel<<<dim3(q, nb), kGradThreads, 0, s>>>(spec, N, U, q, num_mc, gp->dX.p, gp->dKinvY.p, w.P.p,
                                                            k.Rm.p, k.T1.p, k.R2.p, k.G1.p, k.winner.p, k.grad.p);
        count_launch();
        CMOE_CUDA(cudaGetLastError());
        k.grad.download(grad_kg + static_cast<size_t>(c0) * q * dim, static_cast<size_t>(nb) * q * dim, s);
      }
      CMOE_CUDA(cudaStreamSynchronize(s));
    }
    unsigned long long st[4] = {0, 0, 0, 0};
    CMOE_CUDA(cudaMemcpyAsync(st, k.stats.p, sizeof(st), cudaMemcpyDeviceToHost, s));
    CMOE_CUDA(cudaStreamSynchronize(s));
    if (stats) {
      stats->mc_samples = static_cast<uint64_t>(num_candidates) * num_mc;
      stats->posterior_evals = st[0];
      stats->line_search_steps = st[1];
      stats->point_evals = st[2];
      stats->line_batches = st[3];
    }
}

}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_kg_eval_large(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner,
                                  const double* inner_bounds, const double* discrete_pts, int num_pts,
                                  const double* candidates, int num_candidates, int q,
                                  const double* points_being_sampled, int p, int num_mc, double best_so_far,
                                  uint64_t seed, const double* normals_table, double* kg, double* grad_kg,
                                  cmoe_kg_stats* stats, int* info) {
  return guarded(info, [&] {
    kg_large_eval(gp, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, candidates, num_candidates, q,
                  points_being_sampled, p, num_mc, best_so_far, seed, normals_table, nullptr, kg, grad_kg, stats);
  });
}

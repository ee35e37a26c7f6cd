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

namespace {

// samples of one call: the sample axis of the scan product is grid.y of gemm_nn (64 samples per CTA row, <= 65535)
constexpr long long kMaxKgLargeSamples = 65535LL * 64;

// the size bounds of cmoe_kg_eval_large, which need no handle
void kg_large_check_sizes(int num_candidates, int q, int p, int num_mc) {
  CMOE_REQUIRE(num_candidates >= 1, CMOE_ERR_BOUNDS, "num_candidates must be >= 1");
  CMOE_REQUIRE(q >= 1 && p >= 0 && num_mc >= 1, CMOE_ERR_BOUNDS, "q >= 1, p >= 0, num_mc >= 1 required");
  CMOE_REQUIRE(static_cast<long long>(q) + p <= CMOE_MAX_KG_LARGE_ROWS, CMOE_ERR_BOUNDS,
               "(q+p)*(1+num_derivatives) must be <= 1024");
  CMOE_REQUIRE(num_mc <= kMaxKgLargeSamples, CMOE_ERR_BOUNDS, "num_mc must be <= 4194240");
}

// Shape and sizes of one GP's evaluation (kg_large_shape)
struct KgLargeShape {
  const KgLargeEntry* entry = nullptr;
  int nf, ps, q, p, U, dim, g, bs, num_pts, num_mc, DIMP, N, n, Q, Np, R, M, qb;
  bool want_grad;
  size_t per_bytes;  // one candidate's chunk workspace
  size_t z_bytes;    // the draws Z
  size_t budget;     // what one GP's chunks may use: 2 GiB less the draws, the inner optimiser's scratch and kCarveSlack
};

// Device inputs of one evaluation, shared by every GP that evaluates it
struct KgLargeInputs {
  const double *Z, *alpha0, *cand, *Xp, *stale;
};

// inner-optimiser scratch (kg_mc_large_kernel's per-lane weight columns), counted in the 2 GiB budget
constexpr size_t kKgLargeScratchBytes = size_t(256) << 20;

// candidates with a singular union factor get the identity instead, so every later stage of the chunk works on finite
// numbers; their value is NaN (kg_value) and the evaluation reports the failure
__global__ void __launch_bounds__(256) kgl_sanitize_kernel(int Q, const int* __restrict__ fail, double* __restrict__ A) {
  const int c = blockIdx.y;
  if (fail[c] == 0) return;
  const size_t QQ = static_cast<size_t>(Q) * Q;
  for (size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; o < QQ;
       o += static_cast<size_t>(gridDim.x) * blockDim.x)
    A[c * QQ + o] = (o % Q == o / Q) ? 1.0 : 0.0;
}

// Device pointers of one GP's run: the slot (the chunk workspace of `chunk` candidates and the inner optimiser's
// scratch) and the GP's inputs and counters
struct KgLargeBufs {
  int chunk = 0, aw_slots = 0;
  double *P, *V, *A, *mu, *stage, *Xt, *Pk, *Afull, *Ad, *KAu, *Bt, *Wd, *WdT, *muA, *S, *C, *Wts, *outVal, *outX,
      *outH, *best, *kg;
  double *Kx = nullptr, *Ct = nullptr, *Rm = nullptr, *Tp = nullptr, *T1 = nullptr, *T2 = nullptr, *R2 = nullptr,
         *G1 = nullptr, *grad = nullptr;
  int *fail, *start, *winner, *work, *dPs;
  double *aw, *D, *KD;
  unsigned long long* stats;
};

// scratch column sets (R rows x kMcThreads lanes) of the inner optimiser: one per resident CTA, at most 3 per SM and
// `bytes` in total, at least one
int kg_large_aw_slots(const KgLargeShape& sh, size_t bytes, int sms) {
  const size_t slot = static_cast<size_t>(sh.R) * kMcThreads * sizeof(double);
  return static_cast<int>(std::max<size_t>(1, std::min<size_t>(3 * static_cast<size_t>(sms), bytes / slot)));
}

// Lays out a slot for `chunk` candidates and `aw_slots` scratch column sets at cv: what the 2 GiB budget counts.
void kg_large_carve_slot(const KgLargeShape& sh, int chunk, int aw_slots, Carve& cv, KgLargeBufs& b) {
  const size_t ch = static_cast<size_t>(chunk), mc = static_cast<size_t>(sh.num_mc), Q = sh.Q, n = sh.n;
  const size_t QQ = Q * Q;
  b.chunk = chunk;
  b.aw_slots = aw_slots;
  b.P = cv.take<double>(ch * sh.U * sh.dim);
  b.V = cv.take<double>(ch * Q * n);
  b.A = cv.take<double>(ch * QQ);
  b.mu = cv.take<double>(ch * Q);
  b.stage = cv.take<double>(ch * ((Q + NB - 1) / NB) * NB * NB);
  b.Xt = cv.take<double>(ch * sh.Np * sh.DIMP);
  b.Pk = cv.take<double>(ch * sh.Np * 2);
  b.Afull = cv.take<double>(ch * sh.U * sh.dim);
  b.Ad = cv.take<double>(ch * sh.M * sh.DIMP);
  b.KAu = cv.take<double>(ch * n * sh.U);
  b.Bt = cv.take<double>(ch * n * Q);
  b.Wd = cv.take<double>(ch * Q * sh.M);
  b.WdT = cv.take<double>(ch * Q * sh.M);
  b.muA = cv.take<double>(ch * sh.M);
  b.S = cv.take<double>(ch * mc * sh.M);
  b.C = cv.take<double>(ch * mc * Q);
  b.Wts = cv.take<double>(ch * mc * sh.R);
  b.outVal = cv.take<double>(ch * mc);
  b.outX = cv.take<double>(ch * mc * sh.DIMP);
  b.outH = cv.take<double>(ch * mc);
  b.best = cv.take<double>(ch);
  b.kg = cv.take<double>(ch);
  b.fail = cv.take<int>(ch);
  b.start = cv.take<int>(ch * mc);
  b.winner = cv.take<int>(ch);
  if (sh.want_grad) {
    b.Kx = cv.take<double>(ch * mc * sh.R);
    b.Ct = cv.take<double>(ch * mc * Q);
    b.Rm = cv.take<double>(ch * sh.R * Q);
    b.Tp = cv.take<double>(ch * QQ);
    b.T1 = cv.take<double>(ch * QQ);
    b.T2 = cv.take<double>(ch * QQ);
    b.R2 = cv.take<double>(ch * n * sh.qb);
    b.G1 = cv.take<double>(ch * sh.q * sh.dim);
    b.grad = cv.take<double>(ch * sh.q * sh.dim);
  }
  b.aw = cv.take<double>(static_cast<size_t>(aw_slots) * sh.R * kMcThreads);
}

size_t kg_large_slot_bytes(const KgLargeShape& sh, int chunk, int aw_slots) {
  Carve cv;
  KgLargeBufs b;
  kg_large_carve_slot(sh, chunk, aw_slots, cv, b);
  return cv.off;
}

// Lays out one GP's inputs and counters at cv (beside the budget, as the call's other inputs and outputs): the
// discrete points, K(X, D), the derivative indices, the work counter and the statistics.
void kg_large_carve_io(const KgLargeShape& sh, Carve& cv, KgLargeBufs& b) {
  b.D = cv.take<double>(static_cast<size_t>(std::max(1, sh.num_pts)) * sh.dim);
  b.KD = cv.take<double>(static_cast<size_t>(sh.n) * std::max(1, sh.num_pts));
  b.dPs = cv.take<int>(std::max(1, sh.g));
  b.work = cv.take<int>(1);
  b.stats = cv.take<unsigned long long>(4);
}

// Every argument check of cmoe_kg_eval_large, in its order, and the workspace sizes; CMOE_ERR_BOUNDS when one
// candidate's workspace does not fit the 2 GiB beside the draws and the scratch.
KgLargeShape kg_large_shape(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner,
                            const double* inner_bounds, int num_pts, int num_candidates, int q, int p, int num_mc,
                            bool want_grad) {
  kg_large_check_sizes(num_candidates, q, p, num_mc);
  CMOE_REQUIRE(gp != nullptr, CMOE_ERR_INVALID_VALUE, "gp is NULL");
  const KernelSpec& spec = gp->spec;
  const int dim = spec.dim, g = spec.g, bs = 1 + g, U = q + p;
  CMOE_REQUIRE(static_cast<long long>(U) * bs <= CMOE_MAX_KG_LARGE_ROWS, CMOE_ERR_BOUNDS,
               "(q+p)*(1+num_derivatives) must be <= 1024");
  CMOE_REQUIRE(num_pts >= 0, CMOE_ERR_BOUNDS, "bad sizes");
  kg_check_inner(spec, num_fidelity, inner, inner_bounds);
  const int ps = dim - num_fidelity;
  const KgLargeEntry* entry = find_kg_large_entry(spec.kernel, dim, g);
  CMOE_REQUIRE(entry != nullptr, CMOE_ERR_BOUNDS, "dim exceeds the largest compiled q-KG kernel (32 dims)");
  KgLargeShape sh;
  sh.entry = entry;
  sh.nf = num_fidelity;
  sh.ps = ps;
  sh.q = q;
  sh.p = p;
  sh.U = U;
  sh.dim = dim;
  sh.g = g;
  sh.bs = bs;
  sh.num_pts = num_pts;
  sh.num_mc = num_mc;
  sh.want_grad = want_grad;
  sh.DIMP = entry->dim;
  sh.N = gp->N;
  sh.n = gp->n;
  sh.Q = U * bs;
  sh.Np = sh.N + U;
  sh.R = sh.Np * bs;
  sh.M = U + num_pts;
  sh.qb = q * bs;
  // device workspace of one candidate: the slot's layout for one candidate.  A chunk of c candidates takes at most
  // c per_bytes + kCarveSlack, since the alignment padding of its pieces does not grow with c.
  sh.per_bytes = kg_large_slot_bytes(sh, 1, 0);
  // per call: the draws Z and the inner optimiser's scratch; the chunks get the rest of the 2 GiB
  sh.z_bytes = static_cast<size_t>(num_mc) * sh.Q * sizeof(double);
  const size_t fixed = sh.z_bytes + kKgLargeScratchBytes + kCarveSlack;
  sh.budget = kSampleWorkspaceBytes > fixed ? kSampleWorkspaceBytes - fixed : 0;
  if (sh.per_bytes > sh.budget) {
    char msg[320];
    snprintf(msg, sizeof(msg),
             "one candidate's q-KG workspace (%zu bytes: Q = %d rows, N + U = %d points, num_mc = %d) does not fit "
             "the %zu bytes left of 2 GiB beside the call's normals and scratch",
             sh.per_bytes, sh.Q, sh.Np, num_mc, sh.budget);
    throw Error(CMOE_ERR_BOUNDS, msg);
  }
  return sh;
}

// doubles of kg_large_setup's region: Z [num_mc][Q], the step sizes, the candidates, the pending and the stale points
size_t kg_large_setup_doubles(const KgLargeShape& sh, const cmoe_gd_params* inner, int num_candidates) {
  return static_cast<size_t>(sh.num_mc) * sh.Q + std::max(1, inner->max_num_steps) +
         static_cast<size_t>(num_candidates) * sh.q * sh.dim + static_cast<size_t>(std::max(1, sh.p)) * sh.dim +
         static_cast<size_t>(sh.q) * sh.dim;
}

// The per-evaluation setup on `s` (returns once it has completed): the draws Z (Philox or the table, kg_prep_kernel's
// layout), the step sizes, the candidates, the pending and the stale points, in `dev` (kg_large_setup_doubles).
KgLargeInputs kg_large_setup(const KgLargeShape& sh, const cmoe_gd_params* inner, const double* candidates,
                             int num_candidates, const double* points_being_sampled, uint64_t seed,
                             const double* normals_table, const double* stale_union, double* dev, cudaStream_t s) {
  const size_t mc = static_cast<size_t>(sh.num_mc);
  KgLargeInputs in;
  double* Z = dev;
  double* alpha0 = Z + mc * sh.Q;
  double* cand = alpha0 + std::max(1, inner->max_num_steps);
  double* Xp = cand + static_cast<size_t>(num_candidates) * sh.q * sh.dim;
  double* stale = Xp + static_cast<size_t>(std::max(1, sh.p)) * sh.dim;
  DevBuf<double> dtable;
  if (normals_table) dtable.upload(normals_table, ((mc + 1) / 2) * sh.Q, s);
  kgl_normals_kernel<<<static_cast<unsigned>((mc * sh.Q + 255) / 256), 256, 0, s>>>(
      sh.Q, sh.num_mc, seed, normals_table ? dtable.p : nullptr, Z);
  count_launch();
  const std::vector<double> a0 = kg_step_sizes(*inner);
  CMOE_CUDA(cudaMemcpyAsync(alpha0, a0.data(), a0.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  CMOE_CUDA(cudaMemcpyAsync(cand, candidates, static_cast<size_t>(num_candidates) * sh.q * sh.dim * sizeof(double),
                            cudaMemcpyHostToDevice, s));
  if (sh.p)
    CMOE_CUDA(cudaMemcpyAsync(Xp, points_being_sampled, static_cast<size_t>(sh.p) * sh.dim * sizeof(double),
                              cudaMemcpyHostToDevice, s));
  if (stale_union)
    CMOE_CUDA(cudaMemcpyAsync(stale, stale_union, static_cast<size_t>(sh.q) * sh.dim * sizeof(double),
                              cudaMemcpyHostToDevice, s));
  // the host copies above are staged before the calls return; the table upload completes before dtable is freed
  CMOE_CUDA(cudaStreamSynchronize(s));
  in.Z = Z;
  in.alpha0 = alpha0;
  in.cand = cand;
  in.Xp = Xp;
  in.stale = stale_union ? stale : nullptr;
  return in;
}

// Enqueues one GP's evaluation of the nc candidates on `s` in chunks of b.chunk; nothing is read back.  kg_out[nc],
// grad_out[nc][q][dim] (if sh.want_grad) and fail_out[nc] (0 or the leading minor of a singular union) are device
// arrays.  hD / hderivs hold the host data of the asynchronous uploads until the caller has synchronised `s`.
void kg_large_run(const cmoe_gp& gp, const KgLargeShape& sh, const cmoe_gd_params* inner, const double* inner_bounds,
                  const KgLargeInputs& in, const KgLargeBufs& b, const double* discrete_pts, double best_so_far,
                  int num_candidates, int sms, cudaStream_t s, double* kg_out, double* grad_out, int* fail_out,
                  std::vector<double>& hD, std::vector<int>& hderivs) {
  const KernelSpec& spec = gp.spec;
  const int dim = sh.dim, g = sh.g, bs = sh.bs, U = sh.U, q = sh.q, ps = sh.ps, num_pts = sh.num_pts;
  const int num_mc = sh.num_mc, DIMP = sh.DIMP, N = sh.N, n = sh.n, Q = sh.Q, Np = sh.Np, R = sh.R, M = sh.M;
  const int qb = sh.qb, chunk = b.chunk;
  const bool want_grad = sh.want_grad;
  const size_t QQ = static_cast<size_t>(Q) * Q, mc = static_cast<size_t>(num_mc);
  const Centre ctr = centre_of(gp);
  // per GP: the discrete points (fidelity coordinates 1), K(X, D), the derivative indices
  hD = kg_pinned_discrete(discrete_pts, num_pts, ps, dim);
  CMOE_CUDA(cudaMemcpyAsync(b.D, hD.data(), hD.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  if (num_pts > 0) build_mix_covariance(spec, gp.dX.p, N, b.D, num_pts, nullptr, 0, b.KD, s);
  hderivs.assign(std::max(1, g), 0);
  for (int a = 0; a < g; ++a) hderivs[a] = spec.derivs[a];
  CMOE_CUDA(cudaMemcpyAsync(b.dPs, hderivs.data(), hderivs.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CMOE_CUDA(cudaMemsetAsync(b.stats, 0, 4 * sizeof(unsigned long long), s));

  // the training then the union points as one row set with per-sample weight columns: no union block, no pack weights
  KgMcParams m = kg_inner_params(gp, ps, M, num_mc, *inner, inner_bounds, in.alpha0);
  m.N = Np;
  m.pk_stride = 2;
  m.stats = b.stats;
  m.aw = b.aw;
  m.aw_slots = b.aw_slots;
  m.work = b.work;
  m.stage_ops = 0;

  for (int c0 = 0; c0 < num_candidates; c0 += chunk) {
    const int nb = std::min(chunk, num_candidates - c0);
    kgl_pack_kernel<<<nb, 256, 0, s>>>(spec, ctr, N, U, q, ps, num_pts, DIMP, gp.dX.p,
                                       in.cand + static_cast<size_t>(c0) * q * dim, in.Xp, b.D, in.stale, b.P, b.Xt,
                                       b.Pk, b.Afull, b.Ad);
    count_launch();
    // posterior of the union: V = L^-1 K*, mu, Var + noise[type], L_U, B = L^-T V
    posterior_cov_large(gp, b.P, b.dPs, b.V, b.mu, b.A, nb, U, g, 0.0, s);
    kgl_noise_kernel<<<static_cast<unsigned>((static_cast<size_t>(nb) * Q + 255) / 256), 256, 0, s>>>(
        nb, Q, bs, gp.dnoise.p, b.A);
    count_launch();
    CMOE_CUDA(cudaMemsetAsync(b.fail, 0, nb * sizeof(int), s));
    potrf_batched(b.A, Q, nb, b.fail, b.stage, s);
    CMOE_CUDA(cudaMemcpyAsync(fail_out + c0, b.fail, nb * sizeof(int), cudaMemcpyDeviceToDevice, s));
    zero_upper(nb, Q, b.A, s);
    kgl_sanitize_kernel<<<dim3(static_cast<unsigned>(std::min<size_t>((QQ + 255) / 256, 1024)), nb), 256, 0, s>>>(
        Q, b.fail, b.A);
    count_launch();
    trsm_lower_blocked(gp.dK.p, n, b.V, n, nb * Q, true, s);
    kgl_best_kernel<<<(nb + 127) / 128, 128, 0, s>>>(nb, U, bs, best_so_far, b.mu, b.best, b.winner);
    count_launch();
    // discretisation set: W = L_U^-1 Cov_n(Xu rows, A), mu_n(A); starts = first strict arg-min of mu_A + W^T z
    build_mix_covariance(spec, gp.dX.p, N, b.Afull, nb * U, nullptr, 0, b.KAu, s);
    // B^T K(X, A) on DMMA: B^T [Q][n] per candidate, then the union part and the shared discrete part of A
    transpose_batched(n, Q, b.V, b.Bt, nb, s);
    gemm_nn(Q, U, n, b.Bt, Q, static_cast<size_t>(Q) * n, b.KAu, n, static_cast<size_t>(n) * U, b.Wd, Q,
            static_cast<size_t>(Q) * M, nb, s);
    if (num_pts > 0)
      gemm_nn(Q, num_pts, n, b.Bt, Q, static_cast<size_t>(Q) * n, b.KD, n, 0, b.Wd + static_cast<size_t>(U) * Q, Q,
              static_cast<size_t>(Q) * M, nb, s);
    const size_t nwd = static_cast<size_t>(M) * (Q + 1);
    kgl_disc_cov_kernel<<<dim3(static_cast<unsigned>((nwd + 255) / 256), nb), 256, 0, s>>>(
        spec, n, U, num_pts, gp.mean, gp.dKinvY.p, b.P, b.Afull, b.D, b.KAu, b.KD, b.Wd, b.muA);
    count_launch();
    for (int c = 0; c < nb; ++c)
      trsm_lower_blocked(b.A + c * QQ, Q, b.Wd + static_cast<size_t>(c) * Q * M, Q, M, false, s);
    transpose_batched(Q, M, b.Wd, b.WdT, nb, s);
    gemm_nn(M, num_mc, Q, b.WdT, M, static_cast<size_t>(M) * Q, in.Z, Q, 0, b.S, M, mc * M, nb, s);
    kgl_argmin_kernel<<<dim3((num_mc + 255) / 256, nb), 256, 0, s>>>(M, num_mc, b.muA, b.S, b.start);
    count_launch();
    // C = L_U^-T Z and the weight columns
    for (int c = 0; c < nb; ++c) {
      double* Cc = b.C + static_cast<size_t>(c) * mc * Q;
      CMOE_CUDA(cudaMemcpyAsync(Cc, in.Z, mc * Q * sizeof(double), cudaMemcpyDeviceToDevice, s));
      trsm_lower_blocked(b.A + c * QQ, Q, Cc, Q, num_mc, true, s);
    }
    gemm_nn(n, num_mc, Q, b.V, n, static_cast<size_t>(n) * Q, b.C, Q, mc * Q, b.Wts, R, mc * R, nb, s);
    kgl_weights_kernel<<<dim3(static_cast<unsigned>((mc * R + 255) / 256), nb), 256, 0, s>>>(spec, n, Q, num_mc,
                                                                                          gp.dKinvY.p, b.C, b.Wts);
    count_launch();
    // inner optimisation of every sample
    KgMcParams prm = m;
    prm.chunk = kg_samples_per_item(nb, num_mc, sms, 3);  // the general path's 3 CTAs per SM
    prm.chunks = (num_mc + prm.chunk - 1) / prm.chunk;
    prm.work_total = prm.chunks * nb;
    prm.Xt = b.Xt;
    prm.Pk = b.Pk;
    prm.A = b.Ad;
    prm.recC = b.C;  // not read by the large-union build
    prm.recStart = b.start;
    prm.Wt = b.Wts;
    prm.outVal = b.outVal;
    prm.outX = b.outX;
    prm.outH = b.outH;
    CMOE_CUDA(cudaMemsetAsync(b.work, 0, sizeof(int), s));
    sh.entry->mc(prm, s);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    if (inner->max_num_restarts <= 0) kg_fill_points(spec, ctr, nb * num_mc, DIMP, b.outX, b.outH, s);
    kg_value(nb, num_mc, b.outVal, b.best, b.fail, b.kg, s);
    CMOE_CUDA(cudaMemcpyAsync(kg_out + c0, b.kg, nb * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if (want_grad) {
      // R = Kx C^T over the samples, [Q][R] (column a of length R = n + Q)
      kgl_kx_kernel<<<dim3(static_cast<unsigned>((mc * R + 255) / 256), nb), 256, 0, s>>>(
          spec, ctr, N, U, num_mc, DIMP, gp.dX.p, b.P, b.outX, b.Kx);
      count_launch();
      transpose_batched(Q, num_mc, b.C, b.Ct, nb, s);
      gemm_nn(R, Q, num_mc, b.Kx, R, mc * R, b.Ct, num_mc, mc * Q, b.Rm, R, static_cast<size_t>(R) * Q, nb, s);
      kg_tprime(nb, n, Q, Q, b.Rm, b.V, b.Tp, s);
      potrs_lower(gp.dK.p, n, b.Rm, R, nb * Q, s);
      kg_g1(spec, ctr, nb, U, q, Q, DIMP, num_mc, b.P, b.C, b.outX, b.G1, s);
      // Lbar = tril(T' L_U^-T) / num_mc, then 2 Sigmabar through the Cholesky adjoint, and R2 = B 2 Sigmabar
      for (int c = 0; c < nb; ++c) trsm_lower_blocked(b.A + c * QQ, Q, b.Tp + c * QQ, Q, Q, false, s);
      kgl_lbar_kernel<<<dim3(static_cast<unsigned>((QQ + 255) / 256), nb), 256, 0, s>>>(Q, num_mc, b.Tp, b.T1);
      count_launch();
      cholesky_adjoint(b.A, Q, nb, b.T1, b.T2, s);
      gemm_nn(n, qb, Q, b.V, n, static_cast<size_t>(n) * Q, b.T1, Q, QQ, b.R2, n, static_cast<size_t>(n) * qb, nb, s);
      kgl_grad_kernel<<<dim3(q, nb), kGradThreads, 0, s>>>(spec, N, U, q, num_mc, gp.dX.p, gp.dKinvY.p, b.P, b.Rm,
                                                          b.T1, b.R2, b.G1, b.winner, b.grad);
      count_launch();
      CMOE_CUDA(cudaGetLastError());
      CMOE_CUDA(cudaMemcpyAsync(grad_out + static_cast<size_t>(c0) * q * dim, b.grad,
                                static_cast<size_t>(nb) * q * dim * sizeof(double), cudaMemcpyDeviceToDevice, s));
    }
  }
}

}  // namespace

void kg_large_eval(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* inner,
                   const double* inner_bounds, const double* discrete_pts, int num_pts, const double* candidates,
                   int num_candidates, int q, const double* points_being_sampled, int p, int num_mc,
                   const double* best_so_far, uint64_t seed, const double* normals_table, const double* stale_union,
                   double* values, double* grads, cmoe_kg_stats* stats) {
  const bool want_grad = grads != nullptr;
  std::vector<KgLargeShape> sh;
  size_t per = 0, slot_max = 0;
  for (int m = 0; m < num_gp; ++m) {
    sh.push_back(kg_large_shape(gps[m], num_fidelity, inner, inner_bounds, num_pts, num_candidates, q, p, num_mc,
                                want_grad));
    per = std::max(per, sh.back().per_bytes);
    slot_max = std::max(slot_max, static_cast<size_t>(sh.back().R) * kMcThreads * sizeof(double));
  }
  require_device(gps[0]->device);
  const int sms = sm_count();
  // Each member in flight gets an even share of the chunks' budget and of the inner optimiser's scratch, so the members
  // in flight are also bounded by one scratch column set each.  A slot then takes at most (budget + kCarveSlack) / width
  // + scratch, so Z and the slots stay within 2 GiB.
  const KgLargeShape& s0 = sh[0];
  const MemberSchedule ms =
      schedule_members(num_gp, num_candidates, s0.budget + kCarveSlack, per, kKgLargeScratchBytes / slot_max);
  const size_t scratch = kKgLargeScratchBytes / ms.width;
  size_t slot_bytes = 0;
  for (const KgLargeShape& x : sh)
    slot_bytes = std::max(slot_bytes, kg_large_slot_bytes(x, ms.chunk, kg_large_aw_slots(x, scratch, sms)));
  slot_bytes = slot_stride(slot_bytes);
  // one region on the first member's handle: the evaluation's inputs (Z first), every member's results, inputs and
  // counters, then the slots
  const size_t ps = static_cast<size_t>(q) * s0.dim, nc = num_candidates;
  std::vector<KgLargeBufs> io(num_gp);
  double *in_dev = nullptr, *dval = nullptr, *dgrad = nullptr;
  int* dfail = nullptr;
  char* slots = nullptr;
  LargeUnionWork& w = carve_large_union_work(*gps[0], [&](Carve& cv) {
    in_dev = cv.take<double>(kg_large_setup_doubles(s0, inner, num_candidates));
    dval = cv.take<double>(static_cast<size_t>(num_gp) * nc);
    dgrad = want_grad ? cv.take<double>(static_cast<size_t>(num_gp) * nc * ps) : nullptr;
    dfail = cv.take<int>(static_cast<size_t>(num_gp) * nc);
    for (int m = 0; m < num_gp; ++m) kg_large_carve_io(sh[m], cv, io[m]);
    slots = cv.take<char>(slot_bytes * ms.width);
  });
  cudaStream_t st0 = gps[0]->stream;
  const KgLargeInputs in = kg_large_setup(s0, inner, candidates, num_candidates, points_being_sampled, seed,
                                          normals_table, stale_union, in_dev, st0);
  std::vector<std::vector<double>> hD(num_gp);
  std::vector<std::vector<int>> hderivs(num_gp);
  run_members(gps, num_gp, ms.width, w, [&](int m, int slot) {
    KgLargeBufs b = io[m];
    Carve sc{slots + slot * slot_bytes};
    kg_large_carve_slot(sh[m], ms.chunk, kg_large_aw_slots(sh[m], scratch, sms), sc, b);
    kg_large_run(*gps[m], sh[m], inner, inner_bounds, in, b, discrete_pts + static_cast<size_t>(m) * num_pts * s0.ps,
                 best_so_far[m], num_candidates, sms, gps[m]->stream, dval + m * nc,
                 want_grad ? dgrad + m * nc * ps : nullptr, dfail + m * nc, hD[m], hderivs[m]);
  });
  std::vector<unsigned long long> st(stats ? 4 * static_cast<size_t>(num_gp) : 0);
  for (int m = 0; m < static_cast<int>(st.size() / 4); ++m)
    CMOE_CUDA(cudaMemcpyAsync(st.data() + 4 * m, io[m].stats, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                              st0));
  drain_members(st0, num_gp, num_candidates, ps, dval, dgrad, dfail, values, grads);  // synchronises st0
  if (stats) {
    *stats = cmoe_kg_stats{};
    stats->mc_samples = static_cast<uint64_t>(num_gp) * num_candidates * num_mc;
    for (int m = 0; m < num_gp; ++m) {
      stats->posterior_evals += st[4 * m];
      stats->line_search_steps += st[4 * m + 1];
      stats->point_evals += st[4 * m + 2];
      stats->line_batches += st[4 * m + 3];
    }
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
    kg_large_eval(&gp, 1, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, candidates, num_candidates, q,
                  points_being_sampled, p, num_mc, &best_so_far, seed, normals_table, nullptr, kg, grad_kg, stats);
  });
}

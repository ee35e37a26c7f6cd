// q-KG evaluation (value + envelope-theorem gradient), batched over candidates: host orchestration and the small
// per-candidate kernels around the fused Monte-Carlo kernel of kg_mc.cuh.
//
// Replaces (reference, moe/optimal_learning/cpp/gpp_knowledge_gradient_optimization.{hpp,cpp}):
//   KnowledgeGradientState ctor / PreCompute          .cpp:246-317
//   KnowledgeGradientEvaluator::ComputeKnowledgeGradient      .cpp:69-115
//   KnowledgeGradientEvaluator::ComputeGradKnowledgeGradient  .cpp:130-227
//   EvaluateKGAtPointList                              .hpp:972-1013
//
// Pipeline per batch of candidates (everything asynchronous on one stream, inputs resident in HBM):
//   posterior set-up (posterior.cu) -> discretisation-set statistics W = L^-1 Cov_n(Xu, A), mu_n(A)
//   -> per-sample prep (normals, c = L^-T z, arg-min over the discretisation set)
//   -> fused MC kernel (inner line-search optimisation of every sample)
//   -> [gradient] accumulate R = sum_i k(X, x*_i) c_i^T, K^-1 R, contraction with dK*, dL  -> KG, grad KG.
#include <algorithm>
#include <cstdlib>
#include <cmath>
#include <cstring>

#include "kg_mc.cuh"

namespace cmoe {

namespace {

std::vector<KgDispatchEntry>& kg_table() {
  static std::vector<KgDispatchEntry> t;
  return t;
}

__device__ __forceinline__ int row_type(int local, const int* derivs) { return local ? derivs[local - 1] : -1; }

// union sets on the device: P[c] = [candidate c ; points being sampled] (build_union_sets)
__global__ void build_union_kernel(const double* __restrict__ cand, const double* __restrict__ Xp, int nc, int q, int p,
                                   int dim, double* __restrict__ P) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t per = static_cast<size_t>(q + p) * dim;
  if (e >= per * nc) return;
  const size_t c = e / per, r = e % per;
  P[e] = (r < static_cast<size_t>(q) * dim) ? cand[c * q * dim + r] : Xp[r - static_cast<size_t>(q) * dim];
}

// Frame of the MC and accumulation kernels' operands.  They form -r^2/2 as x.y - |x|^2/2 - |y|^2/2 (e_j, e_u, outH),
// whose absolute error grows with |x|^2 + |y|^2 in length-scale units, so every operand they read is taken relative to
// the GP's centre (cmoe_gp::centre, the frame of the fit's covariance build): the training points (Xt), the union points
// (Xu), the start points (A, fidelity coordinates too), the inner bounds (KgMcParams::lo/hi) and, through them, the
// minimisers (outX, outH).  The kernels are translation invariant.  The difference-form consumers (build_mix_covariance,
// kg_discrete_kernel, the posterior batch, kg_grad_kernel's dK* terms) keep raw coordinates: D, Afull and pb.P stay raw,
// and kg_g1_kernel moves outX back before differencing.
//
// scaled + zero-padded training points [N][DIMP]
__global__ void pack_xt_kernel(const __grid_constant__ KernelSpec spec, const __grid_constant__ Centre ctr,
                               const double* __restrict__ X, int N, int DIMP, double* __restrict__ Xt) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * DIMP) return;
  const int j = e / DIMP, d = e % DIMP;
  Xt[e] = (d < spec.dim) ? (X[static_cast<size_t>(j) * spec.dim + d] - ctr.c[d]) * spec.inv_len[d] : 0.0;
}

// per-candidate operand packs for the MC kernel.  g == 0: the pack row of training point j is [ e_j | beta_j, B_j,0..QP-1 ]
// (stride QP + 2).  g > 0: training point j owns rows r = (j, m), m = 0..g; the pack row is [ e_j | 0 ] and the weights go
// to the table Wt[1+QP][N(1+g)]: Wt[0][r] = beta~_r, Wt[1+u][r] = B~_(r,u)  (~ = divided by l_t, t = derivs[m-1], so
// that derivative rows multiply plain scaled coordinate differences in the kernel).
// Xu and A are in the centred frame; Afull keeps raw coordinates.
__global__ void __launch_bounds__(256) kg_pack_kernel(const __grid_constant__ KernelSpec spec,
                                                      const __grid_constant__ Centre ctr, int N, int U, int ps,
                                                      int num_pts, int DIMP, int QP, int stride,
                                                      const double* __restrict__ Xt, const double* __restrict__ beta,
                                                      const double* __restrict__ B, const double* __restrict__ P,
                                                      const double* __restrict__ D, double* __restrict__ Pk,
                                                      double* __restrict__ Xu, double* __restrict__ A,
                                                      double* __restrict__ Afull, const double* __restrict__ stale,
                                                      int q, double* __restrict__ Wt) {
  const int c = blockIdx.x, tid = threadIdx.x, dim = spec.dim, b1 = 1 + spec.g, n = N * b1, Q = U * b1;
  const bool se = spec.kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL;
  const double lna = log(spec.alpha);
  double* pk = Pk + static_cast<size_t>(c) * N * stride;
  const double* Bc = B + static_cast<size_t>(c) * Q * n;
  for (int j = tid; j < N; j += blockDim.x) {
    double nrm = 0.0;
    for (int d = 0; d < DIMP; ++d) nrm = fma(Xt[j * DIMP + d], Xt[j * DIMP + d], nrm);
    double* o = pk + static_cast<size_t>(j) * stride;
    o[0] = se ? (lna - 0.5 * nrm) : nrm;
    if (spec.g == 0) {
      o[1] = beta[j];
      for (int u = 0; u < QP; ++u) o[2 + u] = (u < Q) ? Bc[static_cast<size_t>(u) * n + j] : 0.0;
    } else {
      o[1] = 0.0;
    }
  }
  if (spec.g > 0) {
    double* wt = Wt + static_cast<size_t>(c) * (1 + QP) * n;
    for (int e = tid; e < (1 + QP) * n; e += blockDim.x) {
      const int u = e / n - 1, r = e % n, m = r % b1;
      const double sc = m ? spec.inv_len[spec.derivs[m - 1]] : 1.0;
      wt[e] = (u < 0) ? beta[r] * sc : ((u < Q) ? Bc[static_cast<size_t>(u) * n + r] * sc : 0.0);
    }
  }
  const double* Pc = P + static_cast<size_t>(c) * U * dim;
  double* xu = Xu + static_cast<size_t>(c) * U * (DIMP + 2);
  for (int u = tid; u < U; u += blockDim.x) {
    double nrm = 0.0;
    for (int d = 0; d < DIMP; ++d) {
      const double v = (d < dim) ? (Pc[u * dim + d] - ctr.c[d]) * spec.inv_len[d] : 0.0;
      xu[u * (DIMP + 2) + d] = v;
      nrm = fma(v, v, nrm);
    }
    xu[u * (DIMP + 2) + DIMP] = se ? (lna - 0.5 * nrm) : nrm;
    xu[u * (DIMP + 2) + DIMP + 1] = 0.0;
  }
  // discretisation set: [union (free coords) ; discrete_pts], fidelity coordinates pinned to 1.0 (...cpp:259-261, 365)
  const int M = U + num_pts;
  double* Ac = A + static_cast<size_t>(c) * M * DIMP;
  double* Af = Afull + static_cast<size_t>(c) * U * dim;
  for (int e = tid; e < M * DIMP; e += blockDim.x) {
    const int j = e / DIMP, d = e % DIMP;
    double v = 0.0;
    if (d < ps) {
      // `stale`: the reference's multistart drivers reuse ONE state whose discretisation set keeps the q points it was
      // constructed with (SetCurrentPoint does not refresh discretized_set,
      // gpp_knowledge_gradient_optimization.cpp:233-243, 259-261) — those points stand in for the current ones here
      v = (j < U) ? ((stale != nullptr && j < q) ? stale[j * dim + d] : Pc[j * dim + d])
                  : D[static_cast<size_t>(j - U) * dim + d];
    } else if (d < dim) {
      v = 1.0;
    }
    Ac[e] = (d < dim) ? v - ctr.c[d] : 0.0;
    if (j < U && d < dim) Af[j * dim + d] = v;
  }
}

// Start-point table (g == 0), one CTA per (discretisation point m, candidate).  The fused MC kernel starts every sample's
// inner descent at A_m = A[recStart]; there mu+ - m and the sums of its POINT round are affine in c = L^-T z:
//     S0 = sum_j beta_j k_j + sum_u c_u (k(a, Xu_u) - sum_j B_ju k_j),  k_j = k(a, X_j)
// and likewise SB (kb in place of k) and s_d (kb X~_jd).  Out[m][r][col], r = 0 (beta part) or 1 + u, col = S0, SB, s_d:
// row r's weights are w_j = beta_j (r = 0) or -B_ju, and 1 on union row u (r = 1 + u).  The kernel values come from the
// MC kernel's own operands (Xt, Pk, Xu: the same e_j and the same exp); every sum runs over the training rows, then the
// union rows, in ascending order, with the POINT round's per-row rounding, so a candidate's table does not depend on its
// batch.  fast: the MC kernel's shared-memory fast path (table exp, and all kernel values 0 beyond kFarRadius).
constexpr int kStartThreads = 256;
constexpr int kStartOuts = 5;  // outputs per thread: (1 + QP)(DIMP + 2) <= 33 x 34 = 1122 <= 5 x 256
static_assert(kStartOuts * kStartThreads >= (1 + CMOE_MAX_KG_ROWS) * (CMOE_MAX_DIM + 2),
              "start table outputs per CTA (QP <= CMOE_MAX_KG_ROWS)");
__global__ void __launch_bounds__(kStartThreads) kg_start_kernel(const __grid_constant__ KernelSpec spec, int N, int U,
                                                                 int M, int DIMP, int QP, int fast,
                                                                 const double* __restrict__ Xt,
                                                                 const double* __restrict__ Pk,
                                                                 const double* __restrict__ Xu,
                                                                 const double* __restrict__ A,
                                                                 double* __restrict__ Out) {
  __shared__ double s_kv[kStartThreads], s_kb[kStartThreads];
  const int m = blockIdx.x, c = blockIdx.y, tid = threadIdx.x, W = DIMP + 2, nout = (1 + QP) * W;
  const bool se = spec.kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL;
  if (fast) exp_table_stage();
  const double* a = A + (static_cast<size_t>(c) * M + m) * DIMP;
  const double* pk = Pk + static_cast<size_t>(c) * N * (QP + 2);
  const double* xu = Xu + static_cast<size_t>(c) * U * (DIMP + 2);
  double nq = 0.0;
  for (int d = 0; d < spec.dim; ++d) {  // the padding coordinates are 0 in every operand
    const double x = a[d] * spec.inv_len[d];
    nq = fma(x, x, nq);
  }
  const double hq = -0.5 * nq;
  double acc[kStartOuts];
#pragma unroll
  for (int k = 0; k < kStartOuts; ++k) acc[k] = 0.0;
  for (int j0 = 0; j0 < N + U; j0 += kStartThreads) {
    const int j = j0 + tid;
    if (j < N + U) {
      const double* xj = (j < N) ? Xt + static_cast<size_t>(j) * DIMP : xu + static_cast<size_t>(j - N) * (DIMP + 2);
      const double pk0 = (j < N) ? pk[static_cast<size_t>(j) * (QP + 2)] : xj[DIMP];
      double dot = 0.0;
      for (int d = 0; d < spec.dim; ++d) dot = fma(a[d] * spec.inv_len[d], xj[d], dot);
      double kv, kb;
      if (!se) {
        kernel_pair<CMOE_KERNEL_MATERN_NU_2P5>(dot, pk0, hq, spec.alpha, kv, kb);
      } else if (fast) {
        kernel_pair<CMOE_KERNEL_SQUARE_EXPONENTIAL, true>(dot, pk0, hq, spec.alpha, kv, kb);
      } else {
        kernel_pair<CMOE_KERNEL_SQUARE_EXPONENTIAL, false>(dot, pk0, hq, spec.alpha, kv, kb);
      }
      s_kv[tid] = kv;
      s_kb[tid] = kb;
    }
    __syncthreads();
    const int jn = min(kStartThreads, N + U - j0);
#pragma unroll
    for (int k = 0; k < kStartOuts; ++k) {
      const int o = tid + k * kStartThreads;
      if (o < nout) {
        const int r = o / W, col = o % W;
        for (int i = 0; i < jn; ++i) {
          const int jj = j0 + i;
          double w;
          const double* xj;
          if (jj < N) {
            const double* pr = pk + static_cast<size_t>(jj) * (QP + 2);
            w = (r == 0) ? pr[1] : -pr[1 + r];
            xj = Xt + static_cast<size_t>(jj) * DIMP;
          } else {
            w = (r == 1 + (jj - N)) ? 1.0 : 0.0;
            xj = xu + static_cast<size_t>(jj - N) * (DIMP + 2);
          }
          if (col == 0 || (se && col == 1)) {  // SquareExponential: SB = S0, as the POINT round sets it
            acc[k] = fma(w, s_kv[i], acc[k]);
          } else if (col == 1) {
            acc[k] += w * s_kb[i];
          } else {
            acc[k] = fma(w * s_kb[i], xj[col - 2], acc[k]);
          }
        }
      }
    }
    __syncthreads();
  }
  double* out = Out + (static_cast<size_t>(c) * M + m) * nout;
  const bool far = fast && nq > kFarRadius * kFarRadius;  // see kFastPathRadius: every kernel value is exactly 0
#pragma unroll
  for (int k = 0; k < kStartOuts; ++k) {
    const int o = tid + k * kStartThreads;
    if (o < nout) out[o] = far ? 0.0 : acc[k];
  }
}

// W = L^-1 Cov_n(Xu rows, A), mu_n(A), best_posterior and its arg-min, one CTA per candidate.
// KAu = K(X rows, A_union part) [n][nc*U], KD = K(X rows, D) [n][num_pts] (shared by all candidates), muD = mu_n(D).
__global__ void __launch_bounds__(256) kg_discrete_kernel(const __grid_constant__ KernelSpec spec, int n, int U,
                                                          int num_pts, int QP, double mean, double best_so_far,
                                                          const double* __restrict__ beta,
                                                          const double* __restrict__ P,
                                                          const double* __restrict__ Afull,
                                                          const double* __restrict__ D,
                                                          const double* __restrict__ KAu,
                                                          const double* __restrict__ KD,
                                                          const double* __restrict__ muD,
                                                          const double* __restrict__ B,
                                                          const double* __restrict__ mu,
                                                          const double* __restrict__ chol,
                                                          const int* __restrict__ fail, double* __restrict__ W,
                                                          double* __restrict__ muA, double* __restrict__ best_post,
                                                          int* __restrict__ winner) {
  extern __shared__ double sm[];
  const int c = blockIdx.x, tid = threadIdx.x, dim = spec.dim, M = U + num_pts, bs = 1 + spec.g, Q = U * bs;
  if (fail[c] != 0) return;
  double* Ls = sm;  // [Q][Q] column-major
  for (int e = tid; e < Q * Q; e += blockDim.x) Ls[e] = chol[static_cast<size_t>(c) * Q * Q + e];
  __syncthreads();
  const double* Pc = P + static_cast<size_t>(c) * U * dim;
  const double* Bc = B + static_cast<size_t>(c) * Q * n;
  double* Wc = W + static_cast<size_t>(c) * M * QP;
  for (int j = tid; j < M; j += blockDim.x) {
    const double* kcol = (j < U) ? (KAu + (static_cast<size_t>(c) * U + j) * n) : (KD + static_cast<size_t>(j - U) * n);
    const double* aj = (j < U) ? (Afull + (static_cast<size_t>(c) * U + j) * dim) : (D + static_cast<size_t>(j - U) * dim);
    double m;
    if (j < U) {
      m = 0.0;
      for (int r = 0; r < n; ++r) m += kcol[r] * beta[r];
      m += mean;
    } else {
      m = muD[j - U];
    }
    muA[static_cast<size_t>(c) * M + j] = m;
    double v[kMaxQ];
    for (int a = 0; a < Q; ++a) {
      const double* ba = Bc + static_cast<size_t>(a) * n;
      double t = 0.0;
      for (int r = 0; r < n; ++r) t += ba[r] * kcol[r];
      const double* pa = Pc + (a / bs) * dim;
      const KParts kp = kernel_parts(spec, weighted_sqdist(spec, pa, aj));
      v[a] = cov_entry(spec, kp, pa, aj, row_type(a % bs, spec.derivs), -1) - t;
    }
    // forward substitution  L w = v
    for (int a = 0; a < Q; ++a) {
      double t = v[a];
      for (int b = 0; b < a; ++b) t -= Ls[a + b * Q] * v[b];
      v[a] = t / Ls[a + a * Q];
    }
    for (int a = 0; a < QP; ++a) Wc[static_cast<size_t>(j) * QP + a] = (a < Q) ? v[a] : 0.0;
  }
  if (tid == 0) {
    // best_posterior = min(best_so_far, min_j mu_j) over the function-value rows, first strict minimiser (...cpp:146-153)
    double bp = best_so_far;
    int w = -1;
    for (int j = 0; j < U; ++j) {
      const double m = mu[static_cast<size_t>(c) * Q + j * bs];
      if (m < bp) {
        bp = m;
        w = j;
      }
    }
    best_post[c] = bp;
    winner[c] = w;
  }
}

// per sample: normals (antithetic pairs), c = L^-T z, arg-min of mu_n(A_j) + W_j . z over the discretisation set
__global__ void __launch_bounds__(256) kg_prep_kernel(int Q, int M, int QP, int num_mc, uint64_t seed,
                                                      const double* __restrict__ table,
                                                      const double* __restrict__ chol, const double* __restrict__ W,
                                                      const double* __restrict__ muA, const int* __restrict__ fail,
                                                      int w_in_smem, double* __restrict__ recC,
                                                      int* __restrict__ recStart) {
  extern __shared__ double sm[];
  const int c = blockIdx.y;
  if (fail[c] != 0) {
    // singular candidate: its KG is NaN, but the MC kernel still runs over its samples; keep their records in range
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < num_mc) {
      recStart[static_cast<size_t>(c) * num_mc + s] = 0;
      for (int a = 0; a < QP; ++a) recC[(static_cast<size_t>(c) * num_mc + s) * QP + a] = 0.0;
    }
    return;
  }
  double* Ls = sm;
  double* Ws = sm + Q * Q;
  double* ms = Ws + (w_in_smem ? static_cast<size_t>(M) * QP : 0);
  for (int e = threadIdx.x; e < Q * Q; e += blockDim.x) Ls[e] = chol[static_cast<size_t>(c) * Q * Q + e];
  const double* Wc = W + static_cast<size_t>(c) * M * QP;
  const double* mc_ = muA + static_cast<size_t>(c) * M;
  if (w_in_smem) {
    for (int e = threadIdx.x; e < M * QP; e += blockDim.x) Ws[e] = Wc[e];
    for (int e = threadIdx.x; e < M; e += blockDim.x) ms[e] = mc_[e];
  }
  __syncthreads();
  const double* Wp = w_in_smem ? Ws : Wc;
  const double* mp = w_in_smem ? ms : mc_;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= num_mc) return;
  const int pair = s >> 1;
  const double sign = (s & 1) ? -1.0 : 1.0;  // odd iterations reuse -z of the previous one (...cpp:88-97)
  double z[kMaxQ];
  if (table != nullptr) {
    for (int i = 0; i < Q; ++i) z[i] = sign * table[static_cast<size_t>(pair) * Q + i];
  } else {
    for (int k = 0; 2 * k < Q; ++k) {
      double a, b;
      philox_normal_pair(seed, static_cast<uint64_t>(pair), k, a, b);
      z[2 * k] = sign * a;
      if (2 * k + 1 < Q) z[2 * k + 1] = sign * b;
    }
  }
  // arg-min over the discretisation set (first strict minimiser, ...cpp:436-449)
  int arg = 0;
  double best = 0.0;
  for (int j = 0; j < M; ++j) {
    double v = mp[j];
    for (int a = 0; a < Q; ++a) v = fma(Wp[static_cast<size_t>(j) * QP + a], z[a], v);
    if (j == 0 || best > v) {
      best = v;
      arg = j;
    }
  }
  recStart[static_cast<size_t>(c) * num_mc + s] = arg;
  // c = L^-T z (back substitution)
  for (int a = Q - 1; a >= 0; --a) {
    double t = z[a];
    for (int b = a + 1; b < Q; ++b) t -= Ls[b + a * Q] * z[b];
    z[a] = t / Ls[a + a * Q];
  }
  double* out = recC + (static_cast<size_t>(c) * num_mc + s) * QP;
  for (int a = 0; a < QP; ++a) out[a] = (a < Q) ? z[a] : 0.0;
}

// Inner max_num_restarts = 0: the MC kernel leaves every sample's minimiser at the reference's fill value, 1.0 in each
// coordinate, but writes it without the centre; put that point in the operands' frame.
__global__ void kg_fill_point_kernel(const __grid_constant__ KernelSpec spec, const __grid_constant__ Centre ctr,
                                     int samples, int DIMP, double* __restrict__ outX, double* __restrict__ outH) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= samples) return;
  double nx = 0.0;
  for (int d = 0; d < DIMP; ++d) {
    const double x = (d < spec.dim) ? (1.0 - ctr.c[d]) * spec.inv_len[d] : 0.0;
    outX[static_cast<size_t>(i) * DIMP + d] = x;
    nx = fma(x, x, nx);
  }
  outH[i] = -0.5 * nx;
}

// KG[c] = best_posterior + mean_i best_function_value_i ; fixed-order reduction
__global__ void __launch_bounds__(256) kg_value_kernel(int num_mc, const double* __restrict__ outVal,
                                                       const double* __restrict__ best_post,
                                                       const int* __restrict__ fail, double* __restrict__ kg) {
  __shared__ double red[8];
  const int c = blockIdx.x;
  if (fail[c] != 0) {
    if (threadIdx.x == 0) kg[c] = nan("");
    return;
  }
  const double* v = outVal + static_cast<size_t>(c) * num_mc;
  double part = 0.0;
  for (int s = threadIdx.x; s < num_mc; s += blockDim.x) part += v[s];
  const double total = block_sum(part, red);
  if (threadIdx.x == 0) kg[c] = best_post[c] + total / static_cast<double>(num_mc);
}

// T' [a', a] = R[a'][n + a] - sum_rows R[a'][row] B[row, a]   (must run BEFORE R is overwritten by K^-1 R)
__global__ void __launch_bounds__(256) kg_tprime_kernel(int n, int Q, int QP, const double* __restrict__ R,
                                                        const double* __restrict__ B, double* __restrict__ Tp) {
  const int c = blockIdx.x;
  const double* Rc = R + static_cast<size_t>(c) * QP * (n + Q);
  const double* Bc = B + static_cast<size_t>(c) * Q * n;
  for (int o = threadIdx.x; o < Q * Q; o += blockDim.x) {
    const int ap = o / Q, a = o % Q;
    const double* r = Rc + static_cast<size_t>(ap) * (n + Q);
    const double* b = Bc + static_cast<size_t>(a) * n;
    double t = 0.0;
    for (int j = 0; j < n; ++j) t += r[j] * b[j];
    Tp[static_cast<size_t>(c) * Q * Q + o] = r[n + a] - t;
  }
}

// G1[p][d] = sum_i sum_m c_i,(p,m) d K(Xu_p row m, x*_i) / d Xu_p,d ; grid nc.  Every output (p, d) is summed by
// kG1Split threads over the samples i = t, t + kG1Split, ... and the partial sums are combined in a fixed order, so the
// result does not depend on scheduling.
constexpr int kG1Split = 16;
// P is raw, outX centred and scaled: x*_i is moved back to raw coordinates before the difference.
__global__ void __launch_bounds__(256) kg_g1_kernel(const __grid_constant__ KernelSpec spec,
                                                    const __grid_constant__ Centre ctr, int U, int q, int QP,
                                                    int DIMP, int num_mc, const double* __restrict__ P,
                                                    const double* __restrict__ recC, const double* __restrict__ outX,
                                                    double* __restrict__ G1) {
  __shared__ double part[256];
  const int cand = blockIdx.x, dim = spec.dim, bs = 1 + spec.g;
  const double* xs = outX + static_cast<size_t>(cand) * num_mc * DIMP;
  const double* cs = recC + static_cast<size_t>(cand) * num_mc * QP;
  double len[CMOE_MAX_DIM];
  for (int e = 0; e < dim; ++e) len[e] = 1.0 / spec.inv_len[e];
  const int outs_per_pass = blockDim.x / kG1Split;
  for (int o0 = 0; o0 < q * dim; o0 += outs_per_pass) {
    const int o = o0 + threadIdx.x / kG1Split, t = threadIdx.x % kG1Split;
    double acc = 0.0;
    if (o < q * dim) {
      const int p = o / dim, d = o % dim;
      const double* pp = P + (static_cast<size_t>(cand) * U + p) * dim;
      for (int i = t; i < num_mc; i += kG1Split) {
        double xi[CMOE_MAX_DIM];
        for (int e = 0; e < dim; ++e) xi[e] = fma(xs[static_cast<size_t>(i) * DIMP + e], len[e], ctr.c[e]);
        const KParts kp = kernel_parts(spec, weighted_sqdist(spec, pp, xi));
        const double* ci = cs + static_cast<size_t>(i) * QP;
        for (int m = 0; m < bs; ++m)
          acc = fma(ci[p * bs + m], grad_cov_entry(spec, kp, pp, xi, row_type(m, spec.derivs), -1, d), acc);
      }
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    if (t == 0 && o < q * dim) {
      double tot = 0.0;
      for (int k = 0; k < kG1Split; ++k) tot += part[threadIdx.x + k];
      G1[static_cast<size_t>(cand) * q * dim + o] = tot;
    }
    __syncthreads();
  }
}

// grad KG[c][p][d] = [p == winner] dmu_p[d] - (1/mc) ( G1 - sum_rows dK*[d,row,(p,m)] (K^-1 R)[row,(p,m)] - <dL_pd, T> )
// G1 comes either from kg_g1_kernel (general) or from the fast-path accumulators Gu/GkB (g == 0).
__global__ void __launch_bounds__(128) kg_grad_kernel(const __grid_constant__ KernelSpec spec, int N, int U, int q,
                                                      int QP, int DIMP, int num_mc, const double* __restrict__ X,
                                                      const double* __restrict__ P, const double* __restrict__ Xu,
                                                      const double* __restrict__ R, const double* __restrict__ Tp,
                                                      const double* __restrict__ Gu, const double* __restrict__ GkB,
                                                      const double* __restrict__ G1, const double* __restrict__ chol,
                                                      const double* __restrict__ gchol,
                                                      const double* __restrict__ gmu, const int* __restrict__ winner,
                                                      const int* __restrict__ fail, double* __restrict__ grad) {
  extern __shared__ double sm[];
  const int c = blockIdx.x, tid = threadIdx.x, dim = spec.dim, b1 = 1 + spec.g, n = N * b1, Q = U * b1;
  if (fail[c] != 0) return;
  double* T = sm;  // [Q][Q] row a', col b
  const double* Lc = chol + static_cast<size_t>(c) * Q * Q;
  // T L^T = T'  ->  row-wise forward substitution
  for (int ap = tid; ap < Q; ap += blockDim.x) {
    for (int b = 0; b < Q; ++b) {
      double t = Tp[static_cast<size_t>(c) * Q * Q + ap * Q + b];
      for (int m = 0; m < b; ++m) t -= T[ap * Q + m] * Lc[b + m * Q];
      T[ap * Q + b] = t / Lc[b + b * Q];
    }
  }
  __syncthreads();
  const double* Pc = P + static_cast<size_t>(c) * U * dim;
  const double* Rc = R + static_cast<size_t>(c) * QP * (n + Q);
  for (int o = tid; o < q * dim; o += blockDim.x) {
    const int p = o / dim, d = o % dim;
    double t1;
    if (G1 != nullptr) {
      t1 = G1[(static_cast<size_t>(c) * q + p) * dim + d];
    } else {
      const double* xu = Xu + (static_cast<size_t>(c) * U + p) * (DIMP + 2);
      t1 = spec.inv_len[d] * (Gu[(static_cast<size_t>(c) * U + p) * DIMP + d] - xu[d] * GkB[static_cast<size_t>(c) * U + p]);
    }
    const double* pp = Pc + p * dim;
    double t2 = 0.0;
    for (int j = 0; j < N; ++j) {
      const double* xj = X + static_cast<size_t>(j) * dim;
      const KParts kp = kernel_parts(spec, weighted_sqdist(spec, pp, xj));
      for (int m = 0; m < b1; ++m) {
        const double* kr = Rc + static_cast<size_t>(p * b1 + m) * (n + Q);  // (K^-1 R)[:, (p, m)]
        for (int cc = 0; cc < b1; ++cc)
          t2 += grad_cov_entry(spec, kp, pp, xj, row_type(m, spec.derivs), row_type(cc, spec.derivs), d) * kr[j * b1 + cc];
      }
    }
    const double* G = gchol + (static_cast<size_t>(c) * q + p) * Q * Q * dim;
    double t3 = 0.0;
    for (int a = 0; a < Q; ++a)
      for (int b = 0; b <= a; ++b) t3 += G[(static_cast<size_t>(a) * Q + b) * dim + d] * T[a * Q + b];
    double g = -(t1 - t2 - t3) / static_cast<double>(num_mc);
    if (winner[c] == p) g += gmu[(static_cast<size_t>(c) * q * b1 + p * b1) * dim + d];
    grad[(static_cast<size_t>(c) * q + p) * dim + d] = g;
  }
}

__global__ void mean_of_points_kernel(int n, int num, double mean, const double* __restrict__ Kcols,
                                      const double* __restrict__ beta, double* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= num) return;
  const double* k = Kcols + static_cast<size_t>(j) * n;
  double t = 0.0;
  for (int r = 0; r < n; ++r) t += k[r] * beta[r];
  out[j] = mean + t;
}

}  // namespace

void drop_cached_plan(const cmoe_gp* gp) {
  if (gp->cached_plan) {
    cmoe_kg_plan_destroy(gp->cached_plan);
    gp->cached_plan = nullptr;
  }
}

bool register_kg_entries(std::initializer_list<KgDispatchEntry> entries) {
  kg_table().insert(kg_table().end(), entries);
  return true;
}

const KgDispatchEntry* find_kg_entry(int kernel, int dim, int Q, int g) {
  const bool need_gen = g > 0, wide = g > kMaxG;
  const KgDispatchEntry* best = nullptr;
  for (const auto& e : kg_table()) {
    if (e.kernel != kernel || e.dim < dim || e.qp < Q) continue;
    if (e.wide != wide) continue;
    if (need_gen && !e.gen) continue;
    if (!best || e.dim < best->dim || (e.dim == best->dim && e.qp < best->qp)) best = &e;
  }
  return best;
}

namespace {
std::vector<KgLargeEntry>& kg_large_table() {
  static std::vector<KgLargeEntry> t;
  return t;
}
}  // namespace

bool register_kg_large_entries(std::initializer_list<KgLargeEntry> entries) {
  kg_large_table().insert(kg_large_table().end(), entries);
  return true;
}

const KgLargeEntry* find_kg_large_entry(int kernel, int dim, int g) {
  const bool wide = g > kMaxG;
  const KgLargeEntry* best = nullptr;
  for (const auto& e : kg_large_table()) {
    if (e.kernel != kernel || e.dim < dim || e.wide != wide) continue;
    if (!best || e.dim < best->dim) best = &e;
  }
  return best;
}

void build_union_sets(const double* cand, const double* Xp, int nc, int q, int p, int dim, double* P, cudaStream_t s) {
  const size_t tot = static_cast<size_t>(nc) * (q + p) * dim;
  build_union_kernel<<<static_cast<unsigned>((tot + 255) / 256), 256, 0, s>>>(cand, Xp, nc, q, p, dim, P);
  count_launch();
}

void kg_check_inner(const KernelSpec& spec, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds) {
  CMOE_REQUIRE(num_fidelity >= 0 && num_fidelity < spec.dim, CMOE_ERR_BOUNDS, "num_fidelity out of range");
  CMOE_REQUIRE(spec.g <= kMaxGWide, CMOE_ERR_BOUNDS, "at most 31 derivative observations per point in the q-KG kernel");
  if (spec.g > kMaxG) {
    // the wide kernel visits the derivative rows by coordinate (KgMcParams::drow)
    for (int a = 0; a < spec.g; ++a)
      for (int b = 0; b < a; ++b)
        CMOE_REQUIRE(spec.derivs[a] != spec.derivs[b], CMOE_ERR_BOUNDS,
                     "a partial derivative is observed twice per point (q-KG with more than 8 derivative observations)");
  }
  CMOE_REQUIRE(inner->max_num_steps <= 4096, CMOE_ERR_BOUNDS, "inner max_num_steps must be <= 4096");
  for (int d = 0; d < spec.dim - num_fidelity; ++d)
    CMOE_REQUIRE(inner_bounds[2 * d] <= inner_bounds[2 * d + 1], CMOE_ERR_BOUNDS, "Tensor product region is EMPTY.");
}

KgMcParams kg_inner_params(const cmoe_gp& gp, int ps, int M, int num_mc, const cmoe_gd_params& inner,
                           const double* inner_bounds, const double* alpha0) {
  const KernelSpec& spec = gp.spec;
  const int dim = spec.dim;
  KgMcParams m{};
  m.ps = ps;
  m.dim = dim;
  m.M = M;
  m.num_mc = num_mc;
  m.g = spec.g;
  for (int k = 0; k < CMOE_MAX_DIM; ++k) m.derivs[k] = (k < spec.g) ? spec.derivs[k] : 0;
  for (int k = 0; k < spec.g; ++k) m.drow[spec.derivs[k]] = 1 + k;
  m.max_steps = inner.max_num_steps;
  m.max_restarts = inner.max_num_restarts;
  m.mean = gp.mean;
  m.mrc = inner.max_relative_change;
  m.tol = inner.tolerance;
  m.step_tol = inner.max_num_steps > 0 ? inner.tolerance / static_cast<double>(inner.max_num_steps) : 0.0;
  m.alpha = spec.alpha;
  m.alpha0 = alpha0;
  for (int d = 0; d < CMOE_MAX_DIM; ++d) {
    m.lo[d] = -1.0e300;
    m.hi[d] = 1.0e300;
    m.inv_len[d] = (d < dim) ? spec.inv_len[d] : 0.0;
  }
  for (int d = 0; d < ps; ++d) {  // the frame of A (kg_pack_kernel, kgl_pack_kernel)
    m.lo[d] = inner_bounds[2 * d] - gp.centre[d];
    m.hi[d] = inner_bounds[2 * d + 1] - gp.centre[d];
  }
  return m;
}

std::vector<double> kg_step_sizes(const cmoe_gd_params& inner) {
  std::vector<double> a0(std::max(1, inner.max_num_steps));
  for (int i = 0; i < inner.max_num_steps; ++i) a0[i] = gd_step_size(inner.pre_mult, inner.gamma, i);
  return a0;
}

std::vector<double> kg_pinned_discrete(const double* discrete_pts, int num_pts, int ps, int dim) {
  std::vector<double> hD(static_cast<size_t>(std::max(1, num_pts)) * dim, 1.0);
  for (int j = 0; j < num_pts; ++j)
    for (int d = 0; d < ps; ++d) hD[static_cast<size_t>(j) * dim + d] = discrete_pts[static_cast<size_t>(j) * ps + d];
  return hD;
}

int kg_samples_per_item(long long candidates, int num_mc, int sms, int ctas_per_sm) {
  const long long target_ctas = 8LL * sms * ctas_per_sm;
  long long chunk = (candidates * num_mc + target_ctas - 1) / target_ctas;
  chunk = std::max<long long>(2 * kMcThreads, std::min<long long>(chunk, 16 * kMcThreads));
  chunk = (chunk + kMcThreads - 1) / kMcThreads * kMcThreads;
  return static_cast<int>(std::min<long long>(chunk, (num_mc + kMcThreads - 1) / kMcThreads * kMcThreads));
}

void kg_value(int nb, int num_mc, const double* outVal, const double* best_post, const int* fail, double* kg,
              cudaStream_t s) {
  kg_value_kernel<<<nb, 256, 0, s>>>(num_mc, outVal, best_post, fail, kg);
  count_launch();
}

void kg_fill_points(const KernelSpec& spec, const Centre& ctr, int samples, int DIMP, double* outX, double* outH,
                    cudaStream_t s) {
  kg_fill_point_kernel<<<(samples + 255) / 256, 256, 0, s>>>(spec, ctr, samples, DIMP, outX, outH);
  count_launch();
}

void kg_tprime(int nb, int n, int Q, int QP, const double* R, const double* B, double* Tp, cudaStream_t s) {
  kg_tprime_kernel<<<nb, 256, 0, s>>>(n, Q, QP, R, B, Tp);
  count_launch();
}

void kg_g1(const KernelSpec& spec, const Centre& ctr, int nb, int U, int q, int QP, int DIMP, int num_mc,
           const double* P, const double* recC, const double* outX, double* G1, cudaStream_t s) {
  kg_g1_kernel<<<nb, 256, 0, s>>>(spec, ctr, U, q, QP, DIMP, num_mc, P, recC, outX, G1);
  count_launch();
}

}  // namespace cmoe

using namespace cmoe;  // NOLINT

// -----------------------------------------------------------------------------------------------------------------
// the device-resident plan
// -----------------------------------------------------------------------------------------------------------------
struct cmoe_kg_plan {
  const cmoe_gp* gp = nullptr;
  uint64_t gp_generation = 0;  // the fit this plan's workspace was sized for
  int nf = 0, num_pts = 0, max_cand = 0, q = 0, p = 0, U = 0, num_mc = 0, ps = 0, M = 0;
  bool want_grad = false;
  double best_so_far = 0.0;
  uint64_t seed = 0;
  cmoe_gd_params inner{};
  std::vector<double> h_inner_bounds, h_discrete, h_Xp;  // host copies (cache key of cmoe_kg_eval)
  KgSelect select = nullptr;  // the instantiation's kg_select
  KgPath path{};              // its builds for this shape, re-selected per upload (the candidates' radius)
  int DIMP = 0, QP = 0, batch = 0, nc = 0;
  int Q = 0, stride = 0;  // rows of the union block U*(1+g); doubles per training point in the operand pack
  double rmax_static = 0.0;   // max scaled norm of training / pending / discrete points (see kFastPathRadius)
  int chunk = 0;
  // static device data
  DevBuf<double> dXt, dD, dKD, dMuD, dAlpha0, dTable, dXp, dCand, dStale;
  KgMcParams mcp{};
  // per-batch device scratch
  PosteriorBatch pb;
  DevBuf<double> dPk, dXu, dA, dAfull, dKAu, dW, dMuA, dBestPost, dRecC, dOutVal, dOutX, dOutH, dR, dGu, dGkB, dTp, dG1;
  DevBuf<int> dWinner, dRecStart, dWork;
  DevBuf<double> dWt, dAw;  // general path: weight table per candidate, per-lane weight columns per resident CTA
  DevBuf<double> dStart;    // g == 0: start-point table [batch][M][1+QP][DIMP+2] (kg_start_kernel)
  int aw_slots = 0;
  DevBuf<unsigned long long> dStats;
  // results
  DevBuf<double> dKG, dGrad;
  DevBuf<int> dFailAll;
  EventTimer t_total, t_mc;
  double mc_ms_accum = 0.0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> mc_events;
  int launches = 0;
  ~cmoe_kg_plan() {
    for (auto& e : mc_events) {
      cudaEventDestroy(e.first);
      cudaEventDestroy(e.second);
    }
  }
};

namespace {

// |(x - centre) / l|: a point's distance from the origin of the MC kernels' frame, in length scales
double centred_radius(const cmoe_gp& gp, const double* x, int nd) {
  double r2 = 0.0;
  for (int d = 0; d < nd; ++d) {
    const double v = (x[d] - gp.centre[d]) * gp.spec.inv_len[d];
    r2 += v * v;
  }
  return std::sqrt(r2);
}

void plan_run_batch(cmoe_kg_plan& pl, int c0, int nb, size_t ev_idx) {
  const cmoe_gp& gp = *pl.gp;
  const KernelSpec& spec = gp.spec;
  cudaStream_t s = gp.stream;
  const int N = gp.N, n = gp.n, dim = spec.dim, U = pl.U, q = pl.q, p = pl.p, M = pl.M, QP = pl.QP, DIMP = pl.DIMP;
  const int mc = pl.num_mc, Q = pl.Q;
  const bool gen = spec.g > 0;
  const Centre ctr = centre_of(gp);
  PosteriorBatch& pb = pl.pb;
  pb.configure(gp, nb, U, spec.derivs, spec.g, pl.want_grad ? q : 0, s);
  build_union_sets(pl.dCand.p + static_cast<size_t>(c0) * q * dim, pl.dXp.p, nb, q, p, dim, pb.P.p, s);
  pb.run(gp, /*diag_mode=*/2, /*want_chol=*/true, pl.want_grad, s);
  CMOE_CUDA(cudaMemcpyAsync(pl.dFailAll.p + c0, pb.fail.p, nb * sizeof(int), cudaMemcpyDeviceToDevice, s));

  kg_pack_kernel<<<nb, 256, 0, s>>>(spec, ctr, N, U, pl.ps, pl.num_pts, DIMP, QP, pl.stride, pl.dXt.p, gp.dKinvY.p, pb.B.p, pb.P.p,
                                    pl.dD.p, pl.dPk.p, pl.dXu.p, pl.dA.p, pl.dAfull.p,
                                    pl.dStale.count ? pl.dStale.p : nullptr, q, gen ? pl.dWt.p : nullptr);
  count_launch();
  if (!gen) {
    kg_start_kernel<<<dim3(M, nb), kStartThreads, 0, s>>>(spec, N, U, M, DIMP, QP, pl.path.use_smem ? 1 : 0, pl.dXt.p,
                                                         pl.dPk.p, pl.dXu.p, pl.dA.p, pl.dStart.p);
    count_launch();
  }
  // K(X, A_union) for all candidates of the batch (value rows only)
  build_mix_covariance(spec, gp.dX.p, N, pl.dAfull.p, nb * U, nullptr, 0, pl.dKAu.p, s);
  const size_t smem_d = static_cast<size_t>(Q) * Q * sizeof(double);
  kg_discrete_kernel<<<nb, 256, smem_d, s>>>(spec, n, U, pl.num_pts, QP, gp.mean, pl.best_so_far, gp.dKinvY.p, pb.P.p,
                                             pl.dAfull.p, pl.dD.p, pl.dKAu.p, pl.dKD.p, pl.dMuD.p, pb.B.p, pb.mu.p,
                                             pb.chol.p, pb.fail.p, pl.dW.p, pl.dMuA.p, pl.dBestPost.p, pl.dWinner.p);
  count_launch();
  const size_t w_bytes = (static_cast<size_t>(M) * QP + M) * sizeof(double);
  const int w_in_smem = (w_bytes + smem_d) <= 160 * 1024;
  const size_t smem_p = smem_d + (w_in_smem ? w_bytes : 0);
  CMOE_CUDA(cudaFuncSetAttribute(kg_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 180 * 1024));
  kg_prep_kernel<<<dim3((mc + 255) / 256, nb), 256, smem_p, s>>>(Q, M, QP, mc, pl.seed,
                                                                 pl.dTable.count ? pl.dTable.p : nullptr, pb.chol.p,
                                                                 pl.dW.p, pl.dMuA.p, pb.fail.p, w_in_smem, pl.dRecC.p,
                                                                 pl.dRecStart.p);
  count_launch();

  KgMcParams prm = pl.mcp;
  prm.Pk = pl.dPk.p;
  prm.Xu = pl.dXu.p;
  prm.A = pl.dA.p;
  prm.recC = pl.dRecC.p;
  prm.recStart = pl.dRecStart.p;
  prm.Start = gen ? nullptr : pl.dStart.p;
  prm.outVal = pl.dOutVal.p;
  prm.outX = pl.dOutX.p;
  prm.outH = pl.dOutH.p;
  prm.stats = pl.dStats.p;
  const int chunks = (mc + pl.chunk - 1) / pl.chunk;
  if (gen) {
    prm.Wt = pl.dWt.p;
    prm.aw = pl.dAw.p;
    prm.work = pl.dWork.p;
    prm.aw_slots = pl.aw_slots;
    prm.chunks = chunks;
    prm.work_total = chunks * nb;
    CMOE_CUDA(cudaMemsetAsync(pl.dWork.p, 0, sizeof(int), s));
  }
  cudaEventRecord(pl.mc_events[ev_idx].first, s);
  pl.path.mc(prm, chunks, nb, s);
  cudaEventRecord(pl.mc_events[ev_idx].second, s);
  count_launch();
  if (pl.inner.max_num_restarts <= 0) {
    kg_fill_point_kernel<<<(nb * mc + 255) / 256, 256, 0, s>>>(spec, ctr, nb * mc, DIMP, pl.dOutX.p, pl.dOutH.p);
    count_launch();
  }
  kg_value_kernel<<<nb, 256, 0, s>>>(mc, pl.dOutVal.p, pl.dBestPost.p, pb.fail.p, pl.dKG.p + c0);
  count_launch();

  if (pl.want_grad) {
    KgAccParams ap{};
    ap.N = N;
    ap.U = U;
    ap.dim = dim;
    ap.num_mc = mc;
    ap.alpha = spec.alpha;
    ap.Xt = pl.dXt.p;
    ap.Xu = pl.dXu.p;
    ap.recC = pl.dRecC.p;
    ap.outX = pl.dOutX.p;
    ap.outH = pl.dOutH.p;
    ap.fast_exp = pl.path.use_smem ? 1 : 0;
    ap.g = spec.g;
    for (int k = 0; k < CMOE_MAX_DIM; ++k) ap.derivs[k] = (k < spec.g) ? spec.derivs[k] : 0;
    for (int d = 0; d < CMOE_MAX_DIM; ++d) ap.inv_len[d] = (d < dim) ? spec.inv_len[d] : 0.0;
    ap.R = pl.dR.p;
    ap.Gu = pl.dGu.p;
    ap.GkB = pl.dGkB.p;
    CMOE_CUDA(cudaMemsetAsync(pl.dR.p, 0, static_cast<size_t>(nb) * QP * (n + Q) * sizeof(double), s));
    pl.path.acc(ap, nb, s);
    if (gen) {
      kg_g1_kernel<<<nb, 256, 0, s>>>(spec, ctr, U, q, QP, DIMP, mc, pb.P.p, pl.dRecC.p, pl.dOutX.p, pl.dG1.p);
      count_launch();
    }
    kg_tprime_kernel<<<nb, 256, 0, s>>>(n, Q, QP, pl.dR.p, pb.B.p, pl.dTp.p);
    count_launch(2);
    // K^-1 R: columns of length n with stride n+Q, nb*QP of them
    potrs_lower(gp.dK.p, n, pl.dR.p, n + Q, nb * QP, s);
    kg_grad_kernel<<<nb, 128, static_cast<size_t>(Q) * Q * sizeof(double), s>>>(
        spec, N, U, q, QP, DIMP, mc, gp.dX.p, pb.P.p, pl.dXu.p, pl.dR.p, pl.dTp.p, pl.dGu.p, pl.dGkB.p,
        gen ? pl.dG1.p : nullptr, pb.chol.p, pb.gchol.p, pb.gmu.p, pl.dWinner.p, pb.fail.p,
        pl.dGrad.p + static_cast<size_t>(c0) * q * dim);
    count_launch();
  }
  CMOE_CUDA(cudaGetLastError());
}

}  // namespace

extern "C" {

int cmoe_kg_plan_create(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds,
                        const double* discrete_pts, int num_pts, int max_candidates, int q,
                        const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                        int want_grad, cmoe_kg_plan** plan_out) {
  if (plan_out) *plan_out = nullptr;
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(plan_out != nullptr, CMOE_ERR_INVALID_VALUE, "plan_out is NULL");
    CMOE_REQUIRE(max_candidates >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    CMOE_REQUIRE(q >= 1 && p >= 0 && num_mc >= 1 && num_pts >= 0, CMOE_ERR_BOUNDS, "bad sizes");
    const KernelSpec& spec = gp->spec;
    const int dim = spec.dim;
    kg_check_inner(spec, num_fidelity, inner, inner_bounds);
    require_device(gp->device);
    std::unique_ptr<cmoe_kg_plan> pl(new cmoe_kg_plan());
    pl->gp = gp;
    pl->gp_generation = gp->generation;
    pl->nf = num_fidelity;
    pl->num_pts = num_pts;
    pl->max_cand = max_candidates;
    pl->q = q;
    pl->p = p;
    pl->U = q + p;
    pl->num_mc = num_mc;
    pl->ps = dim - num_fidelity;
    pl->M = pl->U + num_pts;
    pl->want_grad = want_grad != 0;
    pl->best_so_far = best_so_far;
    pl->seed = seed;
    pl->inner = *inner;
    pl->h_inner_bounds.assign(inner_bounds, inner_bounds + 2 * static_cast<size_t>(pl->ps));
    pl->h_discrete.assign(discrete_pts, discrete_pts + static_cast<size_t>(num_pts) * pl->ps);
    if (p) pl->h_Xp.assign(points_being_sampled, points_being_sampled + static_cast<size_t>(p) * dim);
    const int U = pl->U, N = gp->N, n = gp->n, ps = pl->ps;
    pl->Q = pl->U * (1 + spec.g);
    const KgDispatchEntry* entry = find_kg_entry(spec.kernel, dim, pl->Q, spec.g);
    CMOE_REQUIRE(entry != nullptr, CMOE_ERR_BOUNDS,
                 "(q+p)*(1+num_derivatives) or dim exceeds the largest compiled q-KG kernel (" CMOE_STR(CMOE_MAX_KG_ROWS)
                 " rows, 32 dims)");
    pl->select = entry->select;
    pl->DIMP = entry->dim;
    pl->QP = entry->qp;
    const int DIMP = pl->DIMP, QP = pl->QP, Q = pl->Q;
    pl->stride = spec.g > 0 ? 2 : QP + 2;
    cudaStream_t s = gp->stream;

    // static data: scaled training points, discrete set (full dim, fidelity coords = 1), K(X, D), mu_n(D)
    pl->dXt.alloc(static_cast<size_t>(N) * DIMP);
    const Centre ctr = centre_of(*gp);
    pack_xt_kernel<<<(N * DIMP + 255) / 256, 256, 0, s>>>(spec, ctr, gp->dX.p, N, DIMP, pl->dXt.p);
    const std::vector<double> hD = kg_pinned_discrete(discrete_pts, num_pts, ps, dim);
    pl->dD.upload(hD.data(), hD.size(), s);
    pl->dKD.alloc(static_cast<size_t>(n) * std::max(1, num_pts));
    pl->dMuD.alloc(std::max(1, num_pts));
    if (num_pts > 0) {
      build_mix_covariance(spec, gp->dX.p, N, pl->dD.p, num_pts, nullptr, 0, pl->dKD.p, s);
      mean_of_points_kernel<<<(num_pts + 127) / 128, 128, 0, s>>>(n, num_pts, gp->mean, pl->dKD.p, gp->dKinvY.p,
                                                                  pl->dMuD.p);
    }
    const std::vector<double> a0 = kg_step_sizes(*inner);
    pl->dAlpha0.upload(a0.data(), a0.size(), s);
    std::vector<double> hXp(static_cast<size_t>(std::max(1, p)) * dim, 0.0);
    if (p) std::copy(points_being_sampled, points_being_sampled + static_cast<size_t>(p) * dim, hXp.begin());
    pl->dXp.upload(hXp.data(), hXp.size(), s);
    pl->dCand.alloc(static_cast<size_t>(max_candidates) * q * dim);
    CMOE_CUDA(cudaStreamSynchronize(s));

    // work decomposition
    const int sms = sm_count();
    {
      // The shared-memory fast path evaluates exp without per-call range guards; that is valid while every scaled
      // coordinate vector it can meet lies within kFastPathRadius length scales of the origin of the kernels' frame,
      // the GP's centre (kg_mc.cuh).
      auto upd = [&](const double* pts, size_t count, int stride, int nd) {
        for (size_t i = 0; i < count; ++i)
          pl->rmax_static = std::max(pl->rmax_static, centred_radius(*gp, pts + i * stride, nd));
      };
      upd(gp->hX.data(), N, dim, dim);
      upd(hD.data(), num_pts, dim, dim);
      if (p) upd(hXp.data(), p, dim, dim);
      // the inner optimiser keeps its iterates inside the inner domain; their fidelity coordinates stay at 1.0
      double r2 = 0.0;
      for (int d = 0; d < dim; ++d) {
        const double lo = d < ps ? inner_bounds[2 * d] : 1.0, hi = d < ps ? inner_bounds[2 * d + 1] : 1.0;
        const double c = std::max(std::fabs(lo - gp->centre[d]), std::fabs(hi - gp->centre[d])) * spec.inv_len[d];
        r2 += c * c;
      }
      pl->rmax_static = std::max(pl->rmax_static, std::sqrt(r2));
    }
    pl->path = pl->select(N, U, spec.g, pl->rmax_static < kFastPathRadius);
    // candidates per batch bounded by ~3 GiB of per-sample records and start-point tables, and by grid.y of the
    // per-candidate launches (kg_start_kernel, kg_prep_kernel, the MC and accumulation kernels)
    const size_t per_cand = static_cast<size_t>(num_mc) * (QP + DIMP + 2) * sizeof(double) +
                            static_cast<size_t>(n) * Q * 4 * sizeof(double) +
                            (spec.g == 0 ? static_cast<size_t>(pl->M) * (1 + QP) * (DIMP + 2) * sizeof(double) : 0);
    pl->batch = static_cast<int>(chunk_items(max_candidates, size_t(3) << 30, per_cand, kMaxGridY));
    // a wave is the selected path's residency (kg_select; 2 CTAs per SM for the tile instantiation at the bench shape)
    pl->chunk = kg_samples_per_item(pl->batch, num_mc, sms, pl->path.ctas_per_sm);
    const int B = pl->batch;
    pl->dPk.alloc(static_cast<size_t>(B) * N * pl->stride);
    pl->dXu.alloc(static_cast<size_t>(B) * U * (DIMP + 2));
    pl->dA.alloc(static_cast<size_t>(B) * pl->M * DIMP);
    pl->dAfull.alloc(static_cast<size_t>(B) * U * dim);
    pl->dKAu.alloc(static_cast<size_t>(B) * U * n);
    pl->dW.alloc(static_cast<size_t>(B) * pl->M * QP);
    pl->dMuA.alloc(static_cast<size_t>(B) * pl->M);
    pl->dBestPost.alloc(B);
    pl->dWinner.alloc(B);
    pl->dRecC.alloc(static_cast<size_t>(B) * num_mc * QP);
    pl->dRecStart.alloc(static_cast<size_t>(B) * num_mc);
    pl->dOutVal.alloc(static_cast<size_t>(B) * num_mc);
    pl->dOutX.alloc(static_cast<size_t>(B) * num_mc * DIMP);
    pl->dOutH.alloc(static_cast<size_t>(B) * num_mc);
    pl->dStats.alloc(4);
    if (spec.g > 0) {
      // one scratch slot (N(1+g) rows x kMcThreads lanes) per resident CTA, at most 3 per SM and ~6 GiB in total
      const size_t slot = static_cast<size_t>(n) * kMcThreads;
      pl->aw_slots = static_cast<int>(std::max<size_t>(1, std::min<size_t>(3 * static_cast<size_t>(sms),
                                                                            (size_t(6) << 30) / (slot * sizeof(double)))));
      pl->dAw.alloc(slot * pl->aw_slots);
      pl->dWt.alloc(static_cast<size_t>(B) * (1 + QP) * n);
      pl->dWork.alloc(1);
    } else {
      pl->dStart.alloc(static_cast<size_t>(B) * pl->M * (1 + QP) * (DIMP + 2));
    }
    if (pl->want_grad) {
      pl->dR.alloc(static_cast<size_t>(B) * QP * (n + Q));
      pl->dGu.alloc(static_cast<size_t>(B) * U * DIMP);
      pl->dGkB.alloc(static_cast<size_t>(B) * U);
      pl->dTp.alloc(static_cast<size_t>(B) * Q * Q);
      pl->dG1.alloc(static_cast<size_t>(B) * q * dim);
    }
    pl->dKG.alloc(max_candidates);
    pl->dGrad.alloc(pl->want_grad ? static_cast<size_t>(max_candidates) * q * dim : 1);
    pl->dFailAll.alloc(max_candidates);
    const int nbatches = (max_candidates + B - 1) / B;
    pl->mc_events.resize(nbatches);
    for (auto& e : pl->mc_events) {
      cudaEventCreate(&e.first);
      cudaEventCreate(&e.second);
    }

    KgMcParams& m = pl->mcp;
    m = kg_inner_params(*gp, ps, pl->M, num_mc, *inner, inner_bounds, pl->dAlpha0.p);
    m.N = N;
    m.U = U;
    m.chunk = pl->chunk;
    m.use_smem = pl->path.use_smem ? 1 : 0;
    m.Q = Q;
    m.pk_stride = pl->stride;
    // general path: park the scaled training points + e_j behind the weight ring when they are small enough to leave room
    // for two CTAs per SM (2 x (90 KB ring + 20 KB) < 227 KB)
    m.stage_ops = (spec.g > 0 && static_cast<size_t>(N) * (DIMP + 2) * sizeof(double) <= 20 * 1024) ? 1 : 0;
    if (const char* e = std::getenv("CMOE_GEN_STAGE")) m.stage_ops = m.stage_ops && std::atoi(e) != 0;
    m.Xt = pl->dXt.p;
    *plan_out = pl.release();
  });
}

void cmoe_kg_plan_destroy(cmoe_kg_plan* plan) {
  if (!plan) return;
  cudaSetDevice(plan->gp->device);
  delete plan;
}

int cmoe_kg_plan_set_table(cmoe_kg_plan* plan, const double* table, int table_len) {
  return guarded(nullptr, [&] {
    require_device(plan->gp->device);
    const int need = ((plan->num_mc + 1) / 2) * plan->Q;
    CMOE_REQUIRE(table_len >= need, CMOE_ERR_INVALID_VALUE, "All random numbers stored in the RNG have been used up!");
    plan->dTable.upload(table, table_len, plan->gp->stream);
    CMOE_CUDA(cudaStreamSynchronize(plan->gp->stream));
  });
}

int cmoe_kg_plan_set_stale_union(cmoe_kg_plan* plan, const double* points_to_sample) {
  return guarded(nullptr, [&] {
    require_device(plan->gp->device);
    if (points_to_sample == nullptr) {
      plan->dStale.release();
      return;
    }
    plan->dStale.upload(points_to_sample, static_cast<size_t>(plan->q) * plan->gp->spec.dim, plan->gp->stream);
    CMOE_CUDA(cudaStreamSynchronize(plan->gp->stream));
  });
}

int cmoe_kg_plan_upload(cmoe_kg_plan* plan, const double* candidates, int num_candidates) {
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(num_candidates >= 1 && num_candidates <= plan->max_cand, CMOE_ERR_BOUNDS,
                 "num_candidates exceeds the plan capacity");
    CMOE_REQUIRE(plan->gp_generation == plan->gp->generation, CMOE_ERR_INVALID_VALUE,
                 "the GaussianProcess was refitted after this plan was created; create a new plan");
    require_device(plan->gp->device);
    plan->nc = num_candidates;
    {
      const KernelSpec& spec = plan->gp->spec;
      double rmax = plan->rmax_static;
      const size_t pts = static_cast<size_t>(num_candidates) * plan->q;
      for (size_t i = 0; i < pts && rmax < kFastPathRadius; ++i)
        rmax = std::max(rmax, centred_radius(*plan->gp, candidates + i * spec.dim, spec.dim));
      // NaN-safe: a NaN norm fails the comparison
      plan->path = plan->select(plan->gp->N, plan->U, spec.g, rmax < kFastPathRadius);
      plan->mcp.use_smem = plan->path.use_smem ? 1 : 0;
    }
    plan->dCand.upload(candidates, static_cast<size_t>(num_candidates) * plan->q * plan->gp->spec.dim,
                       plan->gp->stream);
  });
}

int cmoe_kg_plan_run(cmoe_kg_plan* plan) {
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(plan->nc >= 1, CMOE_ERR_INVALID_VALUE, "no candidates uploaded");
    CMOE_REQUIRE(plan->gp_generation == plan->gp->generation, CMOE_ERR_INVALID_VALUE,
                 "the GaussianProcess was refitted after this plan was created; create a new plan");
    require_device(plan->gp->device);
    cudaStream_t s = plan->gp->stream;
    const int l0 = launches_issued();
    plan->t_total.start(s);
    CMOE_CUDA(cudaMemsetAsync(plan->dStats.p, 0, 4 * sizeof(unsigned long long), s));
    size_t ev = 0;
    for (int c0 = 0; c0 < plan->nc; c0 += plan->batch, ++ev)
      plan_run_batch(*plan, c0, std::min(plan->batch, plan->nc - c0), ev);
    plan->t_total.stop(s);
    plan->launches = launches_issued() - l0;
  });
}

int cmoe_kg_plan_sync(cmoe_kg_plan* plan, int* info) {
  return guarded(info, [&] {
    require_device(plan->gp->device);
    cudaStream_t s = plan->gp->stream;
    std::vector<int> f(plan->nc);
    plan->dFailAll.download(f.data(), plan->nc, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    for (int c = 0; c < plan->nc; ++c)
      if (f[c] != 0) throw_singular_union(f[c]);
  });
}

int cmoe_kg_plan_download(cmoe_kg_plan* plan, double* kg, double* grad_kg, cmoe_kg_stats* stats) {
  return guarded(nullptr, [&] {
    require_device(plan->gp->device);
    cudaStream_t s = plan->gp->stream;
    if (kg) plan->dKG.download(kg, plan->nc, s);
    if (grad_kg) {
      CMOE_REQUIRE(plan->want_grad, CMOE_ERR_INVALID_VALUE, "plan was created without gradients");
      plan->dGrad.download(grad_kg, static_cast<size_t>(plan->nc) * plan->q * plan->gp->spec.dim, s);
    }
    unsigned long long st[4] = {0, 0, 0, 0};
    if (stats) CMOE_CUDA(cudaMemcpyAsync(st, plan->dStats.p, sizeof(st), cudaMemcpyDeviceToHost, s));
    CMOE_CUDA(cudaStreamSynchronize(s));
    if (stats) {
      stats->mc_samples = static_cast<uint64_t>(plan->nc) * plan->num_mc;
      stats->posterior_evals = st[0];
      stats->line_search_steps = st[1];
      stats->point_evals = st[2];
      stats->line_batches = st[3];
    }
  });
}

int cmoe_kg_plan_timings(const cmoe_kg_plan* plan, double* total_ms, double* mc_kernel_ms, int* launches) {
  return guarded(nullptr, [&] {
    require_device(plan->gp->device);
    cmoe_kg_plan* pl = const_cast<cmoe_kg_plan*>(plan);
    if (total_ms) *total_ms = pl->t_total.ms();
    if (mc_kernel_ms) {
      double t = 0.0;
      const int nbatches = (plan->nc + plan->batch - 1) / plan->batch;
      for (int b = 0; b < nbatches; ++b) {
        float ms = 0.f;
        cudaEventSynchronize(pl->mc_events[b].second);
        cudaEventElapsedTime(&ms, pl->mc_events[b].first, pl->mc_events[b].second);
        t += ms;
      }
      *mc_kernel_ms = t;
    }
    if (launches) *launches = plan->launches;
  });
}

int cmoe_kg_eval(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds,
                 const double* discrete_pts, int num_pts, const double* candidates, int num_candidates, int q,
                 const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                 const double* normals_table, double* kg, double* grad_kg, cmoe_kg_stats* stats, int* info) {
  // Reuse the GP's cached plan when the configuration matches (same discrete set, bounds, inner optimiser, sizes);
  // best_so_far and the seed are plain parameters and are refreshed in place.
  const int ps = gp->spec.dim - num_fidelity, dim = gp->spec.dim;
  cmoe_kg_plan* plan = gp->cached_plan;
  const bool want_grad = grad_kg != nullptr;
  bool reuse = plan != nullptr && num_fidelity >= 0 && ps >= 1 && plan->nf == num_fidelity &&
               plan->num_pts == num_pts && plan->q == q && plan->p == p && plan->num_mc == num_mc &&
               plan->want_grad == want_grad && plan->max_cand >= num_candidates &&
               std::memcmp(&plan->inner, inner, sizeof(cmoe_gd_params)) == 0 &&
               std::equal(plan->h_inner_bounds.begin(), plan->h_inner_bounds.end(), inner_bounds) &&
               std::equal(plan->h_discrete.begin(), plan->h_discrete.end(), discrete_pts) &&
               (p == 0 || std::equal(plan->h_Xp.begin(), plan->h_Xp.end(), points_being_sampled));
  int rc = CMOE_OK;
  if (!reuse) {
    drop_cached_plan(gp);
    plan = nullptr;
    rc = cmoe_kg_plan_create(gp, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, num_candidates, q,
                             points_being_sampled, p, num_mc, best_so_far, seed, want_grad ? 1 : 0, &plan);
    if (rc != CMOE_OK) return rc;
    gp->cached_plan = plan;
  } else {
    plan->best_so_far = best_so_far;
    plan->seed = seed;
  }
  if (normals_table) {
    rc = cmoe_kg_plan_set_table(plan, normals_table, ((num_mc + 1) / 2) * (q + p) * (1 + gp->spec.g));
  } else if (plan->dTable.count) {
    plan->dTable.release();
  }
  (void)dim;
  if (rc == CMOE_OK) rc = cmoe_kg_plan_upload(plan, candidates, num_candidates);
  if (rc == CMOE_OK) rc = cmoe_kg_plan_run(plan);
  if (rc == CMOE_OK) rc = cmoe_kg_plan_sync(plan, info);
  if (rc == CMOE_OK) rc = cmoe_kg_plan_download(plan, kg, grad_kg, stats);
  return rc;
}

}  // extern "C"

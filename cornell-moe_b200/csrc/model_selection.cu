// Hyper-parameter gradient of the log marginal likelihood on the device (SURVEY.md 8f rank 2):
//   d log p / d theta_k = 1/2 tr[(a a^T - K^-1) dK/d theta_k],   a = K^-1 (y - m)
// Replaces LogMarginalLikelihoodEvaluator::ComputeGradLogLikelihood (gpp_model_selection.cpp:629-690) with the per-pair
// blocks of SquareExponential / MaternNu2p5 ::HyperparameterGradCovariance (gpp_covariance.cpp:245-317, 461-489) and
// the noise rows of BuildHyperparameterGradCovarianceMatrix (gpp_model_selection.cpp:386-444).  Python boundary:
// compute_hyperparameter_grad_log_likelihood (gpp_python_model_selection.cpp:89-140, :404).
//
// One device fit (covariance build, Cholesky, K^-1 (y - m)) with the reference's 1e-6 jitter, K^-1 by the blocked
// multi-RHS triangular solves on the identity, then ONE fused contraction kernel: a thread per point pair re-evaluates
// the (1 + dim) x (1+g) x (1+g) hyper-gradient block on the fly (dK/d theta is never materialised) and the CTA reduces
// its 1 + dim partial sums in a fixed order; the host adds the per-CTA partials in launch order.
// Quirks kept (pinned by tests/test_oracle_vs_reference.py::test_grad_log_marginal_likelihood): the Matern routine fills
// only the value-value entry of a block, returns d/d alpha = 1 at coincident points and zero length derivatives there.
//
// Log marginal likelihood at a list of hyper-parameter sets (DESIGN.md K10): EvaluateLogLikelihoodAtPointList
// (gpp_model_selection.hpp:1274-1308), Python boundary evaluate_log_likelihood_at_hyperparameter_list
// (gpp_python_model_selection.cpp:281-341).  Per chunk of sets, three steps that treat every set independently:
//   K_s = K(X, X; theta_s) + diag(noise_s + 1e-6)   lml_cov_kernel, lower 64 x 64 tiles, grid (tiles, 1, sets)
//   L_s L_s^T = K_s                                 potrf_batched (sample.cu), failure flag per set
//   -1/2 z^T z - sum log L_ii - n/2 log 2 pi,       lml_solve_kernel, one CTA per set, z = L_s^-1 (y - m)
// so a set's value does not depend on the other sets of the call or on the chunking.
//
// Value and hyper-parameter gradient at a list of sets (DESIGN.md K11): the same chunks, plus a = K_s^-1 (y - m) from
// the solve kernel, K_s^-1 = L^-T L^-1 by a blocked triangular inverse on DMMA tiles, the single call's per-pair
// contraction for every set and a fixed-order reduction per set.
#include <algorithm>
#include <cmath>
#include <limits>

#include "device_math.cuh"
#include "internal.cuh"
#include "linalg_dev.cuh"

namespace cmoe {
namespace {

__global__ void identity_kernel(double* __restrict__ A, int n) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<size_t>(n) * n) return;
  A[e] = (e / n == e % n) ? 1.0 : 0.0;
}

constexpr int kHgTx = 32, kHgTy = 8;

// The hyper-gradient block of one point pair (row point j at p1, column point i at p2): acc[h], h in [0, dim], zero on
// entry, receives sum_{m,nn} W[j*bs+m, i*bs+nn] * dK/d theta_h [j*bs+m, i*bs+nn], where Wf(row, col) returns the entry
// of W = a a^T - K^-1.  Shared by the single-set and the list contraction kernels.  kExact = false keeps the reference's
// Matern quirk; kExact = true differentiates every entry of the Matern derivative block (the SE branch is exact either
// way).  With g = 0 the two Matern branches are the same function, and the host launches the quirk build there.
template <bool kExact, class WF>
__device__ __forceinline__ void hyper_grad_pair(const KernelSpec& spec, const double* p1, const double* p2, int j, int i,
                                                const WF& Wf, double (&acc)[CMOE_MAX_DIM + 1]) {
  const int dim = spec.dim, bs = 1 + spec.g;
  const double r2 = weighted_sqdist(spec, p1, p2);
  if (kExact && spec.kernel != CMOE_KERNEL_SQUARE_EXPONENTIAL) {
    // cov_entry's block at alpha = 1, (A, B, C) of kernel_parts over alpha, u_a = (p2_a - p1_a) / l_a^2:
    //   c(0,0) = A, c(m,0) = B u_a, c(0,n) = -B u_b, c(m,n) = -C u_a u_b + [a==b] B / l_a^2
    // d/d r^2 of (A, B, C) is (-B/2, -C/2, -sqrt(5) C / (2 r)); the last multiplies only u_a u_b = O(r^2), so it is
    // taken as 0 at r = 0.  d r^2 / d l_k = -2 D_k^2 / l_k^3 and d u_a / d l_k = -2 [a==k] u_a / l_a.  Lengths enter
    // through inv_len (no division in the loops).
    const double r = sqrt(r2), arg = kSqrt5 * r, e = exp(-arg);
    const double A1 = e * (1.0 + arg + 5.0 / 3.0 * r2), B1 = 5.0 / 3.0 * e * (1.0 + arg), C1 = 25.0 / 3.0 * e;
    const double dC1 = r2 > 0.0 ? -0.5 * kSqrt5 * C1 / r : 0.0;
    for (int m = 0; m < bs; ++m) {
      const int ta = m ? spec.derivs[m - 1] : -1;
      const double ila = ta >= 0 ? spec.inv_len[ta] : 0.0;
      const double ua = (ta >= 0) ? (p2[ta] - p1[ta]) * ila * ila : 0.0;
      for (int nn = 0; nn < bs; ++nn) {
        const int tb = nn ? spec.derivs[nn - 1] : -1;
        const double ilb = tb >= 0 ? spec.inv_len[tb] : 0.0;
        const double ub = (tb >= 0) ? (p2[tb] - p1[tb]) * ilb * ilb : 0.0;
        // the entry E, and dE/d l_k = cs ds_k + ([a==k] ca + [b==k] cb) / l_k
        double E, cs, ca = 0.0, cb = 0.0;
        if (ta < 0 && tb < 0) {
          E = A1;
          cs = -0.5 * B1;
        } else if (tb < 0) {
          E = B1 * ua;
          cs = -0.5 * C1 * ua;
          ca = -2.0 * B1 * ua;
        } else if (ta < 0) {
          E = -B1 * ub;
          cs = 0.5 * C1 * ub;
          cb = 2.0 * B1 * ub;
        } else {
          E = -C1 * ua * ub;
          cs = -dC1 * ua * ub;
          ca = cb = 2.0 * C1 * ua * ub;
          if (ta == tb) {
            const double il2 = ila * ila;
            E += B1 * il2;
            cs += -0.5 * C1 * il2;
            ca += -2.0 * B1 * il2;
          }
        }
        const double W = Wf(j * bs + m, i * bs + nn);
        acc[0] = fma(W, E, acc[0]);
        const double aW = spec.alpha * W;
        for (int k = 0; k < dim; ++k) {
          const double il = spec.inv_len[k];
          const double Dl = (p1[k] - p2[k]) * il;
          double dE = cs * (-2.0 * Dl * Dl * il);
          if (ta == k) dE += ca * il;
          if (tb == k) dE += cb * il;
          acc[k + 1] = fma(aW, dE, acc[k + 1]);
        }
      }
    }
  } else if (spec.kernel != CMOE_KERNEL_SQUARE_EXPONENTIAL) {
    // value-value entry only (gpp_covariance.cpp:461-489)
    const double W = Wf(j * bs, i * bs);
    if (r2 == 0.0) {
      acc[0] = W;
    } else {
      const double arg = kSqrt5 * sqrt(r2);
      const double poly = arg + 5.0 / 3.0 * r2;
      const double e = exp(-arg);
      acc[0] = W * (1.0 + poly) * e;
      for (int k = 0; k < dim; ++k) {
        const double len = sqrt(spec.lsq[k]);
        const double dl = (p1[k] - p2[k]) / len;
        const double dr2 = -2.0 * dl * dl / len;
        const double dr = 0.5 * dr2 / sqrt(r2);
        acc[k + 1] = W * spec.alpha * e * (5.0 / 3.0 * dr2 - poly * kSqrt5 * dr);
      }
    }
  } else {
    // every entry is k * P, P in {1, u_a, -u_b, -u_a u_b + [a==b]/l_a^2}, u_a = (p2_a - p1_a)/l_a^2 (:245-317)
    const double kv = spec.alpha * exp(-0.5 * r2);
    for (int m = 0; m < bs; ++m) {
      for (int nn = 0; nn < bs; ++nn) {
        const int ta = m ? spec.derivs[m - 1] : -1, tb = nn ? spec.derivs[nn - 1] : -1;
        const double ua = (ta >= 0) ? (p2[ta] - p1[ta]) / spec.lsq[ta] : 0.0;
        const double ub = (tb >= 0) ? (p2[tb] - p1[tb]) / spec.lsq[tb] : 0.0;
        double P;
        if (ta < 0 && tb < 0) {
          P = 1.0;
        } else if (tb < 0) {
          P = ua;
        } else if (ta < 0) {
          P = -ub;
        } else {
          P = -ua * ub + ((ta == tb) ? 1.0 / spec.lsq[ta] : 0.0);
        }
        const double W = Wf(j * bs + m, i * bs + nn);
        acc[0] = fma(W, kv * P / spec.alpha, acc[0]);
        for (int k = 0; k < dim; ++k) {
          const double len = sqrt(spec.lsq[k]);
          const double D = p1[k] - p2[k];
          double dP = 0.0;
          if (ta >= 0 && tb < 0 && ta == k) dP = -2.0 * ua / len;
          if (ta < 0 && tb >= 0 && tb == k) dP = 2.0 * ub / len;
          if (ta >= 0 && tb >= 0) {
            if (ta == k) dP += 2.0 * ua * ub / len;
            if (tb == k) dP += 2.0 * ua * ub / len;
            if (ta == tb && ta == k) dP += -2.0 / (spec.lsq[ta] * len);
          }
          acc[k + 1] = fma(W, kv * P * (D / len) * (D / len) / len + kv * dP, acc[k + 1]);
        }
      }
    }
  }
}

// partial[cta][h], h in [0, dim]: 1/2 sum over this CTA's point pairs (row point j, column point i) of
//   sum_{m,nn} W[j*bs+m, i*bs+nn] * dK/d theta_h [j*bs+m, i*bs+nn]
__global__ void __launch_bounds__(kHgTx * kHgTy)
    hyper_grad_contract_kernel(const __grid_constant__ KernelSpec spec, const double* __restrict__ X, int N,
                               const double* __restrict__ a, const double* __restrict__ Kinv,
                               double* __restrict__ partial) {
  __shared__ double scratch[kHgTx * kHgTy / 32];
  const int dim = spec.dim, g = spec.g, bs = 1 + g, hd = dim + 1, n = N * bs;
  // 1-D block (block_sum's warp bookkeeping assumes it): thread -> (row point fast, column point slow)
  const int j = blockIdx.x * kHgTx + (threadIdx.x % kHgTx);  // row point (fast)
  const int i = blockIdx.y * kHgTy + (threadIdx.x / kHgTx);  // column point
  double acc[CMOE_MAX_DIM + 1];
  for (int h = 0; h < hd; ++h) acc[h] = 0.0;
  if (i < N && j < N) {
    hyper_grad_pair<false>(spec, X + static_cast<size_t>(j) * dim, X + static_cast<size_t>(i) * dim, j, i,
                           [&](int row, int col) { return a[row] * a[col] - Kinv[static_cast<size_t>(col) * n + row]; },
                           acc);
  }
  const int cta = blockIdx.y * gridDim.x + blockIdx.x;
  for (int h = 0; h < hd; ++h) {
    const double s = block_sum(acc[h], scratch);
    if (threadIdx.x == 0) partial[static_cast<size_t>(cta) * hd + h] = 0.5 * s;
    __syncthreads();
  }
}

// diagW[row] = a[row]^2 - Kinv[row, row]
__global__ void hyper_grad_diag_kernel(const double* __restrict__ a, const double* __restrict__ Kinv, int n,
                                       double* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) out[r] = a[r] * a[r] - Kinv[static_cast<size_t>(r) * n + r];
}

// ---- log marginal likelihood at a list of hyper-parameter sets ---------------------------------------------------
constexpr int kLmlCovThreads = 256;
constexpr int kLmlSolveThreads = 256;
constexpr double kLog2Pi = 1.8378770664093453;
static_assert(sizeof(KernelSpec) % sizeof(unsigned long long) == 0, "KernelSpec is staged as 8-byte words");

// K_s = K(X, X; theta_s) + diag(noise_s by observation type), lower 64 x 64 tiles of the column-major n x n matrix of
// every set; grid (tiles, 1, sets).  The set's KernelSpec is staged in shared memory, the (at most 64) points of the
// tile's rows and columns beside it; entries are cov_build_generic_kernel's (kernel_parts / weighted_sqdist / cov_entry
// on the raw points).  Only the lower triangle is written: potrf_batched reads nothing else.
__global__ void __launch_bounds__(kLmlCovThreads) lml_cov_kernel(const KernelSpec* __restrict__ specs,
                                                                 const double* __restrict__ noise,
                                                                 const double* __restrict__ X, int N,
                                                                 double* __restrict__ K) {
  extern __shared__ double lml_pts[];  // [NB][dim] row points, then [NB][dim] column points
  __shared__ KernelSpec spec;
  const int set = blockIdx.z, tid = threadIdx.x;
  {
    const auto* src = reinterpret_cast<const unsigned long long*>(specs + set);
    auto* dst = reinterpret_cast<unsigned long long*>(&spec);
    for (int w = tid; w < static_cast<int>(sizeof(KernelSpec) / sizeof(unsigned long long)); w += blockDim.x)
      dst[w] = src[w];
  }
  __syncthreads();
  const int dim = spec.dim, b = 1 + spec.g, n = N * b;
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int row0 = ti * NB, col0 = tj * NB;
  const int rows = min(NB, n - row0), cols = min(NB, n - col0);
  const int pr0 = row0 / b, pc0 = col0 / b;
  const int npr = (row0 + rows - 1) / b - pr0 + 1, npc = (col0 + cols - 1) / b - pc0 + 1;
  double* Pr = lml_pts;
  double* Pc = lml_pts + NB * dim;
  for (int e = tid; e < npr * dim; e += blockDim.x) Pr[e] = X[static_cast<size_t>(pr0) * dim + e];
  for (int e = tid; e < npc * dim; e += blockDim.x) Pc[e] = X[static_cast<size_t>(pc0) * dim + e];
  __syncthreads();
  const double* nz = noise + static_cast<size_t>(set) * b;
  double* Ks = K + static_cast<size_t>(set) * n * n;
  for (int e = tid; e < NB * NB; e += blockDim.x) {
    const int r = e % NB, c = e / NB;  // consecutive threads store consecutive rows of one column
    const int gr = row0 + r, gc = col0 + c;
    if (r >= rows || c >= cols || gr < gc) continue;
    const double* p1 = Pr + (gr / b - pr0) * dim;
    const double* p2 = Pc + (gc / b - pc0) * dim;
    const KParts kp = kernel_parts(spec, weighted_sqdist(spec, p1, p2));
    const int m = gr % b, cn = gc % b;
    double v = cov_entry(spec, kp, p1, p2, m ? spec.derivs[m - 1] : -1, cn ? spec.derivs[cn - 1] : -1);
    if (gr == gc) v += nz[m];
    Ks[static_cast<size_t>(gc) * n + gr] = v;
  }
}

// One CTA per set: z = L^-1 r by blocked forward substitution over 64-row blocks (warp 0 solves the diagonal block out
// of shared memory; then every thread updates its rows below, summing the block's products in ascending column order),
// then  -1/2 z^T z - sum_i log L_ii - n/2 log 2 pi  with a fixed thread-to-row assignment and block_sum.  A set whose
// factorisation failed (fail[set] != 0) gets -inf.  With a_out, the kernel then goes on to a = L^-T z = K^-1 r by
// blocked backward substitution (the value is computed before and does not depend on it): a_out[set][n].
__global__ void __launch_bounds__(kLmlSolveThreads) lml_solve_kernel(const double* __restrict__ L, int n,
                                                                     const double* __restrict__ r,
                                                                     const int* __restrict__ fail,
                                                                     double* __restrict__ out,
                                                                     double* __restrict__ a_out) {
  extern __shared__ double lml_z[];         // [n] right-hand side -> solution
  double* D = lml_z + n;                    // [NB][NB + 1] diagonal block, D[c * (NB + 1) + row]
  __shared__ double scratch[kLmlSolveThreads / 32];
  const int set = blockIdx.x, tid = threadIdx.x;
  if (fail[set] != 0) {
    if (tid == 0) out[set] = -INFINITY;
    return;
  }
  const double* Ls = L + static_cast<size_t>(set) * n * n;
  for (int i = tid; i < n; i += blockDim.x) lml_z[i] = r[i];
  cta_forward_subst(Ls, n, lml_z, D);
  double zz = 0.0, logdiag = 0.0;
  for (int i = tid; i < n; i += blockDim.x) {
    zz = fma(lml_z[i], lml_z[i], zz);
    logdiag += log(Ls[static_cast<size_t>(i) * n + i]);
  }
  zz = block_sum(zz, scratch);
  logdiag = block_sum(logdiag, scratch);
  if (tid == 0) out[set] = -0.5 * zz - logdiag - 0.5 * static_cast<double>(n) * kLog2Pi;
  if (a_out == nullptr) return;
  cta_backward_subst(Ls, n, lml_z, D);
  for (int i = tid; i < n; i += blockDim.x) a_out[static_cast<size_t>(set) * n + i] = lml_z[i];
}

// ---- hyper-parameter gradient at a list of sets (DESIGN.md K11) ----------------------------------------------------
// K_s^-1 = L^-T L^-1 with L^-1 held row-major in its own n x n buffer per set (Linv[r * n + c] = (L^-1)_rc): its
// diagonal 64 x 64 blocks by substitution, its off-diagonal blocks one block row at a time and K^-1 in one launch,
// both as DMMA tile products (tile_mma64).  Only the lower triangle of L^-1 (and the zero upper triangle of its
// diagonal blocks) is ever read.
constexpr int kInvThreads = 128;

// (L^-1)_bb = (L_bb)^-1 for every diagonal block b = blockIdx.x of every set: thread c solves column c by forward
// substitution.  The whole 64 x 64 block is written, zeros above the diagonal.
__global__ void __launch_bounds__(NB) tri_inv_diag_kernel(const double* __restrict__ L, int n,
                                                          const int* __restrict__ fail, double* __restrict__ Linv) {
  extern __shared__ double inv_smem[];
  double (*S)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(inv_smem);            // L_bb, S[row][col]
  double (*Xs)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(inv_smem + NB * (NB + 1));  // its inverse
  const int set = blockIdx.z, tid = threadIdx.x;
  if (fail[set] != 0) return;
  const int k0 = blockIdx.x * NB, nb = min(NB, n - k0);
  const double* Ls = L + static_cast<size_t>(set) * n * n;
  for (int e = tid; e < NB * NB; e += blockDim.x) {
    const int r = e % NB, c = e / NB;
    S[r][c] = (r < nb && c < nb && r >= c) ? Ls[static_cast<size_t>(k0 + c) * n + k0 + r] : 0.0;
  }
  __syncthreads();
  const int c = tid;
  for (int r = 0; r < nb; ++r) {
    double v = 0.0;
    if (r == c) {
      v = 1.0 / S[c][c];
    } else if (r > c) {
      double acc = 0.0;
      for (int k = c; k < r; ++k) acc = fma(S[r][k], Xs[k][c], acc);
      v = -acc / S[r][r];
    }
    Xs[r][c] = v;
  }
  __syncthreads();
  double* Li = Linv + static_cast<size_t>(set) * n * n;
  for (int e = tid; e < NB * NB; e += blockDim.x) {
    const int cc = e % NB, r = e / NB;
    if (r < nb && cc < nb) Li[static_cast<size_t>(k0 + r) * n + k0 + cc] = Xs[r][cc];
  }
}

// Block row bi of L^-1 left of the diagonal, for every set: tile (bi, bj = blockIdx.x < bi)
//   (L^-1)_{bi,bj} = -(L^-1)_{bi,bi} sum_{k=bj}^{bi-1} L_{bi,k} (L^-1)_{k,bj}
// Block rows above bi are final (earlier launches).  Blocks k < bi are full 64-row blocks.
__global__ void __launch_bounds__(kInvThreads) tri_inv_offdiag_kernel(const double* __restrict__ L, int n, int bi,
                                                                      const int* __restrict__ fail,
                                                                      double* __restrict__ Linv) {
  extern __shared__ double inv_smem[];
  const int set = blockIdx.z;
  if (fail[set] != 0) return;
  L += static_cast<size_t>(set) * n * n;
  Linv += static_cast<size_t>(set) * n * n;
  double* As = inv_smem;
  double* Bs = inv_smem + NB * LDT;
  const int row0 = bi * NB, col0 = blockIdx.x * NB, rows = min(NB, n - row0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  for (int k0 = col0; k0 < row0; k0 += NB) {
    __syncthreads();  // the previous product's reads of As / Bs are done
    for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
      const int x = e % NB, y = e / NB;
      // As[k][r] = L[row0 + r, k0 + k] (column-major L), Bs[k][c] = L^-1[k0 + k, col0 + c] (row-major L^-1)
      const double* src = L + static_cast<size_t>(k0 + y) * n + row0 + x;
      cp_async8(As + y * LDT + x, x < rows ? src : L, x < rows);
      cp_async8(Bs + y * LDT + x, Linv + static_cast<size_t>(k0 + y) * n + col0 + x, true);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    tile_mma64(As, Bs, acc, wm, wn, lr, lc);
  }
  __syncthreads();
  // T = the sum above -> Bs[k][c]; (L^-1)_{bi,bi} -> As[k][r] = L^-1[row0 + r, row0 + k]
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        Bs[(wm + i * 8 + lr) * LDT + wn + j * 8 + lc * 2 + h] = acc[i][j][h];
        acc[i][j][h] = 0.0;
      }
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int k = e % NB, r = e / NB;
    As[k * LDT + r] = (r < rows && k < rows) ? Linv[static_cast<size_t>(row0 + r) * n + row0 + k] : 0.0;
  }
  __syncthreads();
  tile_mma64(As, Bs, acc, wm, wn, lr, lc);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (r < rows) Linv[static_cast<size_t>(row0 + r) * n + col0 + wn + j * 8 + lc * 2 + h] = -acc[i][j][h];
  }
}

// K^-1 = L^-T L^-1 on the lower 64 x 64 tiles (ti >= tj) of every set: sum over block rows k >= ti of
// (L^-1)_{k,ti}^T (L^-1)_{k,tj}, written column-major over the factor (which is no longer needed).
__global__ void __launch_bounds__(kInvThreads) inv_syrk_kernel(const double* __restrict__ Linv, int n,
                                                               const int* __restrict__ fail,
                                                               double* __restrict__ Kinv) {
  extern __shared__ double inv_smem[];
  const int set = blockIdx.z;
  if (fail[set] != 0) return;
  Linv += static_cast<size_t>(set) * n * n;
  Kinv += static_cast<size_t>(set) * n * n;
  double* As = inv_smem;
  double* Bs = inv_smem + NB * LDT;
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int row0 = ti * NB, col0 = tj * NB, rows = min(NB, n - row0), cols = min(NB, n - col0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  for (int k0 = row0; k0 < n; k0 += NB) {
    const int kb = min(NB, n - k0);
    __syncthreads();
    for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
      const int x = e % NB, k = e / NB;
      const double* src = Linv + static_cast<size_t>(k0 + k) * n;
      const bool oka = k < kb && x < rows, okb = k < kb && x < cols;
      cp_async8(As + k * LDT + x, oka ? src + row0 + x : Linv, oka);
      cp_async8(Bs + k * LDT + x, okb ? src + col0 + x : Linv, okb);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    tile_mma64(As, Bs, acc, wm, wn, lr, lc);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h;
        if (r < rows && c < cols && row0 + r >= col0 + c) Kinv[static_cast<size_t>(col0 + c) * n + row0 + r] = acc[i][j][h];
      }
  }
}

// partial[set][cta][h], h in [0, dim]: hyper_grad_contract_kernel for every set, grid (point-pair tiles, 1, sets) with
// CTA (bx, by) = (x % gx, x / gx).  The set's KernelSpec is staged in shared memory; W is read from the lower
// triangle of K^-1 only.  kExact: hyper_grad_pair's exact Matern block.
template <bool kExact>
__global__ void __launch_bounds__(kHgTx * kHgTy)
    lml_grad_contract_kernel(const KernelSpec* __restrict__ specs, const double* __restrict__ X, int N, int gx,
                             const double* __restrict__ a, const double* __restrict__ Kinv,
                             const int* __restrict__ fail, double* __restrict__ partial) {
  __shared__ double scratch[kHgTx * kHgTy / 32];
  __shared__ KernelSpec spec;
  const int set = blockIdx.z, tid = threadIdx.x;
  if (fail[set] != 0) return;
  {
    const auto* src = reinterpret_cast<const unsigned long long*>(specs + set);
    auto* dst = reinterpret_cast<unsigned long long*>(&spec);
    for (int w = tid; w < static_cast<int>(sizeof(KernelSpec) / sizeof(unsigned long long)); w += blockDim.x)
      dst[w] = src[w];
  }
  __syncthreads();
  const int dim = spec.dim, hd = dim + 1, n = N * (1 + spec.g);
  const int j = (blockIdx.x % gx) * kHgTx + (tid % kHgTx);  // row point (fast)
  const int i = (blockIdx.x / gx) * kHgTy + (tid / kHgTx);  // column point
  const double* as = a + static_cast<size_t>(set) * n;
  const double* Ks = Kinv + static_cast<size_t>(set) * n * n;
  double acc[CMOE_MAX_DIM + 1];
  for (int h = 0; h < hd; ++h) acc[h] = 0.0;
  if (i < N && j < N) {
    hyper_grad_pair<kExact>(spec, X + static_cast<size_t>(j) * dim, X + static_cast<size_t>(i) * dim, j, i,
                            [&](int row, int col) {
                              const int lo = min(row, col), hi = max(row, col);
                              return as[row] * as[col] - Ks[static_cast<size_t>(lo) * n + hi];
                            },
                            acc);
  }
  for (int h = 0; h < hd; ++h) {
    const double s = block_sum(acc[h], scratch);
    if (tid == 0) partial[(static_cast<size_t>(set) * gridDim.x + blockIdx.x) * hd + h] = 0.5 * s;
    __syncthreads();
  }
}

// One CTA per set, one thread per output: out[set][0] = value; out[set][1 + h] = the set's CTA partials in CTA order
// (h <= dim), or 1/2 sum of a_r^2 - K^-1_rr over the rows r of observation type t in row order (h = dim + 1 + t).  A
// failed set keeps its -inf value and gets zeros.
__global__ void lml_grad_reduce_kernel(const double* __restrict__ values, const double* __restrict__ partial,
                                       int nctas, const double* __restrict__ a, const double* __restrict__ Kinv, int n,
                                       int hd, int bs, const int* __restrict__ fail, double* __restrict__ out) {
  const int set = blockIdx.x, h = threadIdx.x, nh = hd + bs;
  double* o = out + static_cast<size_t>(set) * (1 + nh);
  if (h == 0) o[0] = values[set];
  if (h >= nh) return;
  double s = 0.0;
  if (fail[set] == 0) {
    if (h < hd) {
      for (int c = 0; c < nctas; ++c) s += partial[(static_cast<size_t>(set) * nctas + c) * hd + h];
    } else {
      const double* as = a + static_cast<size_t>(set) * n;
      const double* Ks = Kinv + static_cast<size_t>(set) * n * n;
      for (int r = h - hd; r < n; r += bs) s += 0.5 * (as[r] * as[r] - Ks[static_cast<size_t>(r) * n + r]);
    }
  }
  o[1 + h] = s;
}

// Device workspace of cmoe_log_marginal_likelihood_list and cmoe_grad_log_marginal_likelihood_list, one per host
// thread, kept for the device of the last call, so that the calls of a sampler loop or a descent do not allocate (it
// grows to at most one chunk: kSampleWorkspaceBytes plus the shared inputs, or one set if that is larger).
struct LmlWork {
  int device = -1;
  cudaStream_t stream = nullptr;
  DevBuf<double> X, r, noise, K, stage, values;
  DevBuf<double> Linv, a, partial, gout;  // gradient list only
  DevBuf<KernelSpec> specs;
  DevBuf<int> fail;
  void reset() {
    X.release(); r.release(); noise.release(); K.release(); stage.release(); values.release();
    Linv.release(); a.release(); partial.release(); gout.release();
    specs.release();
    fail.release();
    if (stream) cudaStreamDestroy(stream);
    stream = nullptr;
    device = -1;
  }
  ~LmlWork() { reset(); }
};

LmlWork& lml_workspace(int device) {
  static thread_local LmlWork ws;
  if (ws.device != device) {
    ws.reset();
    CMOE_CUDA(cudaStreamCreateWithFlags(&ws.stream, cudaStreamNonBlocking));
    ws.device = device;
  }
  return ws;
}

// bytes of one set in a likelihood-list chunk without the gradient: K and its factor, the staged diagonal factors, the
// noise variances, the value, the spec and the failure flag
size_t lml_set_bytes(int n, int b) {
  const size_t nsteps = (n + NB - 1) / NB;
  return sizeof(double) * (static_cast<size_t>(n) * n + nsteps * NB * NB + b + 1) + sizeof(KernelSpec) + sizeof(int);
}

// CTAs of one set's gradient contraction: gx point tiles along the rows times the tiles along the columns
int lml_grad_ctas(int N, int& gx) {
  gx = (N + kHgTx - 1) / kHgTx;
  return gx * ((N + kHgTy - 1) / kHgTy);
}

// bytes of one set in a chunk with the gradient: lml_set_bytes plus L^-1 (n x n), a, the contraction's CTA partials and
// the [1 + nh] output row
size_t lml_grad_set_bytes(int N, int dim, int g) {
  const int b = 1 + g, n = N * b;
  int gx;
  const int nctas = lml_grad_ctas(N, gx);
  return lml_set_bytes(n, b) +
         sizeof(double) * (static_cast<size_t>(n) * n + n + static_cast<size_t>(nctas) * (dim + 1) + 1 + 2 + dim + g);
}

// y - m, m = average of the function values in the reference's order (gpp_model_selection.cpp:556-560); it does not
// depend on the set
std::vector<double> centred_values(const double* points_sampled_value, int N, int b) {
  double m = 0.0;
  for (int i = 0; i < N; ++i) m += points_sampled_value[static_cast<size_t>(i) * b];
  m /= N;
  std::vector<double> rc(points_sampled_value, points_sampled_value + static_cast<size_t>(N) * b);
  for (int i = 0; i < N; ++i) rc[static_cast<size_t>(i) * b] -= m;
  return rc;
}

// Uploads the points and y - m and sizes w's buffers for chunks of `chunk` sets (with the gradient's when `grads`).
// Every buffer lml_stages uses is sized here, so lml_stages allocates nothing and can be captured in a graph.
void lml_prepare(LmlWork& w, const double* points_sampled, const double* points_sampled_value, int N, int dim, int g,
                 int chunk, bool grads, cudaStream_t s) {
  const int b = 1 + g, n = N * b, t = (n + NB - 1) / NB;
  int gx;
  const int nctas = lml_grad_ctas(N, gx);
  const std::vector<double> rc = centred_values(points_sampled_value, N, b);
  w.X.upload(points_sampled, static_cast<size_t>(N) * dim, s);
  w.r.upload(rc.data(), n, s);
  w.specs.ensure(chunk);
  w.noise.ensure(static_cast<size_t>(chunk) * b);
  w.K.ensure(static_cast<size_t>(chunk) * n * n);
  w.stage.ensure(static_cast<size_t>(chunk) * t * NB * NB);  // what potrf_batched would grow it to
  w.values.ensure(chunk);
  w.fail.ensure(chunk);
  const size_t smem_solve = (static_cast<size_t>(n) + NB * (NB + 1)) * sizeof(double);
  const size_t smem_inv = 2 * NB * LDT * sizeof(double), smem_diag = 2 * NB * (NB + 1) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(lml_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_solve)));
  if (grads) {
    w.Linv.ensure(static_cast<size_t>(chunk) * n * n);
    w.a.ensure(static_cast<size_t>(chunk) * n);
    w.partial.ensure(static_cast<size_t>(chunk) * nctas * (dim + 1));
    w.gout.ensure(static_cast<size_t>(chunk) * (1 + 2 + dim + g));
    CMOE_CUDA(cudaFuncSetAttribute(tri_inv_offdiag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(smem_inv)));
    CMOE_CUDA(cudaFuncSetAttribute(inv_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(smem_inv)));
    CMOE_CUDA(cudaFuncSetAttribute(tri_inv_diag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(smem_diag)));
  }
}

// The K10 stages, and with `grads` the K11 stages, for the nc sets whose specs, noise and failure flags (zero, or
// preset to skip a set) are in w: values in w.values, and with `grads` the rows [value, gradient] in w.gout.
// `exact` selects the exact Matern contraction when there are derivative rows.  Asynchronous on s.
void lml_stages(LmlWork& w, int N, int dim, int g, int kernel, int nc, bool grads, bool exact, cudaStream_t s) {
  const int b = 1 + g, n = N * b, t = (n + NB - 1) / NB, nh = 2 + dim + g;
  int gx;
  const int nctas = lml_grad_ctas(N, gx);
  const size_t smem_cov = 2 * static_cast<size_t>(NB) * dim * sizeof(double);
  const size_t smem_solve = (static_cast<size_t>(n) + NB * (NB + 1)) * sizeof(double);
  const size_t smem_inv = 2 * NB * LDT * sizeof(double), smem_diag = 2 * NB * (NB + 1) * sizeof(double);
  lml_cov_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kLmlCovThreads, smem_cov, s>>>(w.specs.p, w.noise.p, w.X.p, N, w.K.p);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
  potrf_batched(w.K.p, n, nc, w.fail.p, w.stage, s);
  lml_solve_kernel<<<nc, kLmlSolveThreads, smem_solve, s>>>(w.K.p, n, w.r.p, w.fail.p, w.values.p,
                                                            grads ? w.a.p : nullptr);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
  if (!grads) return;
  tri_inv_diag_kernel<<<dim3(t, 1, nc), NB, smem_diag, s>>>(w.K.p, n, w.fail.p, w.Linv.p);
  for (int bi = 1; bi < t; ++bi)
    tri_inv_offdiag_kernel<<<dim3(bi, 1, nc), kInvThreads, smem_inv, s>>>(w.K.p, n, bi, w.fail.p, w.Linv.p);
  inv_syrk_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kInvThreads, smem_inv, s>>>(w.Linv.p, n, w.fail.p, w.K.p);
  // with g = 0 the exact contraction is the quirk one's function: the same build keeps the bits
  if (exact && g > 0 && kernel == CMOE_KERNEL_MATERN_NU_2P5)
    lml_grad_contract_kernel<true><<<dim3(nctas, 1, nc), kHgTx * kHgTy, 0, s>>>(w.specs.p, w.X.p, N, gx, w.a.p, w.K.p,
                                                                              w.fail.p, w.partial.p);
  else
    lml_grad_contract_kernel<false><<<dim3(nctas, 1, nc), kHgTx * kHgTy, 0, s>>>(w.specs.p, w.X.p, N, gx, w.a.p,
                                                                               w.K.p, w.fail.p, w.partial.p);
  lml_grad_reduce_kernel<<<nc, ((nh + 31) / 32) * 32, 0, s>>>(w.values.p, w.partial.p, nctas, w.a.p, w.K.p, n, dim + 1,
                                                              b, w.fail.p, w.gout.p);
  count_launch(t + 3);
  CMOE_CUDA(cudaGetLastError());
}

// The argument and size checks of the list calls (and of the calls built on the list stages).
void check_lml_problem(int kernel, const double* points_sampled, const double* points_sampled_value,
                       const int* derivatives, int num_derivatives, int dim, int num_sampled) {
  CMOE_REQUIRE(points_sampled != nullptr && points_sampled_value != nullptr, CMOE_ERR_INVALID_VALUE, "NULL argument");
  CMOE_REQUIRE(kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL || kernel == CMOE_KERNEL_MATERN_NU_2P5,
               CMOE_ERR_INVALID_VALUE, "unknown covariance kernel id");
  CMOE_REQUIRE(dim >= 1 && dim <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, CMOE_MAX_DIM]");
  CMOE_REQUIRE(num_sampled >= 1, CMOE_ERR_BOUNDS, "num_sampled must be >= 1");
  CMOE_REQUIRE(num_derivatives >= 0 && num_derivatives <= dim, CMOE_ERR_BOUNDS, "num_derivatives out of range");
  CMOE_REQUIRE(num_derivatives == 0 || derivatives != nullptr, CMOE_ERR_INVALID_VALUE, "derivatives is NULL");
  for (int k = 0; k < num_derivatives; ++k)
    CMOE_REQUIRE(derivatives[k] >= 0 && derivatives[k] < dim, CMOE_ERR_BOUNDS, "derivative index out of range");
  CMOE_REQUIRE(static_cast<long long>(num_sampled) * (1 + num_derivatives) <= kMaxSampleQ, CMOE_ERR_BOUNDS,
               "num_sampled * (1 + num_derivatives) must be <= 8192");
}

void check_hyper_prior(int prior) {
  CMOE_REQUIRE(prior == CMOE_HYPER_PRIOR_NONE || prior == CMOE_HYPER_PRIOR_DEFAULT, CMOE_ERR_INVALID_VALUE,
               "prior must be CMOE_HYPER_PRIOR_NONE or CMOE_HYPER_PRIOR_DEFAULT");
}

// The drivers that keep all their sets on the device at once need them in one likelihood chunk of per_set bytes each.
// `what` opens the message ("num_starts = 5000 exceeds").
void check_one_chunk(int sets, size_t per_set, int n, const std::string& what) {
  const size_t chunk = chunk_items(kMaxChunkSets, kSampleWorkspaceBytes, per_set);
  CMOE_REQUIRE(static_cast<size_t>(sets) <= chunk, CMOE_ERR_BOUNDS,
               what + " one likelihood chunk (" + std::to_string(chunk) + " sets at n = " + std::to_string(n) + ")");
}

}  // namespace
}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_grad_log_marginal_likelihood(int kernel, double alpha, const double* lengths,
                                                 const double* points_sampled, const double* points_sampled_value,
                                                 const double* noise_variance, const int* derivatives,
                                                 int num_derivatives, int dim, int num_sampled, int device,
                                                 double* grad, int* info) {
  if (num_derivatives < 0 || noise_variance == nullptr || grad == nullptr || dim < 1) {
    return guarded(info, [&] { CMOE_REQUIRE(false, CMOE_ERR_INVALID_VALUE, "invalid argument"); });
  }
  const int nh = dim + 1 + 1 + num_derivatives;
  std::fill(grad, grad + nh, 0.0);
  std::vector<double> nz(noise_variance, noise_variance + 1 + num_derivatives);
  for (double& v : nz) v += 1.0e-6;  // gpp_model_selection.cpp:546-549
  cmoe_gp* gp = nullptr;
  int linfo = 0;
  const int rc = cmoe_gp_create(kernel, alpha, lengths, points_sampled, points_sampled_value, nz.data(), derivatives,
                                num_derivatives, dim, num_sampled, device, &gp, &linfo);
  if (rc == CMOE_ERR_SINGULAR) {  // the reference carries on with a garbage factor; report zeros and the leading minor
    if (info) *info = linfo;
    return CMOE_OK;
  }
  if (rc != CMOE_OK) {
    if (info) *info = linfo;
    return rc;
  }
  const int out = guarded(info, [&] {
    require_device(gp->device);
    cudaStream_t s = gp->stream;
    const int N = gp->N, n = gp->n, bs = 1 + gp->spec.g, hd = dim + 1;
    DevBuf<double> Kinv(static_cast<size_t>(n) * n), diagW(n);
    identity_kernel<<<static_cast<unsigned>((static_cast<size_t>(n) * n + 255) / 256), 256, 0, s>>>(Kinv.p, n);
    count_launch();
    potrs_lower(gp->dK.p, n, Kinv.p, n, n, s);
    const dim3 grid((N + kHgTx - 1) / kHgTx, (N + kHgTy - 1) / kHgTy);
    const size_t nctas = static_cast<size_t>(grid.x) * grid.y;
    DevBuf<double> partial(nctas * hd);
    hyper_grad_contract_kernel<<<grid, kHgTx * kHgTy, 0, s>>>(gp->spec, gp->dX.p, N, gp->dKinvY.p, Kinv.p, partial.p);
    hyper_grad_diag_kernel<<<(n + 255) / 256, 256, 0, s>>>(gp->dKinvY.p, Kinv.p, n, diagW.p);
    count_launch(2);
    CMOE_CUDA(cudaGetLastError());
    std::vector<double> hp(nctas * hd), hw(n);
    partial.download(hp.data(), hp.size(), s);
    diagW.download(hw.data(), n, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    for (size_t c = 0; c < nctas; ++c)
      for (int h = 0; h < hd; ++h) grad[h] += hp[c * hd + h];
    for (int row = 0; row < n; ++row) grad[hd + row % bs] += 0.5 * hw[row];
  });
  cmoe_gp_destroy(gp);
  return out;
}

namespace {

// The body of the list calls: values[num_sets], and with grads != NULL also grads[num_sets][2 + dim + g] (exact: the
// exact Matern derivative block).
void lml_list(int kernel, const double* hyperparameters, int num_sets, const double* points_sampled,
              const double* points_sampled_value, const int* derivatives, int num_derivatives, int dim,
              int num_sampled, int device, double* values, double* grads, bool exact) {
  {
    CMOE_REQUIRE(num_sets >= 1, CMOE_ERR_BOUNDS, "num_sets must be >= 1");
    CMOE_REQUIRE(hyperparameters != nullptr && values != nullptr, CMOE_ERR_INVALID_VALUE, "NULL argument");
    check_lml_problem(kernel, points_sampled, points_sampled_value, derivatives, num_derivatives, dim, num_sampled);
    const int g = num_derivatives, b = 1 + g, nh = 2 + dim + g, N = num_sampled;
    // per set: the covariance hyper-parameters as cmoe_gp_create takes them (InitializeCovariance's checks,
    // gpp_covariance.cpp:74-98, naming the set), the noise with the single call's 1e-6 added first
    std::vector<KernelSpec> specs(num_sets);
    std::vector<double> noise(static_cast<size_t>(num_sets) * b);
    for (int s = 0; s < num_sets; ++s) {
      const double* h = hyperparameters + static_cast<size_t>(s) * nh;
      if (!(h[0] > 0.0))
        throw Error(CMOE_ERR_BOUNDS, "hyperparameter set " + std::to_string(s) + ": Invalid hyperparameter (alpha).");
      for (int k = 0; k < dim; ++k)
        if (!(h[1 + k] > 0.0))
          throw Error(CMOE_ERR_BOUNDS,
                      "hyperparameter set " + std::to_string(s) + ": Invalid hyperparameter (length).");
      fill_kernel_spec(specs[s], kernel, dim, g, derivatives, h[0], h + 1);
      for (int t = 0; t < b; ++t) noise[static_cast<size_t>(s) * b + t] = h[1 + dim + t] + 1.0e-6;
    }
    require_device(device);

    LmlWork& w = lml_workspace(device);
    cudaStream_t s = w.stream;
    const size_t per_set = grads ? lml_grad_set_bytes(N, dim, g) : lml_set_bytes(N * b, b);
    const int chunk = static_cast<int>(chunk_items(num_sets, kSampleWorkspaceBytes, per_set, kMaxChunkSets));
    lml_prepare(w, points_sampled, points_sampled_value, N, dim, g, chunk, grads != nullptr, s);
    std::vector<double> hout(grads ? static_cast<size_t>(chunk) * (1 + nh) : 0);
    for (int c0 = 0; c0 < num_sets; c0 += chunk) {
      const int nc = std::min(chunk, num_sets - c0);
      w.specs.upload(specs.data() + c0, nc, s);
      w.noise.upload(noise.data() + static_cast<size_t>(c0) * b, static_cast<size_t>(nc) * b, s);
      CMOE_CUDA(cudaMemsetAsync(w.fail.p, 0, nc * sizeof(int), s));
      lml_stages(w, N, dim, g, kernel, nc, grads != nullptr, exact, s);
      if (!grads) {
        w.values.download(values + c0, nc, s);
        CMOE_CUDA(cudaStreamSynchronize(s));
        continue;
      }
      w.gout.download(hout.data(), static_cast<size_t>(nc) * (1 + nh), s);
      CMOE_CUDA(cudaStreamSynchronize(s));
      for (int k = 0; k < nc; ++k) {
        const double* o = hout.data() + static_cast<size_t>(k) * (1 + nh);
        values[c0 + k] = o[0];
        std::copy(o + 1, o + 1 + nh, grads + static_cast<size_t>(c0 + k) * nh);
      }
    }
  }
}

}  // namespace

extern "C" int cmoe_log_marginal_likelihood_list(int kernel, const double* hyperparameters, int num_sets,
                                                 const double* points_sampled, const double* points_sampled_value,
                                                 const int* derivatives, int num_derivatives, int dim,
                                                 int num_sampled, int device, double* values, int* info) {
  return guarded(info, [&] {
    lml_list(kernel, hyperparameters, num_sets, points_sampled, points_sampled_value, derivatives, num_derivatives,
             dim, num_sampled, device, values, nullptr, false);
  });
}

extern "C" int cmoe_grad_log_marginal_likelihood_list(int kernel, const double* hyperparameters, int num_sets,
                                                      const double* points_sampled,
                                                      const double* points_sampled_value, const int* derivatives,
                                                      int num_derivatives, int dim, int num_sampled, int device,
                                                      double* values, double* grads, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(grads != nullptr, CMOE_ERR_INVALID_VALUE, "NULL argument");
    lml_list(kernel, hyperparameters, num_sets, points_sampled, points_sampled_value, derivatives, num_derivatives,
             dim, num_sampled, device, values, grads, false);
  });
}

extern "C" int cmoe_grad_log_marginal_likelihood_list_exact(int kernel, const double* hyperparameters, int num_sets,
                                                            const double* points_sampled,
                                                            const double* points_sampled_value,
                                                            const int* derivatives, int num_derivatives, int dim,
                                                            int num_sampled, int device, double* values, double* grads,
                                                            int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(grads != nullptr, CMOE_ERR_INVALID_VALUE, "NULL argument");
    lml_list(kernel, hyperparameters, num_sets, points_sampled, points_sampled_value, derivatives, num_derivatives,
             dim, num_sampled, device, values, grads, true);
  });
}

// ---- hyper-parameter MCMC (DESIGN.md K12) --------------------------------------------------------------------------
// emcee 2.2.1's EnsembleSampler.sample with the stretch move (a = 2) on GaussianProcessLogLikelihoodMCMC's
// log-probability (log_likelihood_mcmc.py:277-312), every half-step on the device:
//   hmc_propose_kernel   one thread per moving walker: draws, z = ((a - 1) u + 1)^2 / a, q = c - z (c - s) rounded as
//                        numpy rounds it, then hyper_trial_set: the box check, the noise pinning, the prior, and the
//                        K10 inputs of q
//   lml_stages           K10 without the gradient on the half-ensemble's sets, in the workspace lml_prepare sized
//   hmc_accept_kernel    one thread per moving walker: lnpdiff = (nh - 1) log z + lnp(q) - lnp(s) and the accept
// The initial evaluation runs the same kernels with the move switched off.  One step is captured as a CUDA graph and
// replayed; the step index lives in a device counter that the second half's accept kernel advances.
namespace cmoe {
namespace {

constexpr int kHmcThreads = 128;
constexpr double kStretchA = 2.0;
constexpr double kLogNoiseFree = -0x1.26bb1bbb55516p+4;  // numpy.log(1e-8), the pinned noise of a noise-free model
constexpr double kSqrt2Pi = 2.5066282746310002;           // scipy.stats.norm's _norm_pdf_C = sqrt(2 pi)

// The model whose log-probability the K12 and K19 kernels evaluate: covariance kernel, the K10 sizes (nh = 2 + dim + g)
// and derivative indices, the prior and whether the noise is fitted.
struct HyperModel {
  int nh, dim, g, kernel, prior, noisy;
  int derivs[CMOE_MAX_DIM];
};

HyperModel hyper_model(int kernel, int prior, int noisy, int dim, int g, const int* derivatives) {
  HyperModel m{};
  m.nh = 2 + dim + g;
  m.dim = dim;
  m.g = g;
  m.kernel = kernel;
  m.prior = prior;
  m.noisy = noisy ? 1 : 0;
  for (int k = 0; k < g; ++k) m.derivs[k] = derivatives[k];
  return m;
}

struct HmcArgs {
  int Wh;
  HyperModel m;
  uint64_t seed, first_step;
  const double* tz;  // table (NULL: Philox): [num_steps][W] z uniform, partner, accept uniform
  const int* tp;
  const double* tu;
  double* pos;       // [W][nh] walker positions
  double* lnp;       // [W] their log-probabilities
  double* prop;      // [Wh][nh] proposals of the moving half
  double* lprior;    // [Wh] their prior, -inf when the likelihood is skipped
  double* zz;        // [Wh] stretch factors
  double* lu;        // [Wh] log of the acceptance uniforms
  unsigned long long* step;  // steps done in this call
  KernelSpec* specs;  // K10 inputs and outputs of the half-ensemble's sets
  double* noise;
  int* fail;
  const double* values;
};

// Philox draws of walker w at absolute step `step`: counter (step_lo, step_hi, w, 2) gives the z uniform (words 0, 1)
// and the acceptance uniform (words 2, 3), 53 bits each in [0, 1); counter (step_lo, step_hi, w, 3) gives the partner
// as the high word of its first 64 bits times Wh.  Word 3 = 0 and 1 are the normals' and the Latin hypercube's streams.
__device__ __forceinline__ void hmc_draws(uint64_t seed, uint64_t step, int w, int Wh, double& uz, int& partner,
                                          double& ua) {
  uint32_t c[4] = {static_cast<uint32_t>(step), static_cast<uint32_t>(step >> 32), static_cast<uint32_t>(w), 2u};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  uz = static_cast<double>(((static_cast<uint64_t>(c[0]) << 32) | c[1]) >> 11) * 0x1.0p-53;
  ua = static_cast<double>(((static_cast<uint64_t>(c[2]) << 32) | c[3]) >> 11) * 0x1.0p-53;
  uint32_t d[4] = {static_cast<uint32_t>(step), static_cast<uint32_t>(step >> 32), static_cast<uint32_t>(w), 3u};
  philox4x32_10(d, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  partner = static_cast<int>(__umul64hi((static_cast<uint64_t>(d[0]) << 32) | d[1], static_cast<uint64_t>(Wh)));
}

// compute_log_likelihood's order (log_likelihood_mcmc.py:277-312) on q[nh] in place: the box (q untouched outside
// it), with noisy == 0 the pinning of the noise entries to log(1e-8), then the prior into lp.  Returns whether the
// likelihood is needed: false outside the box or where the prior is -inf.  With dlp != NULL, dlp[nh] receives d lp / d q
// (zero for pinned entries and when the likelihood is skipped).  Shared by K12's proposals and K19's trial points.
__device__ __forceinline__ bool hyper_box_prior(double* q, int nh, int dim, int b, int prior, int noisy, double& lp,
                                                double* dlp) {
  if (dlp)
    for (int k = 0; k < nh; ++k) dlp[k] = 0.0;
  bool inbox = true;
  for (int k = 0; k < nh; ++k)
    if (q[k] < -20.0 || q[k] > 20.0) inbox = false;
  lp = 1.0;
  if (inbox) {
    if (!noisy)
      for (int t = 0; t < b; ++t) q[1 + dim + t] = kLogNoiseFree;
    if (prior == CMOE_HYPER_PRIOR_DEFAULT) {
      // NormalPrior(0, 1).lnprob returns the pdf (base_prior.py:338-354); TophatPrior(-2, 3) over the lengths
      // (:104-123); HorseshoePrior(0.1) per noise entry in order (:183-201)
      lp = exp(-(q[0] * q[0]) / 2.0) / kSqrt2Pi;
      if (dlp) dlp[0] = -q[0] * lp;
      for (int k = 0; k < dim; ++k)
        if (q[1 + k] < -2.0 || q[1 + k] > 3.0) lp = -INFINITY;
      for (int t = 0; t < b; ++t) {
        const double th = q[1 + dim + t];
        const double r = 0.1 / th;
        const double L = log(1.0 + 3.0 * (r * r));
        lp += (th == 0.0) ? INFINITY : log(L);
        // d/d th log(log(1 + 3 (0.1 / th)^2)) = -6 r^2 / (th (1 + 3 r^2) L), the term as written (not
        // HorseshoePrior.gradient, which is in terms of exp(th))
        if (dlp && noisy && th != 0.0) dlp[1 + dim + t] = -6.0 * (r * r) / (th * (1.0 + 3.0 * (r * r)) * L);
      }
    }
  }
  const bool need = inbox && lp != -INFINITY;
  if (dlp && !need)
    for (int k = 0; k < nh; ++k) dlp[k] = 0.0;
  return need;
}

// The K10 inputs of one set at log-scale q as lml_list builds them on the host; a skipped set gets the finite
// placeholder theta = 0 (its failure flag is preset, so the Cholesky skips it and lml_solve_kernel writes -inf).
__device__ __forceinline__ void hyper_set_inputs(const double* q, bool skip, int kernel, int dim, int g,
                                                 const int* derivs, KernelSpec& sp, double* noise) {
  sp.kernel = kernel;
  sp.dim = dim;
  sp.g = g;
  sp.alpha = exp(skip ? 0.0 : q[0]);
  for (int k = 0; k < CMOE_MAX_DIM; ++k) {
    double lsq = 1.0, il = 0.0;
    if (k < dim) {
      const double l = exp(skip ? 0.0 : q[1 + k]);
      lsq = l * l;
      il = 1.0 / l;
    }
    sp.lsq[k] = lsq;
    sp.inv_len[k] = il;
    sp.derivs[k] = derivs[k];
  }
  for (int t = 0; t < 1 + g; ++t) noise[t] = exp(skip ? 0.0 : q[1 + dim + t]) + 1.0e-6;
}

// Trial set j of the K12 or K19 kernel arguments `a` at log-scale q[nh]: hyper_box_prior on q unless the set is not
// live, its prior into a.lprior[j] (-inf when the likelihood is skipped), its K10 inputs, and a.fail[j] preset to skip
// it.  dlp as hyper_box_prior's.
template <class Args>
__device__ __forceinline__ void hyper_trial_set(const Args& a, int j, bool live, double* q, double* dlp) {
  const HyperModel& m = a.m;
  double lp;
  const bool need = live && hyper_box_prior(q, m.nh, m.dim, 1 + m.g, m.prior, m.noisy, lp, dlp);
  a.lprior[j] = need ? lp : -INFINITY;
  hyper_set_inputs(q, !need, m.kernel, m.dim, m.g, m.derivs, a.specs[j], a.noise + static_cast<size_t>(j) * (1 + m.g));
  a.fail[j] = need ? 0 : -1;
}

// Moving walker w = half * Wh + j.  With move == 0 the proposal is the walker itself (the initial evaluation).
__global__ void __launch_bounds__(kHmcThreads) hmc_propose_kernel(const __grid_constant__ HmcArgs a, int half,
                                                                  int move) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.Wh) return;
  const int nh = a.m.nh, w = half * a.Wh + j;
  const double* s = a.pos + static_cast<size_t>(w) * nh;
  double* q = a.prop + static_cast<size_t>(j) * nh;
  if (move) {
    const unsigned long long step = *a.step;
    double uz, ua;
    int p;
    if (a.tz) {
      const size_t e = static_cast<size_t>(step) * (2 * a.Wh) + w;
      uz = a.tz[e];
      p = a.tp[e];
      ua = a.tu[e];
    } else {
      hmc_draws(a.seed, a.first_step + step, w, a.Wh, uz, p, ua);
    }
    // zz = ((a - 1) rand + 1) ** 2 / a; q = c[rint] - zz (c[rint] - s): each operation rounded as numpy rounds it
    const double t = __dadd_rn(__dmul_rn(kStretchA - 1.0, uz), 1.0);
    const double z = __ddiv_rn(__dmul_rn(t, t), kStretchA);
    const double* c = a.pos + static_cast<size_t>((1 - half) * a.Wh + p) * nh;
    for (int k = 0; k < nh; ++k) q[k] = __dsub_rn(c[k], __dmul_rn(z, __dsub_rn(c[k], s[k])));
    a.zz[j] = z;
    a.lu[j] = log(ua);
  } else {
    for (int k = 0; k < nh; ++k) q[k] = s[k];
  }
  hyper_trial_set(a, j, true, q, nullptr);
}

__global__ void __launch_bounds__(kHmcThreads) hmc_accept_kernel(const __grid_constant__ HmcArgs a, int half,
                                                                 int move) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.Wh) return;
  const int nh = a.m.nh, w = half * a.Wh + j;
  const double lq = a.lprior[j] + a.values[j];  // -inf + -inf for a skipped proposal
  bool take = true;
  if (move) {
    // lnpdiff = (dim - 1.) * np.log(zz) + newlnprob - lnprob0, left to right; accept = lnpdiff > log(rand)
    const double d = __dsub_rn(__dadd_rn(__dmul_rn(static_cast<double>(nh - 1), log(a.zz[j])), lq), a.lnp[w]);
    take = d > a.lu[j];
    if (half == 1 && j == 0) *a.step += 1;
  }
  if (take) {
    const double* q = a.prop + static_cast<size_t>(j) * nh;
    double* p = a.pos + static_cast<size_t>(w) * nh;
    for (int k = 0; k < nh; ++k) p[k] = q[k];
    a.lnp[w] = lq;
  }
}

struct GraphGuard {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  ~GraphGuard() {
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
  }
};

void hyper_mcmc(int kernel, int prior, int noisy, const double* initial_positions, int num_walkers, int num_steps,
                uint64_t seed, uint64_t first_step, const cmoe_mcmc_table* table, const double* points_sampled,
                const double* points_sampled_value, const int* derivatives, int num_derivatives, int dim,
                int num_sampled, int device, double* positions, double* log_probabilities) {
  CMOE_REQUIRE(initial_positions != nullptr && positions != nullptr && log_probabilities != nullptr,
               CMOE_ERR_INVALID_VALUE, "NULL argument");
  check_lml_problem(kernel, points_sampled, points_sampled_value, derivatives, num_derivatives, dim, num_sampled);
  check_hyper_prior(prior);
  const int g = num_derivatives, b = 1 + g, nh = 2 + dim + g, N = num_sampled, W = num_walkers, Wh = W / 2;
  // EnsembleSampler.__init__'s checks
  CMOE_REQUIRE(W % 2 == 0, CMOE_ERR_BOUNDS, "num_walkers must be even");
  CMOE_REQUIRE(W >= 2 * nh, CMOE_ERR_BOUNDS, "num_walkers must be at least twice the number of hyperparameters");
  CMOE_REQUIRE(num_steps >= 1, CMOE_ERR_BOUNDS, "num_steps must be >= 1");
  // the half-ensemble is one K10 chunk of lml_list without the gradient
  check_one_chunk(Wh, lml_set_bytes(N * b, b), N * b, "num_walkers / 2 = " + std::to_string(Wh) + " sets exceed");
  for (size_t e = 0; e < static_cast<size_t>(W) * nh; ++e)
    CMOE_REQUIRE(std::isfinite(initial_positions[e]), CMOE_ERR_INVALID_VALUE, "initial position is not finite");
  const size_t tcount = static_cast<size_t>(num_steps) * W;
  if (table) {
    CMOE_REQUIRE(table->z_uniform != nullptr && table->partner != nullptr && table->accept_uniform != nullptr,
                 CMOE_ERR_INVALID_VALUE, "NULL table array");
    for (size_t e = 0; e < tcount; ++e)
      CMOE_REQUIRE(table->partner[e] >= 0 && table->partner[e] < Wh, CMOE_ERR_BOUNDS,
                   "table partner out of range [0, num_walkers / 2)");
  }
  require_device(device);

  LmlWork& w = lml_workspace(device);
  cudaStream_t s = w.stream;
  // every buffer is sized before the capture
  lml_prepare(w, points_sampled, points_sampled_value, N, dim, g, Wh, false, s);
  DevBuf<double> pos, lnp(W), prop(static_cast<size_t>(Wh) * nh), lprior(Wh), zz(Wh), lu(Wh), tz, tu;
  DevBuf<int> tp;
  DevBuf<unsigned long long> step(1);
  pos.upload(initial_positions, static_cast<size_t>(W) * nh, s);
  if (table) {
    tz.upload(table->z_uniform, tcount, s);
    tp.upload(table->partner, tcount, s);
    tu.upload(table->accept_uniform, tcount, s);
  }
  step.zero(s);
  HmcArgs a{};
  a.Wh = Wh;
  a.m = hyper_model(kernel, prior, noisy, dim, g, derivatives);
  a.seed = seed;
  a.first_step = first_step;
  a.tz = table ? tz.p : nullptr;
  a.tp = table ? tp.p : nullptr;
  a.tu = table ? tu.p : nullptr;
  a.pos = pos.p;
  a.lnp = lnp.p;
  a.prop = prop.p;
  a.lprior = lprior.p;
  a.zz = zz.p;
  a.lu = lu.p;
  a.step = step.p;
  a.specs = w.specs.p;
  a.noise = w.noise.p;
  a.fail = w.fail.p;
  a.values = w.values.p;
  const unsigned blocks = static_cast<unsigned>((Wh + kHmcThreads - 1) / kHmcThreads);
  auto half_step = [&](int half, int move) {
    hmc_propose_kernel<<<blocks, kHmcThreads, 0, s>>>(a, half, move);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    lml_stages(w, N, dim, g, kernel, Wh, false, false, s);
    hmc_accept_kernel<<<blocks, kHmcThreads, 0, s>>>(a, half, move);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
  };
  // run_mcmc evaluates the initial positions first (and pins their noise)
  half_step(0, 0);
  half_step(1, 0);
  GraphGuard gg;
  CMOE_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed));
  try {
    half_step(0, 1);
    half_step(1, 1);
  } catch (...) {
    cudaStreamEndCapture(s, &gg.graph);  // leave the cached stream usable
    throw;
  }
  CMOE_CUDA(cudaStreamEndCapture(s, &gg.graph));
  CMOE_CUDA(cudaGraphInstantiate(&gg.exec, gg.graph, 0));
  for (int i = 0; i < num_steps; ++i) CMOE_CUDA(cudaGraphLaunch(gg.exec, s));
  pos.download(positions, static_cast<size_t>(W) * nh, s);
  lnp.download(log_probabilities, W, s);
  CMOE_CUDA(cudaStreamSynchronize(s));
}

}  // namespace
}  // namespace cmoe

extern "C" int cmoe_hyperparameter_mcmc(int kernel, int prior, int noisy, const double* initial_positions,
                                        int num_walkers, int num_steps, uint64_t seed, uint64_t first_step,
                                        const cmoe_mcmc_table* table, const double* points_sampled,
                                        const double* points_sampled_value, const int* derivatives,
                                        int num_derivatives, int dim, int num_sampled, int device, double* positions,
                                        double* log_probabilities, int* info) {
  return guarded(info, [&] {
    hyper_mcmc(kernel, prior, noisy, initial_positions, num_walkers, num_steps, seed, first_step, table,
               points_sampled, points_sampled_value, derivatives, num_derivatives, dim, num_sampled, device, positions,
               log_probabilities);
  });
}

// ---- hyper-parameter MAP fit (DESIGN.md K19) ------------------------------------------------------------------------
// scipy's _minimize_bfgs with an analytic gradient on nll(theta) = -compute_log_likelihood(theta)
// (log_likelihood_mcmc.py:241-312), every start in lock step.  One round evaluates one trial point of every active start:
//   map_prep_kernel   one thread per start: the box, the pinning, the prior and the K10 inputs (hyper_trial_set)
//   lml_stages        (K10/K11, the exact contraction) on all starts; finished or skipped starts have fail = -1
//   map_step_kernel   one warp per start: the trial's value and gradient, one step of the strong-Wolfe line search
//                     (scipy's scalar_search_wolfe2 and _zoom), and on acceptance the BFGS update of H and the next
//                     direction
// The host reads the number of active starts every kMapPoll rounds.  No sum crosses starts.
namespace cmoe {
namespace {

constexpr int kMapWarps = 4;      // starts per CTA of map_step_kernel
constexpr int kMapPoll = 4;       // rounds between reads of the active count
constexpr int kMapLsIter = 10;    // bracketing steps and zoom trials of the line search
constexpr int kMapMaxNh = 2 + 2 * CMOE_MAX_DIM;
constexpr int kMapPer = (kMapMaxNh + 31) / 32;  // entries per lane
constexpr double kMapC1 = 1.0e-4, kMapC2 = 0.9, kMapAmax = 1.0e100;

enum MapPhase : int { kMapInit = 0, kMapBracket = 1, kMapZoom = 2, kMapDone = 3 };

struct MapState {
  double f, f_old;                 // objective at x, and at the previous iterate (old_old_fval)
  double phi0, dphi0;              // the line search's phi(0) and phi'(0)
  double at;                       // step of the pending trial
  double alpha0, phi_a0, dphi_a0;  // bracketing: the previous step
  double a_lo, a_hi, phi_lo, phi_hi, dphi_lo, a_rec, phi_rec;  // zoom
  int phase, li, iters, evals, status;
};

struct MapArgs {
  int S;
  HyperModel m;
  int max_iter;
  double gtol;
  MapState* st;
  double* x;       // [S][nh] iterates
  double* gr;      // [S][nh] their gradients
  double* p;       // [S][nh] search directions
  double* xt;      // [S][nh] pending trial points
  double* q;       // [S][nh] the trial points after the pinning
  double* dprior;  // [S][nh] d prior / d q
  double* lprior;  // [S] prior, -inf when the likelihood is skipped
  double* H;       // [S][nh][nh] inverse Hessian approximations, row-major
  const double* out;  // [S][1 + nh] value and linear-space gradient of the likelihood (lml_grad_reduce_kernel)
  KernelSpec* specs;
  double* noise;
  int* fail;
  int* active;
};

__global__ void __launch_bounds__(kHmcThreads) map_prep_kernel(const __grid_constant__ MapArgs a) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s == 0) *a.active = 0;
  if (s >= a.S) return;
  const int nh = a.m.nh;
  double* q = a.q + static_cast<size_t>(s) * nh;
  const double* xt = a.xt + static_cast<size_t>(s) * nh;
  for (int k = 0; k < nh; ++k) q[k] = xt[k];
  hyper_trial_set(a, s, a.st[s].phase != kMapDone, q, a.dprior + static_cast<size_t>(s) * nh);
}

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// scipy's _cubicmin / _quadmin: NaN where numpy would raise (a zero divisor, a negative radical) or the result is not
// finite
__device__ __forceinline__ double map_cubicmin(double a, double fa, double fpa, double b, double fb, double c, double fc) {
  const double C = fpa, db = b - a, dc = c - a;
  const double denom = (db * dc) * (db * dc) * (db - dc);
  const double v0 = fb - fa - C * db, v1 = fc - fa - C * dc;
  if (denom == 0.0 || !isfinite(denom)) return NAN;
  const double A = (dc * dc * v0 - db * db * v1) / denom;
  const double B = (-(dc * dc * dc) * v0 + db * db * db * v1) / denom;
  const double radical = B * B - 3.0 * A * C;
  if (A == 0.0 || !(radical >= 0.0)) return NAN;
  const double xmin = a + (-B + sqrt(radical)) / (3.0 * A);
  return isfinite(xmin) ? xmin : NAN;
}

__device__ __forceinline__ double map_quadmin(double a, double fa, double fpa, double b, double fb) {
  const double db = b - a;
  if (db * db == 0.0) return NAN;
  const double B = (fb - fa - fpa * db) / (db * db);
  if (B == 0.0) return NAN;
  const double xmin = a - fpa / (2.0 * B);
  return isfinite(xmin) ? xmin : NAN;
}

// _zoom's next trial step (trial i of this zoom)
__device__ __forceinline__ double map_zoom_trial(const MapState& t, int i) {
  const double dalpha = t.a_hi - t.a_lo;
  const double lo = dalpha < 0 ? t.a_hi : t.a_lo, hi = dalpha < 0 ? t.a_lo : t.a_hi;
  double aj = NAN;
  if (i > 0) {
    const double cchk = 0.2 * dalpha;
    aj = map_cubicmin(t.a_lo, t.phi_lo, t.dphi_lo, t.a_hi, t.phi_hi, t.a_rec, t.phi_rec);
    if (isnan(aj) || aj > hi - cchk || aj < lo + cchk) aj = NAN;
  }
  if (isnan(aj)) {
    const double qchk = 0.1 * dalpha;
    aj = map_quadmin(t.a_lo, t.phi_lo, t.dphi_lo, t.a_hi, t.phi_hi);
    if (isnan(aj) || aj > hi - qchk || aj < lo + qchk) aj = t.a_lo + 0.5 * dalpha;
  }
  return aj;
}

// The line search's decision at a trial with value ft and slope dphi (scalar_search_wolfe2's loop body in the bracket
// phase, _zoom's in the zoom phase; a +inf or NaN trial fails sufficient decrease).  Returns 1 to accept the trial, -1
// when the line search fails, 0 with t.at = the next trial.
__device__ __forceinline__ int map_line_search(MapState& t, double ft, double dphi) {
  if (t.phase == kMapBracket) {
    const double a1 = t.at;
    if (t.li >= kMapLsIter) return 1;  // the loop ran out: scipy takes alpha1 untested
    if (!(ft <= t.phi0 + kMapC1 * a1 * t.dphi0) || (t.li > 0 && ft >= t.phi_a0)) {
      t.a_lo = t.alpha0; t.a_hi = a1; t.phi_lo = t.phi_a0; t.phi_hi = ft; t.dphi_lo = t.dphi_a0;
    } else if (fabs(dphi) <= -kMapC2 * t.dphi0) {
      return 1;
    } else if (dphi >= 0.0) {
      t.a_lo = a1; t.a_hi = t.alpha0; t.phi_lo = ft; t.phi_hi = t.phi_a0; t.dphi_lo = dphi;
    } else {
      t.alpha0 = a1;
      t.at = fmin(2.0 * a1, kMapAmax);
      t.phi_a0 = ft;
      t.dphi_a0 = dphi;
      t.li += 1;
      return t.alpha0 > kMapAmax ? -1 : 0;
    }
    t.phase = kMapZoom;
    t.phi_rec = t.phi0;
    t.a_rec = 0.0;
    t.li = 0;
    t.at = map_zoom_trial(t, 0);
    return 0;
  }
  const double aj = t.at;
  if (!(ft <= t.phi0 + kMapC1 * aj * t.dphi0) || ft >= t.phi_lo) {
    t.phi_rec = t.phi_hi; t.a_rec = t.a_hi; t.a_hi = aj; t.phi_hi = ft;
  } else if (fabs(dphi) <= -kMapC2 * t.dphi0) {
    return 1;
  } else {
    if (dphi * (t.a_hi - t.a_lo) >= 0.0) {
      t.phi_rec = t.phi_hi; t.a_rec = t.a_hi; t.a_hi = t.a_lo; t.phi_hi = t.phi_lo;
    } else {
      t.phi_rec = t.phi_lo; t.a_rec = t.a_lo;
    }
    t.a_lo = aj; t.phi_lo = ft; t.dphi_lo = dphi;
  }
  t.li += 1;
  if (t.li >= kMapLsIter) return -1;
  t.at = map_zoom_trial(t, t.li);
  return 0;
}

// One warp per start; lane l owns entries l + 32 m.  The scalar state is in shared memory and only lane 0 changes it
// (no scalar then has to stay in a register across the divisions' slow-path calls); the vector work and the fixed-order
// warp reductions are shared by all lanes, with __syncwarp between the two.
__global__ void __launch_bounds__(kMapWarps * 32) map_step_kernel(const __grid_constant__ MapArgs a) {
  __shared__ double sh_s[kMapWarps][kMapMaxNh], sh_v[kMapWarps][kMapMaxNh];
  __shared__ MapState sh_t[kMapWarps];
  __shared__ int sh_act[kMapWarps];  // 1 accept, -1 fail, 0 next trial; then 1 = start a line search
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s = blockIdx.x * kMapWarps + warp;
  if (s >= a.S) return;
  MapState& t = sh_t[warp];
  if (lane == 0) t = a.st[s];
  __syncwarp();
  if (t.phase == kMapDone) return;
  const bool first = t.phase == kMapInit;
  const int nh = a.m.nh, dim = a.m.dim;
  const size_t off = static_cast<size_t>(s) * nh;
  double* x = a.x + off;
  double* gr = a.gr + off;
  double* p = a.p + off;
  double* xt = a.xt + off;
  const double* q = a.q + off;
  const double* dp = a.dprior + off;
  const double* o = a.out + static_cast<size_t>(s) * (1 + nh);
  double* ss = sh_s[warp];
  double* sv = sh_v[warp];

  // the trial's nll and gradient: f = -(prior + log p), g_k = -(d prior / d q_k + e^{q_k} d log p / d theta_k), with 0
  // for pinned noise entries; the preset failure flag leaves o[0] = -inf and a zero gradient for a skipped trial
  const double lp = a.lprior[s];
  const double ft = -(lp + o[0]);
  double gt[kMapPer];
  double dphi = 0.0;
#pragma unroll
  for (int m = 0; m < kMapPer; ++m) {
    const int k = lane + 32 * m;
    double v = 0.0;
    if (k < nh && lp != -INFINITY && !(a.m.noisy == 0 && k > dim)) v = -(dp[k] + exp(q[k]) * o[1 + k]);
    gt[m] = v;
    if (k < nh) dphi = fma(v, p[k], dphi);
  }
  dphi = warp_sum(dphi);
  __syncwarp();  // every lane has read t before lane 0 changes it
  if (lane == 0) {
    t.evals += 1;
    int act = 1;
    if (!first) act = map_line_search(t, ft, dphi);
    if (act < 0) {
      t.status = 2;  // scipy's _LineSearchError: warnflag 2, x stays at the last iterate
      t.phase = kMapDone;
    }
    sh_act[warp] = act;
  }
  __syncwarp();

  if (sh_act[warp] == 1) {
    // accept: s = alpha p, y = g_t - g; x = the evaluated trial, g = g_t
    double ys = 0.0, gsq = 0.0, gmax = 0.0;
    bool nan = false;
#pragma unroll
    for (int m = 0; m < kMapPer; ++m) {
      const int k = lane + 32 * m;
      if (k >= nh) continue;
      if (!first) {
        const double sk = __dmul_rn(t.at, p[k]);
        ys = fma(gt[m] - gr[k], sk, ys);
        ss[k] = sk;
        sv[k] = gt[m] - gr[k];
      }
      x[k] = xt[k];
      gr[k] = gt[m];
      gsq = fma(gt[m], gt[m], gsq);
      gmax = fmax(gmax, fabs(gt[m]));
      nan = nan || isnan(gt[m]) || isnan(xt[k]);
    }
    ys = warp_sum(ys);
    gsq = warp_sum(gsq);
    for (int o2 = 16; o2 > 0; o2 >>= 1) gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, o2));
    nan = __any_sync(0xffffffffu, nan) || isnan(ft);
    __syncwarp();
    if (lane == 0) {
      const bool finite_t = isfinite(ft);
      t.f_old = first ? ft + sqrt(gsq) / 2.0 : t.f;
      t.f = ft;
      if (!first) t.iters += 1;
      int st = -1;
      if (first && !finite_t) {
        st = 2;  // the start itself is outside the box, under a -inf prior or singular
      } else if (!nan && gmax <= a.gtol) {
        st = 0;
      } else if (!finite_t) {
        st = 2;
      } else if (t.iters >= a.max_iter) {
        st = 1;
      } else if (nan) {
        st = 3;
      }
      t.status = st;
      if (st >= 0) t.phase = kMapDone;
    }
    __syncwarp();
    if (t.phase != kMapDone) {
      const double* H0 = a.H + static_cast<size_t>(s) * nh * nh;
      if (!first) {
        // H <- (I - rho s y^T) H (I - rho y s^T) + rho s s^T, rho = 1 / y^T s (1000 when y^T s == 0), expanded:
        // H - rho s (y^T H) - rho (H y) s^T + (rho^2 y^T H y + rho) s s^T
        double* H = a.H + static_cast<size_t>(s) * nh * nh;
        const double rho = ys == 0.0 ? 1000.0 : 1.0 / ys;
        double hy[kMapPer], yh[kMapPer], yhy = 0.0;
#pragma unroll
        for (int m = 0; m < kMapPer; ++m) {
          const int k = lane + 32 * m;
          double r = 0.0, c = 0.0;
          if (k < nh)
            for (int jj = 0; jj < nh; ++jj) {
              r = fma(H[static_cast<size_t>(k) * nh + jj], sv[jj], r);
              c = fma(sv[jj], H[static_cast<size_t>(jj) * nh + k], c);
            }
          hy[m] = r;
          yh[m] = c;
          if (k < nh) yhy = fma(sv[k], r, yhy);
        }
        yhy = warp_sum(yhy);
        __syncwarp();
#pragma unroll
        for (int m = 0; m < kMapPer; ++m) {
          const int k = lane + 32 * m;
          if (k < nh) sv[k] = yh[m];  // sv <- y^T H
        }
        __syncwarp();
        const double css = rho * rho * yhy + rho;
#pragma unroll
        for (int m = 0; m < kMapPer; ++m) {
          const int k = lane + 32 * m;
          if (k >= nh) continue;
          const double sk = ss[k];
          for (int jj = 0; jj < nh; ++jj) {
            double& h = H[static_cast<size_t>(k) * nh + jj];
            h = h - rho * sk * sv[jj] - rho * hy[m] * ss[jj] + css * sk * ss[jj];
          }
        }
        __syncwarp();
      }
      // p = -H g, then scalar_search_wolfe2's start
#pragma unroll
      for (int m = 0; m < kMapPer; ++m) {
        const int k = lane + 32 * m;
        if (k < nh) sv[k] = gr[k];
      }
      __syncwarp();
      double d0 = 0.0;
#pragma unroll
      for (int m = 0; m < kMapPer; ++m) {
        const int k = lane + 32 * m;
        if (k >= nh) continue;
        double r = 0.0;
        for (int jj = 0; jj < nh; ++jj) r = fma(H0[static_cast<size_t>(k) * nh + jj], sv[jj], r);
        p[k] = -r;
        d0 = fma(sv[k], -r, d0);
      }
      d0 = warp_sum(d0);
      __syncwarp();
      if (lane == 0) {
        t.phi0 = t.f;
        t.dphi0 = d0;
        double a1 = 1.0;
        if (d0 != 0.0) a1 = fmin(1.0, 1.01 * 2.0 * (t.phi0 - t.f_old) / d0);
        if (a1 < 0.0) a1 = 1.0;
        t.at = fmin(a1, kMapAmax);
        t.alpha0 = 0.0;
        t.phi_a0 = t.phi0;
        t.dphi_a0 = d0;
        t.li = 0;
        t.phase = kMapBracket;
        if (t.at == 0.0) {
          t.status = 2;  // "Rounding errors prevent the line search from converging"
          t.phase = kMapDone;
        }
      }
      __syncwarp();
    }
  }
  if (t.phase != kMapDone) {
    // the next trial x + at p, with the product rounded first as scipy's s = alpha p
#pragma unroll
    for (int m = 0; m < kMapPer; ++m) {
      const int k = lane + 32 * m;
      if (k < nh) xt[k] = __dadd_rn(x[k], __dmul_rn(t.at, p[k]));
    }
    if (lane == 0) atomicAdd(a.active, 1);
  }
  __syncwarp();
  if (lane == 0) a.st[s] = t;
}

__global__ void map_init_kernel(const __grid_constant__ MapArgs a) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nh = a.m.nh;
  if (e >= static_cast<size_t>(a.S) * nh * nh) return;
  const size_t r = e % (nh * nh);
  a.H[e] = (r / nh == r % nh) ? 1.0 : 0.0;
}

void hyper_map(int kernel, int prior, int noisy, const double* starts, int num_starts, const cmoe_map_opts* opts,
               const double* points_sampled, const double* points_sampled_value, const int* derivatives,
               int num_derivatives, int dim, int num_sampled, int device, double* positions, double* values,
               double* gradients, int* iterations, int* evaluations, int* status) {
  CMOE_REQUIRE(starts != nullptr && positions != nullptr && values != nullptr && gradients != nullptr &&
                   iterations != nullptr && evaluations != nullptr && status != nullptr,
               CMOE_ERR_INVALID_VALUE, "NULL argument");
  check_lml_problem(kernel, points_sampled, points_sampled_value, derivatives, num_derivatives, dim, num_sampled);
  check_hyper_prior(prior);
  CMOE_REQUIRE(noisy == 0 || noisy == 1, CMOE_ERR_INVALID_VALUE, "noisy must be 0 or 1");
  const int g = num_derivatives, b = 1 + g, nh = 2 + dim + g, N = num_sampled, S = num_starts;
  double gtol = 1.0e-5;
  int max_iter = 200 * nh;
  if (opts) {
    CMOE_REQUIRE(opts->gtol >= 0.0, CMOE_ERR_INVALID_VALUE, "gtol must be >= 0");
    CMOE_REQUIRE(opts->max_iterations >= 0, CMOE_ERR_INVALID_VALUE, "max_iterations must be >= 0 (0: 200 nh)");
    gtol = opts->gtol;
    if (opts->max_iterations > 0) max_iter = opts->max_iterations;
  }
  CMOE_REQUIRE(S >= 1, CMOE_ERR_BOUNDS, "num_starts must be >= 1");
  // every start is one set of a K11 chunk, with its BFGS state beside it
  const size_t per_set = lml_grad_set_bytes(N, dim, g) + sizeof(MapState) +
                         sizeof(double) * (static_cast<size_t>(nh) * nh + 6 * static_cast<size_t>(nh) + 1);
  check_one_chunk(S, per_set, N * b, "num_starts = " + std::to_string(S) + " exceeds");
  require_device(device);

  LmlWork& w = lml_workspace(device);
  cudaStream_t s = w.stream;
  lml_prepare(w, points_sampled, points_sampled_value, N, dim, g, S, true, s);
  const size_t v = static_cast<size_t>(S) * nh;
  DevBuf<MapState> st(S);
  DevBuf<double> x, gr(v), p(v), xt, q(v), dprior(v), lprior(S), H(v * nh);
  DevBuf<int> active(1);
  x.upload(starts, v, s);
  xt.upload(starts, v, s);
  std::vector<MapState> h0(S);
  for (MapState& m : h0) {
    m = MapState{};
    m.phase = kMapInit;
    m.status = -1;
  }
  st.upload(h0.data(), S, s);
  MapArgs a{};
  a.S = S;
  a.m = hyper_model(kernel, prior, noisy, dim, g, derivatives);
  a.max_iter = max_iter;
  a.gtol = gtol;
  a.st = st.p;
  a.x = x.p;
  a.gr = gr.p;
  a.p = p.p;
  a.xt = xt.p;
  a.q = q.p;
  a.dprior = dprior.p;
  a.lprior = lprior.p;
  a.H = H.p;
  a.out = w.gout.p;
  a.specs = w.specs.p;
  a.noise = w.noise.p;
  a.fail = w.fail.p;
  a.active = active.p;
  map_init_kernel<<<static_cast<unsigned>((v * nh + 255) / 256), 256, 0, s>>>(a);
  p.zero(s);
  count_launch();
  // a start makes at most 1 + 2 kMapLsIter evaluations per iteration
  const long long max_rounds = 1 + static_cast<long long>(max_iter) * (2 * kMapLsIter + 1);
  const unsigned prep_blocks = static_cast<unsigned>((S + kHmcThreads - 1) / kHmcThreads);
  const unsigned step_blocks = static_cast<unsigned>((S + kMapWarps - 1) / kMapWarps);
  int* h_active = nullptr;
  CMOE_CUDA(cudaMallocHost(reinterpret_cast<void**>(&h_active), sizeof(int)));
  std::unique_ptr<int, cudaError_t (*)(void*)> keep(h_active, cudaFreeHost);
  for (long long round = 0; round < max_rounds; ++round) {
    map_prep_kernel<<<prep_blocks, kHmcThreads, 0, s>>>(a);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    lml_stages(w, N, dim, g, kernel, S, true, true, s);
    map_step_kernel<<<step_blocks, kMapWarps * 32, 0, s>>>(a);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    if ((round + 1) % kMapPoll == 0 || round + 1 == max_rounds) {
      CMOE_CUDA(cudaMemcpyAsync(h_active, active.p, sizeof(int), cudaMemcpyDeviceToHost, s));
      CMOE_CUDA(cudaStreamSynchronize(s));
      if (*h_active == 0) break;
    }
  }
  std::vector<MapState> hs(S);
  st.download(hs.data(), S, s);
  x.download(positions, v, s);
  gr.download(gradients, v, s);
  CMOE_CUDA(cudaStreamSynchronize(s));
  for (int k = 0; k < S; ++k) {
    values[k] = hs[k].f;
    iterations[k] = hs[k].iters;
    evaluations[k] = hs[k].evals;
    status[k] = hs[k].status < 0 ? 1 : hs[k].status;
  }
}

}  // namespace
}  // namespace cmoe

extern "C" int cmoe_hyperparameter_map(int kernel, int prior, int noisy, const double* starts, int num_starts,
                                       const cmoe_map_opts* opts, const double* points_sampled,
                                       const double* points_sampled_value, const int* derivatives,
                                       int num_derivatives, int dim, int num_sampled, int device, double* positions,
                                       double* values, double* gradients, int* iterations, int* evaluations,
                                       int* status, int* info) {
  return guarded(info, [&] {
    hyper_map(kernel, prior, noisy, starts, num_starts, opts, points_sampled, points_sampled_value, derivatives,
              num_derivatives, dim, num_sampled, device, positions, values, gradients, iterations, evaluations,
              status);
  });
}

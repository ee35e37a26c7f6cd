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
// of W = a a^T - K^-1.  Shared by the single-set and the list contraction kernels.
template <class WF>
__device__ __forceinline__ void hyper_grad_pair(const KernelSpec& spec, const double* p1, const double* p2, int j, int i,
                                                const WF& Wf, double (&acc)[CMOE_MAX_DIM + 1]) {
  const int dim = spec.dim, bs = 1 + spec.g;
  const double r2 = weighted_sqdist(spec, p1, p2);
  if (spec.kernel != CMOE_KERNEL_SQUARE_EXPONENTIAL) {
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
    hyper_grad_pair(spec, X + static_cast<size_t>(j) * dim, X + static_cast<size_t>(i) * dim, j, i,
                    [&](int row, int col) { return a[row] * a[col] - Kinv[static_cast<size_t>(col) * n + row]; }, acc);
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
// triangle of K^-1 only.
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
    hyper_grad_pair(spec, X + static_cast<size_t>(j) * dim, X + static_cast<size_t>(i) * dim, j, i,
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

// The body of both list calls: values[num_sets], and with grads != NULL also grads[num_sets][2 + dim + g].
void lml_list(int kernel, const double* hyperparameters, int num_sets, const double* points_sampled,
              const double* points_sampled_value, const int* derivatives, int num_derivatives, int dim,
              int num_sampled, int device, double* values, double* grads) {
  {
    CMOE_REQUIRE(num_sets >= 1, CMOE_ERR_BOUNDS, "num_sets must be >= 1");
    CMOE_REQUIRE(hyperparameters != nullptr && points_sampled != nullptr && points_sampled_value != nullptr &&
                     values != nullptr,
                 CMOE_ERR_INVALID_VALUE, "NULL argument");
    CMOE_REQUIRE(kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL || kernel == CMOE_KERNEL_MATERN_NU_2P5,
                 CMOE_ERR_INVALID_VALUE, "unknown covariance kernel id");
    CMOE_REQUIRE(dim >= 1 && dim <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, CMOE_MAX_DIM]");
    CMOE_REQUIRE(num_sampled >= 1, CMOE_ERR_BOUNDS, "num_sampled must be >= 1");
    CMOE_REQUIRE(num_derivatives >= 0 && num_derivatives <= dim, CMOE_ERR_BOUNDS, "num_derivatives out of range");
    CMOE_REQUIRE(num_derivatives == 0 || derivatives != nullptr, CMOE_ERR_INVALID_VALUE, "derivatives is NULL");
    for (int k = 0; k < num_derivatives; ++k)
      CMOE_REQUIRE(derivatives[k] >= 0 && derivatives[k] < dim, CMOE_ERR_BOUNDS, "derivative index out of range");
    const int g = num_derivatives, b = 1 + g, nh = 2 + dim + g, N = num_sampled;
    CMOE_REQUIRE(static_cast<long long>(N) * b <= kMaxSampleQ, CMOE_ERR_BOUNDS,
                 "num_sampled * (1 + num_derivatives) must be <= 8192");
    const int n = N * b;
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
      KernelSpec& sp = specs[s];
      sp = KernelSpec{};
      sp.kernel = kernel;
      sp.dim = dim;
      sp.g = g;
      sp.alpha = h[0];
      for (int k = 0; k < CMOE_MAX_DIM; ++k) {
        sp.lsq[k] = 1.0;
        sp.inv_len[k] = 0.0;
        sp.derivs[k] = 0;
      }
      for (int k = 0; k < dim; ++k) {
        sp.lsq[k] = h[1 + k] * h[1 + k];
        sp.inv_len[k] = 1.0 / h[1 + k];
      }
      for (int k = 0; k < g; ++k) sp.derivs[k] = derivatives[k];
      for (int t = 0; t < b; ++t) noise[static_cast<size_t>(s) * b + t] = h[1 + dim + t] + 1.0e-6;
    }
    require_device(device);
    // y - m, m = average of the function values in the reference's order (gpp_model_selection.cpp:556-560); it does
    // not depend on the set
    double m = 0.0;
    for (int i = 0; i < N; ++i) m += points_sampled_value[static_cast<size_t>(i) * b];
    m /= N;
    std::vector<double> rc(points_sampled_value, points_sampled_value + n);
    for (int i = 0; i < N; ++i) rc[static_cast<size_t>(i) * b] -= m;

    LmlWork& w = lml_workspace(device);
    cudaStream_t s = w.stream;
    const int nsteps = (n + NB - 1) / NB;
    // the gradient adds L^-1 (n x n), a, the contraction's CTA partials and the [1 + nh] output row per set
    const int gx = (N + kHgTx - 1) / kHgTx, nctas = gx * ((N + kHgTy - 1) / kHgTy);
    size_t per_set = lml_set_bytes(n, b);
    if (grads)
      per_set += sizeof(double) * (static_cast<size_t>(n) * n + n + static_cast<size_t>(nctas) * (dim + 1) + 1 + nh);
    const int chunk = static_cast<int>(chunk_items(num_sets, kSampleWorkspaceBytes, per_set, kMaxChunkSets));
    w.X.upload(points_sampled, static_cast<size_t>(N) * dim, s);
    w.r.upload(rc.data(), n, s);
    w.specs.ensure(chunk);
    w.noise.ensure(static_cast<size_t>(chunk) * b);
    w.K.ensure(static_cast<size_t>(chunk) * n * n);
    w.values.ensure(chunk);
    w.fail.ensure(chunk);
    const size_t smem_cov = 2 * static_cast<size_t>(NB) * dim * sizeof(double);
    const size_t smem_solve = (static_cast<size_t>(n) + NB * (NB + 1)) * sizeof(double);
    const size_t smem_inv = 2 * NB * LDT * sizeof(double), smem_diag = 2 * NB * (NB + 1) * sizeof(double);
    CMOE_CUDA(cudaFuncSetAttribute(lml_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(smem_solve)));
    if (grads) {
      w.Linv.ensure(static_cast<size_t>(chunk) * n * n);
      w.a.ensure(static_cast<size_t>(chunk) * n);
      w.partial.ensure(static_cast<size_t>(chunk) * nctas * (dim + 1));
      w.gout.ensure(static_cast<size_t>(chunk) * (1 + nh));
      CMOE_CUDA(cudaFuncSetAttribute(tri_inv_offdiag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(smem_inv)));
      CMOE_CUDA(cudaFuncSetAttribute(inv_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(smem_inv)));
      CMOE_CUDA(cudaFuncSetAttribute(tri_inv_diag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(smem_diag)));
    }
    const int t = nsteps;
    std::vector<double> hout(grads ? static_cast<size_t>(chunk) * (1 + nh) : 0);
    for (int c0 = 0; c0 < num_sets; c0 += chunk) {
      const int nc = std::min(chunk, num_sets - c0);
      w.specs.upload(specs.data() + c0, nc, s);
      w.noise.upload(noise.data() + static_cast<size_t>(c0) * b, static_cast<size_t>(nc) * b, s);
      CMOE_CUDA(cudaMemsetAsync(w.fail.p, 0, nc * sizeof(int), s));
      lml_cov_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kLmlCovThreads, smem_cov, s>>>(w.specs.p, w.noise.p, w.X.p, N,
                                                                                  w.K.p);
      count_launch();
      CMOE_CUDA(cudaGetLastError());
      potrf_batched(w.K.p, n, nc, w.fail.p, w.stage, s);
      lml_solve_kernel<<<nc, kLmlSolveThreads, smem_solve, s>>>(w.K.p, n, w.r.p, w.fail.p, w.values.p,
                                                                grads ? w.a.p : nullptr);
      count_launch();
      CMOE_CUDA(cudaGetLastError());
      if (!grads) {
        w.values.download(values + c0, nc, s);
        CMOE_CUDA(cudaStreamSynchronize(s));
        continue;
      }
      tri_inv_diag_kernel<<<dim3(t, 1, nc), NB, smem_diag, s>>>(w.K.p, n, w.fail.p, w.Linv.p);
      for (int bi = 1; bi < t; ++bi)
        tri_inv_offdiag_kernel<<<dim3(bi, 1, nc), kInvThreads, smem_inv, s>>>(w.K.p, n, bi, w.fail.p, w.Linv.p);
      inv_syrk_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kInvThreads, smem_inv, s>>>(w.Linv.p, n, w.fail.p, w.K.p);
      lml_grad_contract_kernel<<<dim3(nctas, 1, nc), kHgTx * kHgTy, 0, s>>>(w.specs.p, w.X.p, N, gx, w.a.p, w.K.p,
                                                                           w.fail.p, w.partial.p);
      lml_grad_reduce_kernel<<<nc, ((nh + 31) / 32) * 32, 0, s>>>(w.values.p, w.partial.p, nctas, w.a.p, w.K.p, n,
                                                                  dim + 1, b, w.fail.p, w.gout.p);
      count_launch(t + 3);
      CMOE_CUDA(cudaGetLastError());
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
             dim, num_sampled, device, values, nullptr);
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
             dim, num_sampled, device, values, grads);
  });
}

// ---- hyper-parameter MCMC (DESIGN.md K12) --------------------------------------------------------------------------
// emcee 2.2.1's EnsembleSampler.sample with the stretch move (a = 2) on GaussianProcessLogLikelihoodMCMC's
// log-probability (log_likelihood_mcmc.py:277-312), every half-step on the device:
//   hmc_propose_kernel   one thread per moving walker: draws, z = ((a - 1) u + 1)^2 / a, q = c - z (c - s) rounded as
//                        numpy rounds it, the box check, the noise pinning, the prior, and the K10 inputs of q
//   lml_cov_kernel, potrf_batched, lml_solve_kernel   (K10, unchanged) on the half-ensemble's sets
//   hmc_accept_kernel    one thread per moving walker: lnpdiff = (nh - 1) log z + lnp(q) - lnp(s) and the accept
// The initial evaluation runs the same kernels with the move switched off.  One step is captured as a CUDA graph and
// replayed; the step index lives in a device counter that the second half's accept kernel advances.
namespace cmoe {
namespace {

constexpr int kHmcThreads = 128;
constexpr double kStretchA = 2.0;
constexpr double kLogNoiseFree = -0x1.26bb1bbb55516p+4;  // numpy.log(1e-8), the pinned noise of a noise-free model
constexpr double kSqrt2Pi = 2.5066282746310002;           // scipy.stats.norm's _norm_pdf_C = sqrt(2 pi)

struct HmcArgs {
  int Wh, nh, dim, g, kernel, prior, noisy;
  int derivs[CMOE_MAX_DIM];
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

// Moving walker w = half * Wh + j.  With move == 0 the proposal is the walker itself (the initial evaluation).
__global__ void __launch_bounds__(kHmcThreads) hmc_propose_kernel(const __grid_constant__ HmcArgs a, int half,
                                                                  int move) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.Wh) return;
  const int nh = a.nh, dim = a.dim, b = 1 + a.g, w = half * a.Wh + j;
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
  // compute_log_likelihood's order: the box (theta untouched outside it), the pinning, the prior
  bool inbox = true;
  for (int k = 0; k < nh; ++k)
    if (q[k] < -20.0 || q[k] > 20.0) inbox = false;
  double lp = 1.0;
  if (inbox) {
    if (!a.noisy)
      for (int t = 0; t < b; ++t) q[1 + dim + t] = kLogNoiseFree;
    if (a.prior == CMOE_HYPER_PRIOR_DEFAULT) {
      // NormalPrior(0, 1).lnprob returns the pdf (base_prior.py:338-354); TophatPrior(-2, 3) over the lengths
      // (:104-123); HorseshoePrior(0.1) per noise entry in order (:183-201)
      lp = exp(-(q[0] * q[0]) / 2.0) / kSqrt2Pi;
      for (int k = 0; k < dim; ++k)
        if (q[1 + k] < -2.0 || q[1 + k] > 3.0) lp = -INFINITY;
      for (int t = 0; t < b; ++t) {
        const double th = q[1 + dim + t];
        const double r = 0.1 / th;
        lp += (th == 0.0) ? INFINITY : log(log(1.0 + 3.0 * (r * r)));
      }
    }
  }
  const bool skip = !inbox || lp == -INFINITY;
  a.lprior[j] = skip ? -INFINITY : lp;
  // the set's KernelSpec and noise as lml_list builds them on the host; a skipped proposal gets the finite placeholder
  // theta = 0 and a preset failure flag, so the Cholesky skips it and lml_solve_kernel writes -inf
  KernelSpec& sp = a.specs[j];
  sp.kernel = a.kernel;
  sp.dim = dim;
  sp.g = a.g;
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
    sp.derivs[k] = a.derivs[k];
  }
  for (int t = 0; t < b; ++t) a.noise[static_cast<size_t>(j) * b + t] = exp(skip ? 0.0 : q[1 + dim + t]) + 1.0e-6;
  a.fail[j] = skip ? -1 : 0;
}

__global__ void __launch_bounds__(kHmcThreads) hmc_accept_kernel(const __grid_constant__ HmcArgs a, int half,
                                                                 int move) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.Wh) return;
  const int nh = a.nh, w = half * a.Wh + j;
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
  CMOE_REQUIRE(initial_positions != nullptr && points_sampled != nullptr && points_sampled_value != nullptr &&
                   positions != nullptr && log_probabilities != nullptr,
               CMOE_ERR_INVALID_VALUE, "NULL argument");
  CMOE_REQUIRE(kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL || kernel == CMOE_KERNEL_MATERN_NU_2P5,
               CMOE_ERR_INVALID_VALUE, "unknown covariance kernel id");
  CMOE_REQUIRE(prior == CMOE_HYPER_PRIOR_NONE || prior == CMOE_HYPER_PRIOR_DEFAULT, CMOE_ERR_INVALID_VALUE,
               "prior must be CMOE_HYPER_PRIOR_NONE or CMOE_HYPER_PRIOR_DEFAULT");
  CMOE_REQUIRE(dim >= 1 && dim <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, CMOE_MAX_DIM]");
  CMOE_REQUIRE(num_sampled >= 1, CMOE_ERR_BOUNDS, "num_sampled must be >= 1");
  CMOE_REQUIRE(num_derivatives >= 0 && num_derivatives <= dim, CMOE_ERR_BOUNDS, "num_derivatives out of range");
  CMOE_REQUIRE(num_derivatives == 0 || derivatives != nullptr, CMOE_ERR_INVALID_VALUE, "derivatives is NULL");
  for (int k = 0; k < num_derivatives; ++k)
    CMOE_REQUIRE(derivatives[k] >= 0 && derivatives[k] < dim, CMOE_ERR_BOUNDS, "derivative index out of range");
  const int g = num_derivatives, b = 1 + g, nh = 2 + dim + g, N = num_sampled, W = num_walkers, Wh = W / 2;
  CMOE_REQUIRE(static_cast<long long>(N) * b <= kMaxSampleQ, CMOE_ERR_BOUNDS,
               "num_sampled * (1 + num_derivatives) must be <= 8192");
  // EnsembleSampler.__init__'s checks
  CMOE_REQUIRE(W % 2 == 0, CMOE_ERR_BOUNDS, "num_walkers must be even");
  CMOE_REQUIRE(W >= 2 * nh, CMOE_ERR_BOUNDS, "num_walkers must be at least twice the number of hyperparameters");
  CMOE_REQUIRE(num_steps >= 1, CMOE_ERR_BOUNDS, "num_steps must be >= 1");
  const int n = N * b, nsteps = (n + NB - 1) / NB;
  // the half-ensemble is one K10 chunk of lml_list without the gradient
  const size_t chunk = chunk_items(kMaxChunkSets, kSampleWorkspaceBytes, lml_set_bytes(n, b));
  CMOE_REQUIRE(static_cast<size_t>(Wh) <= chunk, CMOE_ERR_BOUNDS,
               "num_walkers / 2 = " + std::to_string(Wh) + " sets exceed one likelihood chunk (" +
                   std::to_string(chunk) + " sets at n = " + std::to_string(n) + ")");
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
  // y - m as lml_list centres it (gpp_model_selection.cpp:556-560)
  double m = 0.0;
  for (int i = 0; i < N; ++i) m += points_sampled_value[static_cast<size_t>(i) * b];
  m /= N;
  std::vector<double> rc(points_sampled_value, points_sampled_value + n);
  for (int i = 0; i < N; ++i) rc[static_cast<size_t>(i) * b] -= m;

  LmlWork& w = lml_workspace(device);
  cudaStream_t s = w.stream;
  // every buffer is sized here, before the capture
  w.X.upload(points_sampled, static_cast<size_t>(N) * dim, s);
  w.r.upload(rc.data(), n, s);
  w.specs.ensure(Wh);
  w.noise.ensure(static_cast<size_t>(Wh) * b);
  w.K.ensure(static_cast<size_t>(Wh) * n * n);
  w.stage.ensure(static_cast<size_t>(Wh) * nsteps * NB * NB);
  w.values.ensure(Wh);
  w.fail.ensure(Wh);
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
  a.nh = nh;
  a.dim = dim;
  a.g = g;
  a.kernel = kernel;
  a.prior = prior;
  a.noisy = noisy ? 1 : 0;
  for (int k = 0; k < g; ++k) a.derivs[k] = derivatives[k];
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
  const size_t smem_cov = 2 * static_cast<size_t>(NB) * dim * sizeof(double);
  const size_t smem_solve = (static_cast<size_t>(n) + NB * (NB + 1)) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(lml_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_solve)));
  const unsigned blocks = static_cast<unsigned>((Wh + kHmcThreads - 1) / kHmcThreads);
  auto half_step = [&](int half, int move) {
    hmc_propose_kernel<<<blocks, kHmcThreads, 0, s>>>(a, half, move);
    lml_cov_kernel<<<dim3(nsteps * (nsteps + 1) / 2, 1, Wh), kLmlCovThreads, smem_cov, s>>>(w.specs.p, w.noise.p,
                                                                                            w.X.p, N, w.K.p);
    count_launch(2);
    CMOE_CUDA(cudaGetLastError());
    potrf_batched(w.K.p, n, Wh, w.fail.p, w.stage, s);
    lml_solve_kernel<<<Wh, kLmlSolveThreads, smem_solve, s>>>(w.K.p, n, w.r.p, w.fail.p, w.values.p, nullptr);
    hmc_accept_kernel<<<blocks, kHmcThreads, 0, s>>>(a, half, move);
    count_launch(2);
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

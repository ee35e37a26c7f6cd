// Joint posterior draws over point sets and Thompson-sampled global optima, batched over sets.
//
// Replaces (reference, moe/optimal_learning/cpp/):
//   GaussianProcess::SamplePointFromGP            gpp_math.cpp:1761-1798  (one point with the GP's derivative rows)
//   GaussianProcess::SamplePointsFromGP           gpp_math.cpp:1803-1848  (joint draw over a set + argmin)
//   GaussianProcess::SampleGlobalOptimaFromGP     gpp_math.cpp:1854-1870
//   ComputeLatinHypercubePointsInDomain           gpp_random.cpp:173-194  (TensorProductDomain::GenerateUniformPointsInDomain)
//
// Per chunk of sets (each set: num points, gs derivative rows per point, Q = num (1 + gs) rows):
//   K* = K(X, P)                       build_mix_covariance, all sets of the chunk at once
//   V  = L^-1 K*                       ONE blocked forward solve over n x (chunk Q) right-hand sides
//   mu                                 post_mean_only_kernel (posterior_mean_points)
//   Var = K(P, P) - V^T V (+ jitter I) cov_tile_kernel: DMMA m16n8k4, the prior block is evaluated in the epilogue
//   L L^T = Var                        batched blocked Cholesky, every launch covers all sets of the chunk
//   y = mu + L w, argmin               sample_rows_kernel + best_of_parts_kernel
// The reference forms Var as (K^-1 K*)^T K* with two triangular solves; V^T V needs one solve (half the solve work)
// and its product is exactly symmetric.  The two differ by rounding only.
//
// Chunking: a chunk holds as many sets as fit in kSampleWorkspaceBytes of device workspace (at least one set).  Every
// set has its own normals (Philox draw first_draw + set index), its own failure flag and fixed-order reductions, and
// every kernel treats the sets of a chunk independently, so a set's result does not depend on the chunking.
#include <algorithm>
#include <climits>
#include <cmath>
#include <functional>

#include "device_math.cuh"
#include "internal.cuh"
#include "linalg_dev.cuh"

namespace cmoe {

namespace {

constexpr int kTileThreads = 128;
constexpr int kRowThreads = 256;

__device__ __forceinline__ int set_row_type(int local, const int* derivs) { return local ? derivs[local - 1] : -1; }

// --------------------------------------------------------------------------------------------------------------
// Latin hypercube: one CTA per (dimension, set).  The strata of a dimension are permuted by ranking Philox keys (ties
// broken by point index); point j lies in stratum rank_j at offset u_j:  x = min + edge rank_j + edge u_j,  clamped to
// max.  Key and offset of point j in dimension i come from one Philox call with counter (draw_lo, draw_hi,
// i num_pts + j, 1); the normals use the fourth counter word 0, so the two streams never overlap.  Multiplications and
// additions are explicitly rounded (no contraction), so the points are a pure function of (seed, draw).
// --------------------------------------------------------------------------------------------------------------
struct Box {
  double lo[CMOE_MAX_DIM];
  double hi[CMOE_MAX_DIM];
};

__device__ __forceinline__ void philox_key_uniform(uint64_t seed, uint64_t draw, uint32_t k, uint64_t& key, double& u) {
  uint32_t c[4] = {static_cast<uint32_t>(draw), static_cast<uint32_t>(draw >> 32), k, 1u};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  key = ((static_cast<uint64_t>(c[0]) << 32) | c[1]) >> 11;
  const uint64_t b = ((static_cast<uint64_t>(c[2]) << 32) | c[3]) >> 11;
  u = __dmul_rn(__dadd_rn(static_cast<double>(b), 0.5), 0x1.0p-53);
}

__global__ void __launch_bounds__(256) lhs_kernel(uint64_t seed, uint64_t first_draw, int num_pts, int dim,
                                                  const __grid_constant__ Box box, double* __restrict__ out) {
  extern __shared__ uint64_t keys[];  // [num_pts]
  const int i = blockIdx.x, set = blockIdx.y;
  const uint64_t draw = first_draw + set;
  const uint32_t kbase = static_cast<uint32_t>(i) * static_cast<uint32_t>(num_pts);
  for (int j = threadIdx.x; j < num_pts; j += blockDim.x) {
    double u;
    philox_key_uniform(seed, draw, kbase + j, keys[j], u);
  }
  __syncthreads();
  const double lo = box.lo[i], hi = box.hi[i];
  const double edge = __ddiv_rn(__dsub_rn(hi, lo), static_cast<double>(num_pts));
  for (int j = threadIdx.x; j < num_pts; j += blockDim.x) {
    uint64_t kj;
    double u;
    philox_key_uniform(seed, draw, kbase + j, kj, u);
    int rank = 0;
    for (int m = 0; m < num_pts; ++m) {
      const uint64_t km = keys[m];
      rank += (km < kj || (km == kj && m < j)) ? 1 : 0;
    }
    double x = __dadd_rn(lo, __dmul_rn(edge, static_cast<double>(rank)));
    x = fmin(__dadd_rn(x, __dmul_rn(edge, u)), hi);
    out[(static_cast<size_t>(set) * num_pts + j) * dim + i] = x;
  }
}

// --------------------------------------------------------------------------------------------------------------
// Var_b = K(P_b, P_b) - V_b^T V_b (+ jitter I), lower 64 x 64 tiles; grid (tiles, 1, sets).  V_b = columns
// [b Q, (b+1) Q) of V (n rows, ld n) are the DMMA operands, streamed in 64-deep chunks; the prior entries come from
// the tile's points, held in shared memory, so K(P, P) is never materialised.  Only the lower triangle is written.
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTileThreads) cov_tile_kernel(const __grid_constant__ KernelSpec spec,
                                                                const double* __restrict__ V, int n, int Q,
                                                                const double* __restrict__ P, int num,
                                                                const int* __restrict__ dPs, int gs, double jitter,
                                                                double* __restrict__ A) {
  extern __shared__ double smem[];
  double* As = smem;               // [NB][LDT]
  double* Bs = As + NB * LDT;      // [NB][LDT]
  double* Pr = Bs + NB * LDT;      // [NB][dim] points of the tile's rows
  double* Pc = Pr + NB * spec.dim; // [NB][dim] points of the tile's columns
  __shared__ int sd[CMOE_MAX_DIM];
  const int set = blockIdx.z, tid = threadIdx.x, dim = spec.dim, bs = 1 + gs;
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int row0 = ti * NB, col0 = tj * NB;
  const int rows = min(NB, Q - row0), cols = min(NB, Q - col0);
  const int pr0 = row0 / bs, pc0 = col0 / bs;
  const double* Pset = P + static_cast<size_t>(set) * num * dim;
  for (int e = tid; e < min(NB, num - pr0) * dim; e += blockDim.x) Pr[e] = Pset[static_cast<size_t>(pr0) * dim + e];
  for (int e = tid; e < min(NB, num - pc0) * dim; e += blockDim.x) Pc[e] = Pset[static_cast<size_t>(pc0) * dim + e];
  if (tid < gs) sd[tid] = dPs[tid];
  const double* Vr = V + (static_cast<size_t>(set) * Q + row0) * n;
  const double* Vc = V + (static_cast<size_t>(set) * Q + col0) * n;
  const int warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  gram_tile_accumulate(Vr, Vc, n, rows, cols, As, Bs, acc, wm, wn, lr, lc);
  double* Ab = A + static_cast<size_t>(set) * Q * Q;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr, gr = row0 + r;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h, gc = col0 + c;
        if (r < rows && c < cols && gr >= gc) {
          const double* p1 = Pr + (gr / bs - pr0) * dim;
          const double* p2 = Pc + (gc / bs - pc0) * dim;
          const KParts kp = kernel_parts(spec, weighted_sqdist(spec, p1, p2));
          double v = cov_entry(spec, kp, p1, p2, set_row_type(gr % bs, sd), set_row_type(gc % bs, sd)) - acc[i][j][h];
          if (gr == gc) v += jitter;
          Ab[static_cast<size_t>(gc) * Q + gr] = v;
        }
      }
  }
}

// --------------------------------------------------------------------------------------------------------------
// Batched blocked Cholesky, one 64-column step = two launches over every set of the chunk (blockIdx.z = set):
//   panel:  every CTA factors the diagonal block in its own shared memory (factor_block64); CTA 0 stores the factor in
//           a per-set staging area, CTA x >= 1 solves PT rows of the panel below.  The diagonal block of A is left as
//           it is during the factorisation (no later step reads it), so no CTA waits for another; one launch at the
//           end copies the staged diagonal factors into place;
//   update: A22 -= L21 L21^T on the lower 64 x 64 tiles of the trailing matrix, DMMA m16n8k4.
// Pivots and multipliers take the reciprocal-square-root form of the large single-matrix path (FAST = true).
// fail[set] holds 0 or the 1-based leading minor of the first pivot that fails `> 1e-16`; a failed set stops updating.
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PT) chol_panel_kernel(double* __restrict__ A, int Q, int k0, int nb,
                                                        int* __restrict__ fail, double* __restrict__ stage) {
  extern __shared__ __align__(16) double panel_smem[];
  double* LT = panel_smem;                                              // [NB][LTS] + NB padding
  double* colbuf = LT + NB * LTS + NB;                                  // [2][64]
  double* rd = colbuf + 128;                                            // [NB]
  double (*S)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(rd + NB);  // [NB][NB+1]
  __shared__ int sfail;
  const int set = blockIdx.z;
  if (fail[set] != 0) return;
  A += static_cast<size_t>(set) * Q * Q;
  const int tid = threadIdx.x;
  double* Ab = A + static_cast<size_t>(k0) * Q + k0;
  {
    const int r = tid & (NB - 1);
    for (int c = tid >> 6; c < NB; c += PT / NB)
      S[r][c] = (r < nb && c < nb && r >= c) ? Ab[static_cast<size_t>(c) * Q + r] : ((r == c && r >= nb) ? 1.0 : 0.0);
    for (int e = tid; e < NB * LTS + NB + 128; e += PT) LT[e] = 0.0;
  }
  const int myrow = k0 + nb + (static_cast<int>(blockIdx.x) - 1) * PT + tid;
  const bool valid = blockIdx.x > 0 && myrow < Q;
  double x[NB];
  if (blockIdx.x > 0) {
    const double* Ar = A + static_cast<size_t>(k0) * Q + myrow;
#pragma unroll
    for (int c = 0; c < NB; ++c) x[c] = (valid && c < nb) ? Ar[static_cast<size_t>(c) * Q] : 0.0;
  }
  __syncthreads();
  const int failed = factor_block64<true>(S, LT, rd, colbuf, &sfail);
  if (failed) {
    if (blockIdx.x == 0 && tid == 0) fail[set] = k0 + failed;
    return;
  }
  if (blockIdx.x == 0) {
    // staging [set][step][NB*NB], column-major lower factor of the diagonal block
    double* D = stage + (static_cast<size_t>(set) * ((Q + NB - 1) / NB) + k0 / NB) * NB * NB;
    const int r = tid & (NB - 1);
    for (int c = tid >> 6; c < NB; c += PT / NB)
      if (r < nb && c < nb && r >= c) D[c * NB + r] = LT[c * LTS + r];
    return;
  }
  double* Aw = A + static_cast<size_t>(k0) * Q + myrow;
  auto emit = [&](int k, double v) {
    if (valid && k < nb) Aw[static_cast<size_t>(k) * Q] = v;
  };
  solve_steps_rot<NB, NB / 2, 4, true>(x, LT, rd, 0, emit);
  double xh[NB / 2];
#pragma unroll
  for (int i = 0; i < NB / 2; ++i) xh[i] = x[i];
  solve_steps_rot<NB / 2, NB / 2, 4, true>(xh, LT, rd, NB / 2, emit);
}

// staged diagonal factors -> diagonal blocks of A; grid (steps, 1, sets).  Failed sets keep their partial state.
__global__ void __launch_bounds__(PT) chol_diag_writeback_kernel(double* __restrict__ A, int Q,
                                                                 const int* __restrict__ fail,
                                                                 const double* __restrict__ stage) {
  const int set = blockIdx.z, step = blockIdx.x;
  if (fail[set] != 0) return;
  const int k0 = step * NB, nb = min(NB, Q - k0);
  const double* D = stage + (static_cast<size_t>(set) * gridDim.x + step) * NB * NB;
  double* Ab = A + static_cast<size_t>(set) * Q * Q + static_cast<size_t>(k0) * Q + k0;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int r = e % NB, c = e / NB;
    if (r < nb && c < nb && r >= c) Ab[static_cast<size_t>(c) * Q + r] = D[e];
  }
}

__global__ void __launch_bounds__(kTileThreads) chol_update_kernel(double* __restrict__ A, int Q, int k0, int nb,
                                                                   const int* __restrict__ fail) {
  extern __shared__ double smem[];
  const int set = blockIdx.z;
  if (fail[set] != 0) return;
  A += static_cast<size_t>(set) * Q * Q;
  double* As = smem;
  double* Bs = smem + NB * LDT;
  const int t0 = k0 + nb;
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int row0 = t0 + ti * NB, col0 = t0 + tj * NB;
  const int rows = min(NB, Q - row0), cols = min(NB, Q - col0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  const double* Ac = A + static_cast<size_t>(k0) * Q + row0;
  const double* Bc = A + static_cast<size_t>(k0) * Q + col0;
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int r = e % NB, c = e / NB;
    const bool oka = r < rows && c < nb, okb = r < cols && c < nb;
    cp_async8(As + c * LDT + r, oka ? Ac + static_cast<size_t>(c) * Q + r : Ac, oka);
    cp_async8(Bs + c * LDT + r, okb ? Bc + static_cast<size_t>(c) * Q + r : Bc, okb);
  }
  cp_async_commit();
  // accumulate +L21 L21^T on top of -C while the operands land; the epilogue stores -acc
  double acc[4][4][2];
  double* Cg = A + static_cast<size_t>(col0) * Q + row0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h;
        acc[i][j][h] = (r < rows && c < cols) ? -Cg[static_cast<size_t>(c) * Q + r] : 0.0;
      }
  }
  cp_async_wait<0>();
  __syncthreads();
  tile_mma64(As, Bs, acc, wm, wn, lr, lc);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h;
        if (r < rows && c < cols && row0 + r >= col0 + c) Cg[static_cast<size_t>(c) * Q + r] = -acc[i][j][h];
      }
  }
}

// --------------------------------------------------------------------------------------------------------------
// y = mu + L w for 256 rows of one set per CTA (grid (row blocks, sets)); row i sums its i+1 products in ascending
// order.  w: Philox draw (draw0 + set), normals 2k, 2k+1 from call k (cmoe_philox_normals), or row `set` of the table.
// Each CTA leaves the lowest-index minimum of its value rows in (part_v, part_i); best_of_parts_kernel combines them.
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) sample_rows_kernel(int Q, int bs, const double* __restrict__ mu,
                                                                  const double* __restrict__ L, uint64_t seed,
                                                                  uint64_t draw0, const double* __restrict__ table,
                                                                  double* __restrict__ y, double* __restrict__ part_v,
                                                                  int* __restrict__ part_i) {
  extern __shared__ double w[];  // [rows this CTA needs]
  __shared__ double bv[kRowThreads / 32];
  __shared__ int bi[kRowThreads / 32];
  const int set = blockIdx.y, tid = threadIdx.x;
  const int row_end = min(Q, static_cast<int>(blockIdx.x + 1) * kRowThreads);
  if (table) {
    for (int i = tid; i < row_end; i += blockDim.x) w[i] = table[static_cast<size_t>(set) * Q + i];
  } else {
    for (int k = tid; 2 * k < row_end; k += blockDim.x) {
      double a, b;
      philox_normal_pair(seed, draw0 + set, k, a, b);
      w[2 * k] = a;
      if (2 * k + 1 < row_end) w[2 * k + 1] = b;
    }
  }
  __syncthreads();
  const int i = blockIdx.x * kRowThreads + tid;
  double best = INFINITY;
  int bidx = INT_MAX;
  if (i < Q) {
    const double* Li = L + static_cast<size_t>(set) * Q * Q + i;
    double acc = 0.0;
    for (int j = 0; j <= i; ++j) acc = fma(Li[static_cast<size_t>(j) * Q], w[j], acc);
    const double v = mu[static_cast<size_t>(set) * Q + i] + acc;
    y[static_cast<size_t>(set) * Q + i] = v;
    if (i % bs == 0 && v < best) {
      best = v;
      bidx = i / bs;
    }
  }
  block_best<false>(best, bidx, bv, bi);
  if (tid == 0) {
    part_v[static_cast<size_t>(set) * gridDim.x + blockIdx.x] = best;
    part_i[static_cast<size_t>(set) * gridDim.x + blockIdx.x] = bidx;
  }
}

// points_optima[set] = P[set][amin[set]]
__global__ void gather_kernel(int nsets, int num, int dim, const double* __restrict__ P, const int* __restrict__ amin,
                              double* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nsets * dim) return;
  const int set = e / dim, d = e % dim;
  out[e] = P[(static_cast<size_t>(set) * num + amin[set]) * dim + d];
}

// strictly upper triangle of every Q x Q matrix -> 0 (the reference's ZeroUpperTriangle)
__global__ void zero_upper_kernel(int nsets, int Q, double* __restrict__ A) {
  const size_t total = static_cast<size_t>(nsets) * Q * Q;
  for (size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t o = e % (static_cast<size_t>(Q) * Q);
    if (static_cast<int>(o % Q) < static_cast<int>(o / Q)) A[e] = 0.0;
  }
}

// strictly upper triangle of every Q x Q matrix <- its lower triangle (a full symmetric matrix from the lower half)
__global__ void mirror_lower_kernel(int nsets, int Q, double* __restrict__ A) {
  const size_t total = static_cast<size_t>(nsets) * Q * Q;
  for (size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t o = e % (static_cast<size_t>(Q) * Q), base = e - o;
    const int r = static_cast<int>(o % Q), c = static_cast<int>(o / Q);
    if (r < c) A[e] = A[base + static_cast<size_t>(r) * Q + c];
  }
}

size_t panel_smem_bytes() {
  return (static_cast<size_t>(NB) * LTS + NB + 128 + NB + NB * (NB + 1)) * sizeof(double);
}

}  // namespace

// declared in internal.cuh; also factors the covariance matrices of cmoe_log_marginal_likelihood_list
void potrf_batched(double* A, int Q, int nsets, int* fail, DevBuf<double>& stage, cudaStream_t s) {
  stage.ensure(static_cast<size_t>(nsets) * ((Q + NB - 1) / NB) * NB * NB);
  potrf_batched(A, Q, nsets, fail, stage.p, s);
}

void potrf_batched(double* A, int Q, int nsets, int* fail, double* stage, cudaStream_t s) {
  const size_t smem_panel = panel_smem_bytes();
  const size_t smem_tile = 2 * NB * LDT * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(chol_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_panel)));
  CMOE_CUDA(cudaFuncSetAttribute(chol_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_tile)));
  const int nsteps = (Q + NB - 1) / NB;
  for (int k0 = 0; k0 < Q; k0 += NB) {
    const int nb = std::min(NB, Q - k0), rem = Q - k0 - nb;
    chol_panel_kernel<<<dim3(1 + (rem + PT - 1) / PT, 1, nsets), PT, smem_panel, s>>>(A, Q, k0, nb, fail, stage);
    count_launch();
    if (rem > 0) {
      const int t = (rem + NB - 1) / NB;
      chol_update_kernel<<<dim3(t * (t + 1) / 2, 1, nsets), kTileThreads, smem_tile, s>>>(A, Q, k0, nb, fail);
      count_launch();
    }
  }
  chol_diag_writeback_kernel<<<dim3(nsteps, 1, nsets), PT, 0, s>>>(A, Q, fail, stage);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

void posterior_cov_large(const cmoe_gp& gp, SampleWork& w, int nc, int num, int gs, double jitter, cudaStream_t s) {
  posterior_cov_large(gp, w.P.p, w.dPs.p, w.V.p, w.mu.p, w.A.p, nc, num, gs, jitter, s);
}

void posterior_cov_large(const cmoe_gp& gp, const double* P, const int* dPs, double* V, double* mu, double* A, int nc,
                         int num, int gs, double jitter, cudaStream_t s) {
  const KernelSpec& spec = gp.spec;
  const int Q = num * (1 + gs), n = gp.n;
  build_mix_covariance(spec, gp.dX.p, gp.N, P, nc * num, dPs, gs, V, s);
  // the blocked kernel whatever the column count, so a set's solve does not depend on how many sets share its chunk
  trsm_lower_blocked(gp.dK.p, n, V, n, nc * Q, false, s);
  posterior_mean_points(gp, P, static_cast<size_t>(nc) * num, dPs, gs, mu, nullptr, s);
  const int t = (Q + NB - 1) / NB;
  const size_t smem_cov = (2 * static_cast<size_t>(NB) * LDT + 2 * static_cast<size_t>(NB) * spec.dim) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(cov_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_cov)));
  cov_tile_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kTileThreads, smem_cov, s>>>(spec, V, n, Q, P, num, dPs, gs, jitter,
                                                                              A);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

void zero_upper(int nsets, int Q, double* A, cudaStream_t s) {
  zero_upper_kernel<<<1024, 256, 0, s>>>(nsets, Q, A);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

void mirror_lower(int nsets, int Q, double* A, cudaStream_t s) {
  mirror_lower_kernel<<<1024, 256, 0, s>>>(nsets, Q, A);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

namespace {

// One chunk of nc sets whose points are in w.P: fills w.mu, w.A (factor), w.y, w.amin and w.fail.
void sample_chunk(const cmoe_gp& gp, SampleWork& w, int nc, int num, int gs, uint64_t seed, uint64_t draw0,
                  const double* dtable, double jitter, cudaStream_t s) {
  const int Q = num * (1 + gs);
  posterior_cov_large(gp, w, nc, num, gs, jitter, s);
  CMOE_CUDA(cudaMemsetAsync(w.fail.p, 0, nc * sizeof(int), s));
  potrf_batched(w.A.p, Q, nc, w.fail.p, w.stage, s);
  const int rb = (Q + kRowThreads - 1) / kRowThreads;
  const size_t smem_rows = static_cast<size_t>(std::min(Q, rb * kRowThreads)) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(sample_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_rows)));
  sample_rows_kernel<<<dim3(rb, nc), kRowThreads, smem_rows, s>>>(Q, 1 + gs, w.mu.p, w.A.p, seed, draw0, dtable, w.y.p,
                                                                  w.part_v.p, w.part_i.p);
  best_of_parts_kernel<false><<<(nc + 127) / 128, 128, 0, s>>>(nc, rb, w.part_v.p, w.part_i.p, w.amin.p, nullptr);
  count_launch(2);
  CMOE_CUDA(cudaGetLastError());
}

// Chunk driver shared by cmoe_gp_sample_joint and cmoe_gp_sample_global_optima.  fill(c0, nc) puts the points of
// sets [c0, c0 + nc) into w.P; collect(c0, nc) reads the results.  The first failing set stops the call.
void run_sampling(const cmoe_gp& gp, int num_sets, int num, const int* derivs_s, int gs, uint64_t seed,
                  uint64_t first_draw, const double* normals_table, double jitter,
                  const std::function<void(SampleWork&, int, int)>& fill,
                  const std::function<void(SampleWork&, int, int)>& collect) {
  cudaStream_t s = gp.stream;
  const int Q = num * (1 + gs), n = gp.n, dim = gp.spec.dim;
  const size_t per_set = sizeof(double) * (static_cast<size_t>(n) * Q + static_cast<size_t>(Q) * Q + 3 * Q +
                                           static_cast<size_t>(num) * dim) +
                         sizeof(double) * static_cast<size_t>((Q + NB - 1) / NB) * NB * NB + sizeof(int) * 2;
  const int chunk = static_cast<int>(chunk_items(num_sets, kSampleWorkspaceBytes, per_set, kMaxChunkSets));
  const size_t cq = static_cast<size_t>(chunk) * Q;
  const int rb = (Q + kRowThreads - 1) / kRowThreads;
  SampleWork& w = sample_work(gp);
  w.P.ensure(static_cast<size_t>(chunk) * num * dim);
  w.V.ensure(cq * n);
  w.A.ensure(cq * Q);
  w.mu.ensure(cq);
  w.y.ensure(cq);
  w.part_v.ensure(static_cast<size_t>(chunk) * rb);
  w.part_i.ensure(static_cast<size_t>(chunk) * rb);
  w.fail.ensure(chunk);
  w.amin.ensure(chunk);
  w.dPs.ensure(gs > 0 ? gs : 1);
  if (gs > 0) w.dPs.upload(derivs_s, gs, s);
  DevBuf<double>& dtable = w.table;
  if (normals_table) dtable.ensure(cq);
  std::vector<int> hfail(chunk);
  for (int c0 = 0; c0 < num_sets; c0 += chunk) {
    const int nc = std::min(chunk, num_sets - c0);
    fill(w, c0, nc);
    if (normals_table) dtable.upload(normals_table + static_cast<size_t>(c0) * Q, static_cast<size_t>(nc) * Q, s);
    sample_chunk(gp, w, nc, num, gs, seed, first_draw + c0, normals_table ? dtable.p : nullptr, jitter, s);
    w.fail.download(hfail.data(), nc, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    for (int c = 0; c < nc; ++c)
      if (hfail[c] != 0)
        throw Error(CMOE_ERR_SINGULAR,
                    "GP-Variance matrix singular. Check for duplicate points_to_sample or points_to_sample duplicating "
                    "points_sampled with 0 noise (or pass jitter > 0).",
                    hfail[c]);
    collect(w, c0, nc);
  }
  CMOE_CUDA(cudaStreamSynchronize(s));
}

void check_jitter(double jitter) {
  CMOE_REQUIRE(std::isfinite(jitter) && jitter >= 0.0, CMOE_ERR_INVALID_VALUE, "jitter must be finite and >= 0");
}

Box check_box(const double* bounds, int dim) {
  CMOE_REQUIRE(dim >= 1 && dim <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, 32]");
  CMOE_REQUIRE(bounds != nullptr, CMOE_ERR_INVALID_VALUE, "domain_bounds is NULL");
  Box b{};
  for (int i = 0; i < dim; ++i) {
    b.lo[i] = bounds[2 * i];
    b.hi[i] = bounds[2 * i + 1];
    CMOE_REQUIRE(std::isfinite(b.lo[i]) && std::isfinite(b.hi[i]) && b.lo[i] <= b.hi[i], CMOE_ERR_INVALID_VALUE,
                 "domain bounds must be finite with min <= max");
  }
  return b;
}

void launch_lhs(uint64_t seed, uint64_t first_draw, int num_sets, int num_pts, int dim, const Box& box, double* out,
                cudaStream_t s) {
  const size_t smem = static_cast<size_t>(num_pts) * sizeof(uint64_t);
  CMOE_CUDA(cudaFuncSetAttribute(lhs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  for (int c0 = 0; c0 < num_sets; c0 += 65535) {
    const int nc = std::min(65535, num_sets - c0);
    lhs_kernel<<<dim3(dim, nc), 256, smem, s>>>(seed, first_draw + c0, num_pts, dim, box,
                                                out + static_cast<size_t>(c0) * num_pts * dim);
    count_launch();
  }
  CMOE_CUDA(cudaGetLastError());
}

}  // namespace

}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_gp_sample_joint(const cmoe_gp* gp, const double* sets, int num_sets, int num_pts,
                                    const int* derivs_s, int g_s, uint64_t seed, uint64_t first_draw,
                                    const double* normals_table, double jitter, double* samples, int* argmin,
                                    double* mean, double* chol, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(gp != nullptr, CMOE_ERR_INVALID_VALUE, "gp is NULL");
    CMOE_REQUIRE(num_sets >= 1 && num_pts >= 1, CMOE_ERR_BOUNDS, "num_sets and num_pts must be >= 1");
    CMOE_REQUIRE(g_s >= 0 && g_s <= gp->spec.dim, CMOE_ERR_BOUNDS, "g_s out of range");
    for (int k = 0; k < g_s; ++k)
      CMOE_REQUIRE(derivs_s[k] >= 0 && derivs_s[k] < gp->spec.dim, CMOE_ERR_BOUNDS, "derivative index out of range");
    CMOE_REQUIRE(static_cast<long long>(num_pts) * (1 + g_s) <= kMaxSampleQ, CMOE_ERR_BOUNDS,
                 "num_pts*(1+g_s) must be <= 8192");
    check_jitter(jitter);
    require_device(gp->device);
    const int Q = num_pts * (1 + g_s), dim = gp->spec.dim;
    cudaStream_t s = gp->stream;
    run_sampling(
        *gp, num_sets, num_pts, derivs_s, g_s, seed, first_draw, normals_table, jitter,
        [&](SampleWork& w, int c0, int nc) {
          w.P.upload(sets + static_cast<size_t>(c0) * num_pts * dim, static_cast<size_t>(nc) * num_pts * dim, s);
        },
        [&](SampleWork& w, int c0, int nc) {
          const size_t off = static_cast<size_t>(c0) * Q, cnt = static_cast<size_t>(nc) * Q;
          if (samples) w.y.download(samples + off, cnt, s);
          if (argmin) w.amin.download(argmin + c0, nc, s);
          if (mean) w.mu.download(mean + off, cnt, s);
          if (chol) {
            zero_upper(nc, Q, w.A.p, s);
            w.A.download(chol + off * Q, cnt * Q, s);
          }
          CMOE_CUDA(cudaStreamSynchronize(s));
        });
  });
}

extern "C" int cmoe_gp_posterior_large(const cmoe_gp* gp, const double* sets, int num_sets, int num_pts,
                                       const int* derivs_s, int g_s, double* mean, double* var, double* chol_var,
                                       int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(gp != nullptr, CMOE_ERR_INVALID_VALUE, "gp is NULL");
    CMOE_REQUIRE(num_sets >= 1 && num_pts >= 1, CMOE_ERR_BOUNDS, "num_sets and num_pts must be >= 1");
    CMOE_REQUIRE(g_s >= 0 && g_s <= gp->spec.dim, CMOE_ERR_BOUNDS, "g_s out of range");
    for (int k = 0; k < g_s; ++k)
      CMOE_REQUIRE(derivs_s[k] >= 0 && derivs_s[k] < gp->spec.dim, CMOE_ERR_BOUNDS, "derivative index out of range");
    CMOE_REQUIRE(static_cast<long long>(num_pts) * (1 + g_s) <= kMaxSampleQ, CMOE_ERR_BOUNDS,
                 "num_pts*(1+g_s) must be <= 8192");
    require_device(gp->device);
    const int Q = num_pts * (1 + g_s), n = gp->n, dim = gp->spec.dim;
    cudaStream_t s = gp->stream;
    const size_t per_set = sizeof(double) * (static_cast<size_t>(n) * Q + static_cast<size_t>(Q) * Q + Q +
                                             static_cast<size_t>(num_pts) * dim +
                                             static_cast<size_t>((Q + NB - 1) / NB) * NB * NB) +
                           sizeof(int);
    const int chunk = static_cast<int>(chunk_items(num_sets, kSampleWorkspaceBytes, per_set, kMaxChunkSets));
    SampleWork& w = sample_work(*gp);
    w.P.ensure(static_cast<size_t>(chunk) * num_pts * dim);
    w.V.ensure(static_cast<size_t>(chunk) * Q * n);
    w.A.ensure(static_cast<size_t>(chunk) * Q * Q);
    w.mu.ensure(static_cast<size_t>(chunk) * Q);
    w.fail.ensure(chunk);
    w.dPs.ensure(g_s > 0 ? g_s : 1);
    if (g_s > 0) w.dPs.upload(derivs_s, g_s, s);
    std::vector<int> hfail(chunk);
    for (int c0 = 0; c0 < num_sets; c0 += chunk) {
      const int nc = std::min(chunk, num_sets - c0);
      const size_t off = static_cast<size_t>(c0) * Q, cnt = static_cast<size_t>(nc) * Q;
      w.P.upload(sets + static_cast<size_t>(c0) * num_pts * dim, static_cast<size_t>(nc) * num_pts * dim, s);
      posterior_cov_large(*gp, w, nc, num_pts, g_s, 0.0, s);
      if (mean) w.mu.download(mean + off, cnt, s);
      if (var) {
        mirror_lower(nc, Q, w.A.p, s);
        w.A.download(var + off * Q, cnt * Q, s);
      }
      if (chol_var) {
        CMOE_CUDA(cudaMemsetAsync(w.fail.p, 0, nc * sizeof(int), s));
        potrf_batched(w.A.p, Q, nc, w.fail.p, w.stage, s);
        w.fail.download(hfail.data(), nc, s);
        CMOE_CUDA(cudaStreamSynchronize(s));
        for (int c = 0; c < nc; ++c)
          if (hfail[c] != 0)
            throw Error(CMOE_ERR_SINGULAR,
                        "GP-Variance matrix singular. Check for duplicate points_to_sample or points_to_sample "
                        "duplicating points_sampled with 0 noise.",
                        hfail[c]);
        zero_upper(nc, Q, w.A.p, s);
        w.A.download(chol_var + off * Q, cnt * Q, s);
      }
      CMOE_CUDA(cudaStreamSynchronize(s));
    }
  });
}

extern "C" int cmoe_latin_hypercube(uint64_t seed, uint64_t first_draw, int num_sets, int num_pts, int dim,
                                    const double* domain_bounds, double* out, int device) {
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(num_sets >= 1 && num_pts >= 1 && num_pts <= kMaxSampleQ, CMOE_ERR_BOUNDS,
                 "num_sets must be >= 1 and num_pts in [1, 8192]");
    const Box box = check_box(domain_bounds, dim);
    require_device(device);
    cudaStream_t s;
    CMOE_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    try {
      const size_t cnt = static_cast<size_t>(num_sets) * num_pts * dim;
      DevBuf<double> d(cnt);
      launch_lhs(seed, first_draw, num_sets, num_pts, dim, box, d.p, s);
      d.download(out, cnt, s);
      CMOE_CUDA(cudaStreamSynchronize(s));
    } catch (...) {
      cudaStreamDestroy(s);
      throw;
    }
    cudaStreamDestroy(s);
  });
}

extern "C" int cmoe_gp_sample_global_optima(const cmoe_gp* gp, int num_optima, int inner_number,
                                            const double* domain_bounds, uint64_t seed, uint64_t first_draw,
                                            double jitter, double* points_optima, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(gp != nullptr, CMOE_ERR_INVALID_VALUE, "gp is NULL");
    CMOE_REQUIRE(num_optima >= 1 && inner_number >= 1 && inner_number <= kMaxSampleQ, CMOE_ERR_BOUNDS,
                 "num_optima must be >= 1 and inner_number in [1, 8192]");
    const int dim = gp->spec.dim;
    const Box box = check_box(domain_bounds, dim);
    check_jitter(jitter);
    require_device(gp->device);
    cudaStream_t s = gp->stream;
    run_sampling(
        *gp, num_optima, inner_number, nullptr, 0, seed, first_draw, nullptr, jitter,
        [&](SampleWork& w, int c0, int nc) { launch_lhs(seed, first_draw + c0, nc, inner_number, dim, box, w.P.p, s); },
        [&](SampleWork& w, int c0, int nc) {
          w.opt.ensure(static_cast<size_t>(nc) * dim);
          gather_kernel<<<(nc * dim + 255) / 256, 256, 0, s>>>(nc, inner_number, dim, w.P.p, w.amin.p, w.opt.p);
          count_launch();
          CMOE_CUDA(cudaGetLastError());
          w.opt.download(points_optima + static_cast<size_t>(c0) * dim, static_cast<size_t>(nc) * dim, s);
          CMOE_CUDA(cudaStreamSynchronize(s));
        });
  });
}

// Batched Cholesky of device-resident matrices against a loop of potrf_lower over the same matrices (both re-factor a
// fresh copy each repeat; the copies are outside the timed region).
extern "C" int cmoe_bench_cholesky_batched(const double* mats, int num_mats, int Q, int repeats, int device,
                                           double* usec_batched, double* usec_loop, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_mats >= 1 && Q >= 1 && Q <= kMaxSampleQ && num_mats <= kMaxChunkSets && repeats >= 1,
                 CMOE_ERR_BOUNDS, "num_mats in [1, 4096], Q in [1, 8192], repeats >= 1");
    require_device(device);
    cudaStream_t s;
    CMOE_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    try {
      const size_t cnt = static_cast<size_t>(num_mats) * Q * Q;
      DevBuf<double> M0(cnt), W(cnt);
      DevBuf<int> fail(num_mats);
      DevBuf<double> stage;
      M0.upload(mats, cnt, s);
      double tb = 0.0, tl = 0.0;
      for (int r = 0; r <= repeats; ++r) {
        CMOE_CUDA(cudaMemcpyAsync(W.p, M0.p, cnt * sizeof(double), cudaMemcpyDeviceToDevice, s));
        CMOE_CUDA(cudaMemsetAsync(fail.p, 0, num_mats * sizeof(int), s));
        EventTimer a;
        a.start(s);
        potrf_batched(W.p, Q, num_mats, fail.p, stage, s);
        a.stop(s);
        const double ta = a.ms();
        std::vector<int> hf(num_mats);
        fail.download(hf.data(), num_mats, s);
        CMOE_CUDA(cudaStreamSynchronize(s));
        for (int b = 0; b < num_mats; ++b)
          if (hf[b]) throw Error(CMOE_ERR_SINGULAR, "matrix singular", hf[b]);
        CMOE_CUDA(cudaMemcpyAsync(W.p, M0.p, cnt * sizeof(double), cudaMemcpyDeviceToDevice, s));
        EventTimer c;
        c.start(s);
        for (int b = 0; b < num_mats; ++b) potrf_lower(W.p + static_cast<size_t>(b) * Q * Q, Q, fail.p + b, s);
        c.stop(s);
        const double tc = c.ms();
        if (r > 0) {
          tb += ta;
          tl += tc;
        }
      }
      *usec_batched = tb * 1e3 / repeats;
      *usec_loop = tl * 1e3 / repeats;
      CMOE_CUDA(cudaStreamSynchronize(s));
    } catch (...) {
      cudaStreamDestroy(s);
      throw;
    }
    cudaStreamDestroy(s);
  });
}

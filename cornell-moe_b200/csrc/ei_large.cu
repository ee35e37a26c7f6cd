// q-EI Monte-Carlo value and reverse-mode gradient for union sets of up to 8192 rows (DESIGN.md K16).
//
// The same estimator as ei.cu (ExpectedImprovementEvaluator, reference gpp_math.cpp:1991-2126) without ei.cu's per-thread
// copy of a sample's normals and without the grad-Cholesky tensor (q U^2 d doubles per candidate).  Per chunk of
// candidates (union set = candidate's q points + the p pending points, U = q + p rows):
//   posterior       the K8 stages (posterior_cov_large): mu, Var + 1e-6 I, C C^T = Var (potrf_batched)
//   forward         ei_mc_tile_kernel: Y - mu = C W as DMMA 64-row x 64-sample tiles; the best improvement
//                   best_so_far - y_j (from 0) and its row per (row block, sample); ei_winner_kernel combines the row
//                   blocks in ascending order, ei_value_kernel sums the improvements in a fixed order
//   winners         ei_bucket_kernel: each row's winning samples in ascending order; ei_cbar_kernel:
//                   Cbar = -tril(E W^T) / num_mc, E the winner indicator (a gather over the winning samples)
//   adjoint         M = C^T Cbar (DMMA, lower tiles), S = M mirrored (= Phi(M) + Phi(M)^T), X = C^-T S,
//                   T = C^-T X^T = 2 Sigmabar (blocked triangular solves), R = B T[:, :q] with B = K^-1 K(X, P) (DMMA)
//   gradient        ei_grad_kernel: for the q candidate points
//                     xbar_i = sum_b T_ib dK(p_i, p_b) - sum_r dK(p_i, x_r) R_ri + mubar_i sum_r dK(p_i, x_r) alpha_r,
//                   mubar = -cnt / num_mc, dK the derivative in p_i (grad_cov_entry)
// The normals W [num_mc][U] are the table, or the Philox table (draw s = sample s, normals 2k, 2k+1 from call k) written
// once per call: every candidate uses the same W (common random numbers), so it is stored once, not per candidate.
// Every kernel treats the candidates of a chunk independently and reduces in a fixed order, so a candidate's result does
// not depend on the batch or the chunking.
#include <algorithm>
#include <climits>

#include "device_math.cuh"
#include "internal.cuh"
#include "linalg_dev.cuh"

namespace cmoe {

namespace {

constexpr int kTileThreads = 128;  // four warps of a 64 x 64 DMMA tile (tile_mma64)
constexpr int kBucketThreads = 1024;

// (v, i) beats (bv, bi): larger improvement, ties to the lower row; row -1 (no improvement) is the lowest.  Applied in
// any order this leaves the first maximiser of a strict `>` scan from (0, -1) (gpp_math.cpp:2092).
__device__ __forceinline__ bool beats(double v, int i, double bv, int bi) { return v > bv || (v == bv && i < bi); }

// one 64-deep chunk of the NN product tile:  As[k][r] = A(r0 + r, k0 + k), Bs[k][c] = B(k0 + k, c0 + c), A and B
// column-major (lda, ldb), zero outside rows x cols x kmax
__device__ __forceinline__ void load_nn_chunk(const double* A, size_t lda, int rows, const double* B, size_t ldb,
                                              int cols, int k0, int kmax, double* As, double* Bs) {
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    {
      const int r = e % NB, k = e / NB;  // consecutive threads, consecutive rows of one A column
      const bool ok = r < rows && k0 + k < kmax;
      cp_async8(As + k * LDT + r, ok ? A + (k0 + k) * lda + r : A, ok);
    }
    {
      const int k = e % NB, c = e / NB;  // consecutive threads, consecutive k of one B column
      const bool ok = c < cols && k0 + k < kmax;
      cp_async8(Bs + k * LDT + c, ok ? B + c * ldb + k0 + k : B, ok);
    }
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
}

// --------------------------------------------------------------------------------------------------------------
// Forward tiles, grid (sample blocks, row blocks, candidates): Y - mu = C W for 64 rows x 64 samples (C's columns past
// the tile's last row are zero, so the depth stops there), then per sample the best (improvement, row) of the tile's
// rows -> part_v / part_i [candidate][row block][num_mc].
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTileThreads) ei_mc_tile_kernel(int U, int num_mc, double best_so_far,
                                                                  const double* __restrict__ W,
                                                                  const double* __restrict__ mu,
                                                                  const double* __restrict__ C,
                                                                  double* __restrict__ part_v,
                                                                  int* __restrict__ part_i) {
  extern __shared__ double smem[];
  double* As = smem;
  double* Bs = smem + NB * LDT;
  __shared__ double hv[NB];
  __shared__ int hi[NB];
  const int set = blockIdx.z, s0 = blockIdx.x * NB, r0 = blockIdx.y * NB;
  const int rows = min(NB, U - r0), cols = min(NB, num_mc - s0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  const double* Cr = C + static_cast<size_t>(set) * U * U + r0;
  const double* Ws = W + static_cast<size_t>(s0) * U;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  const int kmax = r0 + rows;
  for (int k0 = 0; k0 < kmax; k0 += NB) {
    if (k0 > 0) __syncthreads();
    load_nn_chunk(Cr, U, rows, Ws, U, cols, k0, kmax, As, Bs);
    tile_mma64(As, Bs, acc, wm, wn, lr, lc);
  }
  const double* mus = mu + static_cast<size_t>(set) * U + r0;
  double bv[4][2];
  int bi[4][2];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      bv[j][h] = 0.0;
      bi[j][h] = -1;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = wm + i * 8 + lr;
        if (r < rows) {
          const double v = best_so_far - (mus[r] + acc[i][j][h]);
          if (beats(v, r0 + r, bv[j][h], bi[j][h])) {
            bv[j][h] = v;
            bi[j][h] = r0 + r;
          }
        }
      }
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv[j][h], off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[j][h], off);
        if (beats(ov, oi, bv[j][h], bi[j][h])) {
          bv[j][h] = ov;
          bi[j][h] = oi;
        }
      }
    }
  if (wm == 32 && lr == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        hv[wn + j * 8 + lc * 2 + h] = bv[j][h];
        hi[wn + j * 8 + lc * 2 + h] = bi[j][h];
      }
  }
  __syncthreads();
  if (wm == 0 && lr == 0) {
    const size_t base = (static_cast<size_t>(set) * gridDim.y + blockIdx.y) * num_mc + s0;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h;
        if (c < cols) {
          double v = bv[j][h];
          int i = bi[j][h];
          if (beats(hv[c], hi[c], v, i)) {
            v = hv[c];
            i = hi[c];
          }
          part_v[base + c] = v;
          part_i[base + c] = i;
        }
      }
  }
}

// per (candidate, sample): the row blocks in ascending order -> improvement and winning row (-1: none)
__global__ void __launch_bounds__(256) ei_winner_kernel(int num_mc, int nrb, const double* __restrict__ part_v,
                                                        const int* __restrict__ part_i, double* __restrict__ imp,
                                                        int* __restrict__ win) {
  const int set = blockIdx.y, s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= num_mc) return;
  double bv = 0.0;
  int bi = -1;
  for (int b = 0; b < nrb; ++b) {
    const size_t o = (static_cast<size_t>(set) * nrb + b) * num_mc + s;
    if (beats(part_v[o], part_i[o], bv, bi)) {
      bv = part_v[o];
      bi = part_i[o];
    }
  }
  imp[static_cast<size_t>(set) * num_mc + s] = bv;
  win[static_cast<size_t>(set) * num_mc + s] = bi;
}

__global__ void __launch_bounds__(256) ei_value_kernel(int num_mc, const double* __restrict__ imp,
                                                       double* __restrict__ ei) {
  __shared__ double red[8];
  const int set = blockIdx.x;
  double part = 0.0;
  for (int s = threadIdx.x; s < num_mc; s += blockDim.x) part += imp[static_cast<size_t>(set) * num_mc + s];
  const double total = block_sum(part, red);
  if (threadIdx.x == 0) ei[set] = total / static_cast<double>(num_mc);
}

// --------------------------------------------------------------------------------------------------------------
// One CTA per candidate: cnt[j] = samples row j wins, start[j] = offset of row j's list in order[], and order[] = the
// winning samples grouped by row, ascending within a row (warps take their turn in sample order).
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBucketThreads) ei_bucket_kernel(int U, int num_mc, const int* __restrict__ win,
                                                                   int* __restrict__ cnt, int* __restrict__ start,
                                                                   int* __restrict__ order) {
  extern __shared__ int cur[];  // [U]
  __shared__ int part[kBucketThreads];
  const int set = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int* wc = win + static_cast<size_t>(set) * num_mc;
  for (int j = tid; j < U; j += blockDim.x) cur[j] = 0;
  __syncthreads();
  for (int s = tid; s < num_mc; s += blockDim.x)
    if (wc[s] >= 0) atomicAdd(&cur[wc[s]], 1);
  __syncthreads();
  const int per = (U + kBucketThreads - 1) / kBucketThreads, lo = min(U, tid * per), hi = min(U, lo + per);
  int local = 0;
  for (int j = lo; j < hi; ++j) local += cur[j];
  part[tid] = local;
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int t = 0; t < kBucketThreads; ++t) {
      const int c = part[t];
      part[t] = run;
      run += c;
    }
  }
  __syncthreads();
  int off = part[tid];
  for (int j = lo; j < hi; ++j) {
    const int c = cur[j];
    cnt[static_cast<size_t>(set) * U + j] = c;
    start[static_cast<size_t>(set) * U + j] = off;
    cur[j] = off;
    off += c;
  }
  __syncthreads();
  int* oc = order + static_cast<size_t>(set) * num_mc;
  for (int c0 = 0; c0 < num_mc; c0 += kBucketThreads) {
    const int s = c0 + tid;
    const int j = s < num_mc ? wc[s] : -1;
    for (int w = 0; w < kBucketThreads / 32; ++w) {
      if (warp == w) {
        const unsigned mask = __match_any_sync(0xffffffffu, j);
        const int rank = __popc(mask & ((1u << lane) - 1u));
        if (j >= 0) oc[cur[j] + rank] = s;
        __syncwarp();
        if (j >= 0 && rank == 0) cur[j] += __popc(mask);
      }
      __syncthreads();
    }
  }
}

// Cbar (column-major, [candidate][U][U]): (j, i) = -sum of W[s][i] over the samples s that row j wins, in ascending
// order, / num_mc for i <= j; 0 above the diagonal.  Thread (j, i) with i fastest: the W reads of a warp are coalesced.
__global__ void __launch_bounds__(256) ei_cbar_kernel(int U, int num_mc, const double* __restrict__ W,
                                                      const int* __restrict__ cnt, const int* __restrict__ start,
                                                      const int* __restrict__ order, double* __restrict__ Cbar) {
  const int set = blockIdx.y;
  const size_t o = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (o >= static_cast<size_t>(U) * U) return;
  const int j = static_cast<int>(o / U), i = static_cast<int>(o % U);
  double acc = 0.0;
  if (i <= j) {
    const int b = start[static_cast<size_t>(set) * U + j], c = cnt[static_cast<size_t>(set) * U + j];
    const int* oc = order + static_cast<size_t>(set) * num_mc + b;
    for (int t = 0; t < c; ++t) acc += W[static_cast<size_t>(oc[t]) * U + i];
    acc = -acc / static_cast<double>(num_mc);
  }
  Cbar[static_cast<size_t>(set) * U * U + static_cast<size_t>(i) * U + j] = acc;
}

// M = C^T Cbar on the lower 64 x 64 tiles (the only ones Phi reads); grid (tiles, 1, candidates)
__global__ void __launch_bounds__(kTileThreads) ei_ctc_kernel(int U, const double* __restrict__ C,
                                                              const double* __restrict__ Cbar,
                                                              double* __restrict__ M) {
  extern __shared__ double smem[];
  double* As = smem;
  double* Bs = smem + NB * LDT;
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int set = blockIdx.z, row0 = ti * NB, col0 = tj * NB;
  const int rows = min(NB, U - row0), cols = min(NB, U - col0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  const size_t off = static_cast<size_t>(set) * U * U;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  gram_tile_accumulate(C + off + static_cast<size_t>(row0) * U, Cbar + off + static_cast<size_t>(col0) * U, U, rows,
                       cols, As, Bs, acc, wm, wn, lr, lc);
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = wm + i * 8 + lr, c = wn + j * 8 + lc * 2 + h;
        if (r < rows && c < cols && row0 + r >= col0 + c)
          M[off + static_cast<size_t>(col0 + c) * U + row0 + r] = acc[i][j][h];
      }
}

constexpr size_t kTileSmem = 2 * static_cast<size_t>(NB) * LDT * sizeof(double);

// out = in^T for nsets U x U matrices
__global__ void __launch_bounds__(256) transpose_kernel(int U, const double* __restrict__ in,
                                                        double* __restrict__ out) {
  const int set = blockIdx.y;
  const size_t o = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (o >= static_cast<size_t>(U) * U) return;
  const size_t off = static_cast<size_t>(set) * U * U;
  const int r = static_cast<int>(o % U), c = static_cast<int>(o / U);
  out[off + o] = in[off + static_cast<size_t>(r) * U + c];
}

// Out = A B (column-major; A m x kd, B kd x nn), 64 x 64 DMMA tiles; grid (row blocks, column blocks, batch)
__global__ void __launch_bounds__(kTileThreads) gemm_nn_kernel(int m, int nn, int kd, const double* __restrict__ A,
                                                               int lda, size_t sa, const double* __restrict__ B,
                                                               int ldb, size_t sb, double* __restrict__ Out, int ldo,
                                                               size_t so) {
  extern __shared__ double smem[];
  double* As = smem;
  double* Bs = smem + NB * LDT;
  const int z = blockIdx.z, r0 = blockIdx.x * NB, c0 = blockIdx.y * NB;
  const int rows = min(NB, m - r0), cols = min(NB, nn - c0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  const double* Az = A + z * sa + r0;
  const double* Bz = B + z * sb + static_cast<size_t>(c0) * ldb;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  for (int k0 = 0; k0 < kd; k0 += NB) {
    if (k0 > 0) __syncthreads();
    load_nn_chunk(Az, lda, rows, Bz, ldb, cols, k0, kd, As, Bs);
    tile_mma64(As, Bs, acc, wm, wn, lr, lc);
  }
  double* Oz = Out + z * so;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = wm + i * 8 + lr, c = wn + j * 8 + lc * 2 + h;
        if (r < rows && c < cols) Oz[static_cast<size_t>(c0 + c) * ldo + r0 + r] = acc[i][j][h];
      }
}

// --------------------------------------------------------------------------------------------------------------
// Gradient of candidate point i < q, grid (q, candidates).  Threads = (component delta, slice of the N + U terms);
// slices are combined in a fixed order.  T = 2 Sigmabar (column-major U x U), R = B T[:, :q] (n x q, ld n).
// --------------------------------------------------------------------------------------------------------------
constexpr int kGradThreads = 128;

__global__ void __launch_bounds__(kGradThreads) ei_grad_kernel(const __grid_constant__ KernelSpec spec, int N,
                                                               const double* __restrict__ X,
                                                               const double* __restrict__ alpha,
                                                               const double* __restrict__ P, int U, int q, int num_mc,
                                                               const double* __restrict__ T,
                                                               const double* __restrict__ R,
                                                               const int* __restrict__ cnt,
                                                               double* __restrict__ grad) {
  __shared__ double Pi[CMOE_MAX_DIM];
  __shared__ double red[kGradThreads];
  const int i = blockIdx.x, set = blockIdx.y, dim = spec.dim, b1 = 1 + spec.g, n = N * b1, tid = threadIdx.x;
  const double* Pset = P + static_cast<size_t>(set) * U * dim;
  for (int e = tid; e < dim; e += blockDim.x) Pi[e] = Pset[static_cast<size_t>(i) * dim + e];
  __syncthreads();
  const int nparts = kGradThreads / dim, delta = tid % dim, part = tid / dim;
  const double mubar = -static_cast<double>(cnt[static_cast<size_t>(set) * U + i]) / static_cast<double>(num_mc);
  const double* Ri = R + (static_cast<size_t>(set) * q + i) * n;
  const double* Ti = T + static_cast<size_t>(set) * U * U + i;  // row i: Ti[b U]
  double acc = 0.0;
  if (part < nparts) {
    for (int t = part; t < N + U; t += nparts) {
      if (t < N) {
        const double* xj = X + static_cast<size_t>(t) * dim;
        const KParts kp = kernel_parts(spec, weighted_sqdist(spec, Pi, xj));
        for (int cc = 0; cc < b1; ++cc) {
          const int r = t * b1 + cc;
          const double g = grad_cov_entry(spec, kp, Pi, xj, -1, cc ? spec.derivs[cc - 1] : -1, delta);
          acc = fma(g, fma(mubar, alpha[r], -Ri[r]), acc);
        }
      } else {
        const int b = t - N;
        const double* pb = Pset + static_cast<size_t>(b) * dim;
        const KParts kp = kernel_parts(spec, weighted_sqdist(spec, Pi, pb));
        acc = fma(grad_cov_entry(spec, kp, Pi, pb, -1, -1, delta), Ti[static_cast<size_t>(b) * U], acc);
      }
    }
  }
  red[tid] = acc;
  __syncthreads();
  if (tid < dim) {
    double t = 0.0;
    for (int pp = 0; pp < nparts; ++pp) t += red[pp * dim + tid];
    grad[(static_cast<size_t>(set) * q + i) * dim + tid] = t;
  }
}


// Device scratch of one chunk beyond the K8 workspace.
struct EiLargeWork {
  DevBuf<double> part_v, imp, ei, T1, T2, R, grad;
  DevBuf<int> part_i, win, cnt, start, order;
};

void ei_large_chunk(const cmoe_gp& gp, SampleWork& w, EiLargeWork& e, const double* candidates, int nc, int q,
                    const double* Xp, int p, int num_mc, double best_so_far, const double* W, double* ei_host,
                    double* grad_host) {
  cudaStream_t s = gp.stream;
  const int U = q + p, dim = gp.spec.dim, n = gp.n;
  const bool want_grad = grad_host != nullptr;
  {
    std::vector<double> h(static_cast<size_t>(nc) * U * dim);
    for (int c = 0; c < nc; ++c) {
      double* dst = h.data() + static_cast<size_t>(c) * U * dim;
      std::copy(candidates + static_cast<size_t>(c) * q * dim, candidates + static_cast<size_t>(c + 1) * q * dim, dst);
      if (p) std::copy(Xp, Xp + static_cast<size_t>(p) * dim, dst + static_cast<size_t>(q) * dim);
    }
    w.P.upload(h.data(), h.size(), s);
    CMOE_CUDA(cudaStreamSynchronize(s));  // h goes out of scope
  }
  // mu, Var + 1e-6 I (gpp_math.cpp:2000-2002) and its factor C, upper triangle zero
  posterior_cov_large(gp, w, nc, U, 0, 1.0e-6, s);
  CMOE_CUDA(cudaMemsetAsync(w.fail.p, 0, nc * sizeof(int), s));
  potrf_batched(w.A.p, U, nc, w.fail.p, w.stage, s);
  std::vector<int> hfail(nc);
  w.fail.download(hfail.data(), nc, s);
  CMOE_CUDA(cudaStreamSynchronize(s));
  for (int c = 0; c < nc; ++c)
    if (hfail[c] != 0)
      throw Error(CMOE_ERR_SINGULAR,
                  "GP-Variance matrix singular. Check for duplicate points_to_sample/being_sampled or "
                  "points_to_sample/being_sampled duplicating points_sampled with 0 noise.",
                  hfail[c]);
  zero_upper(nc, U, w.A.p, s);
  // forward
  const int nrb = (U + NB - 1) / NB, nsb = (num_mc + NB - 1) / NB;
  CMOE_CUDA(cudaFuncSetAttribute(ei_mc_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(kTileSmem)));
  ei_mc_tile_kernel<<<dim3(nsb, nrb, nc), kTileThreads, kTileSmem, s>>>(U, num_mc, best_so_far, W, w.mu.p, w.A.p,
                                                                        e.part_v.p, e.part_i.p);
  ei_winner_kernel<<<dim3((num_mc + 255) / 256, nc), 256, 0, s>>>(num_mc, nrb, e.part_v.p, e.part_i.p, e.imp.p,
                                                                  e.win.p);
  ei_value_kernel<<<nc, 256, 0, s>>>(num_mc, e.imp.p, e.ei.p);
  count_launch(3);
  CMOE_CUDA(cudaGetLastError());
  e.ei.download(ei_host, nc, s);
  if (want_grad) {
    const size_t UU = static_cast<size_t>(U) * U;
    const unsigned gUU = static_cast<unsigned>((UU + 255) / 256);
    // B = K^-1 K(X, P) = L^-T V in place of V (cov_tile_kernel has consumed V)
    trsm_lower_blocked(gp.dK.p, n, w.V.p, n, nc * U, true, s);
    const size_t smem_bucket = static_cast<size_t>(U) * sizeof(int);
    CMOE_CUDA(cudaFuncSetAttribute(ei_bucket_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(smem_bucket)));
    ei_bucket_kernel<<<nc, kBucketThreads, smem_bucket, s>>>(U, num_mc, e.win.p, e.cnt.p, e.start.p, e.order.p);
    ei_cbar_kernel<<<dim3(gUU, nc), 256, 0, s>>>(U, num_mc, W, e.cnt.p, e.start.p, e.order.p, e.T1.p);
    count_launch(2);
    cholesky_adjoint(w.A.p, U, nc, e.T1.p, e.T2.p, s);
    // R = B T[:, :q]
    gemm_nn(n, q, U, w.V.p, n, static_cast<size_t>(n) * U, e.T1.p, U, UU, e.R.p, n, static_cast<size_t>(n) * q, nc, s);
    ei_grad_kernel<<<dim3(q, nc), kGradThreads, 0, s>>>(gp.spec, gp.N, gp.dX.p, gp.dKinvY.p, w.P.p, U, q, num_mc,
                                                        e.T1.p, e.R.p, e.cnt.p, e.grad.p);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    e.grad.download(grad_host, static_cast<size_t>(nc) * q * dim, s);
  }
  CMOE_CUDA(cudaStreamSynchronize(s));
}

}  // namespace

void gemm_nn(int m, int nn, int kd, const double* A, int lda, size_t sa, const double* B, int ldb, size_t sb,
             double* Out, int ldo, size_t so, int batch, cudaStream_t s) {
  CMOE_CUDA(cudaFuncSetAttribute(gemm_nn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(kTileSmem)));
  gemm_nn_kernel<<<dim3((m + NB - 1) / NB, (nn + NB - 1) / NB, batch), kTileThreads, kTileSmem, s>>>(
      m, nn, kd, A, lda, sa, B, ldb, sb, Out, ldo, so);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

void cholesky_adjoint(const double* C, int U, int nc, double* T1, double* T2, cudaStream_t s) {
  const size_t UU = static_cast<size_t>(U) * U;
  const unsigned gUU = static_cast<unsigned>((UU + 255) / 256);
  const int t = (U + NB - 1) / NB;
  CMOE_CUDA(cudaFuncSetAttribute(ei_ctc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(kTileSmem)));
  ei_ctc_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kTileThreads, kTileSmem, s>>>(U, C, T1, T2);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
  mirror_lower(nc, U, T2, s);  // S = Phi(M) + Phi(M)^T
  for (int c = 0; c < nc; ++c)  // X = C^-T S
    trsm_lower_blocked(C + c * UU, U, T2 + c * UU, U, U, true, s);
  transpose_kernel<<<dim3(gUU, nc), 256, 0, s>>>(U, T2, T1);
  count_launch();
  for (int c = 0; c < nc; ++c)  // T = C^-T X^T = C^-T S C^-1 = 2 Sigmabar
    trsm_lower_blocked(C + c * UU, U, T1 + c * UU, U, U, true, s);
}

void ei_large_eval_batch(const cmoe_gp& gp, const double* candidates, int nc, int q, const double* Xp, int p,
                         int num_mc, double best_so_far, uint64_t seed, const double* dtable, double* ei_host,
                         double* grad_host) {
  CMOE_REQUIRE(q >= 1 && p >= 0 && num_mc >= 1, CMOE_ERR_BOUNDS, "q >= 1, p >= 0, num_mc >= 1 required");
  CMOE_REQUIRE(static_cast<long long>(q) + p <= kMaxSampleQ, CMOE_ERR_BOUNDS, "q + p must be <= 8192");
  CMOE_REQUIRE(static_cast<size_t>(num_mc) * (q + p) <= kSampleWorkspaceBytes / sizeof(double), CMOE_ERR_BOUNDS,
               "num_mc * (q + p) normals must fit in 2 GiB");
  cudaStream_t s = gp.stream;
  const int U = q + p, dim = gp.spec.dim, n = gp.n;
  const bool want_grad = grad_host != nullptr;
  DevBuf<double> Wgen;
  const double* W = dtable;
  if (W == nullptr) {
    Wgen.alloc(static_cast<size_t>(num_mc) * U);
    philox_normals_device(seed, 0, num_mc, U, Wgen.p, s);
    W = Wgen.p;
  }
  const size_t UU = static_cast<size_t>(U) * U, nrb = (U + NB - 1) / NB;
  const size_t per_cand =
      sizeof(double) * (static_cast<size_t>(n) * U + UU + U + static_cast<size_t>(U) * dim + nrb * NB * NB + 1 +
                        nrb * num_mc + num_mc) +
      sizeof(int) * (2 + nrb * num_mc + num_mc) +
      (want_grad ? sizeof(double) * (2 * UU + static_cast<size_t>(n) * q + static_cast<size_t>(q) * dim) +
                       sizeof(int) * (2 * static_cast<size_t>(U) + num_mc)
                 : 0);
  const int chunk = static_cast<int>(chunk_items(nc, kSampleWorkspaceBytes, per_cand, kMaxChunkSets));
  SampleWork& w = sample_work(gp);
  w.P.ensure(static_cast<size_t>(chunk) * U * dim);
  w.V.ensure(static_cast<size_t>(chunk) * U * n);
  w.A.ensure(static_cast<size_t>(chunk) * UU);
  w.mu.ensure(static_cast<size_t>(chunk) * U);
  w.fail.ensure(chunk);
  w.dPs.ensure(1);
  EiLargeWork e;
  e.part_v.alloc(static_cast<size_t>(chunk) * nrb * num_mc);
  e.part_i.alloc(static_cast<size_t>(chunk) * nrb * num_mc);
  e.imp.alloc(static_cast<size_t>(chunk) * num_mc);
  e.win.alloc(static_cast<size_t>(chunk) * num_mc);
  e.ei.alloc(chunk);
  if (want_grad) {
    e.T1.alloc(static_cast<size_t>(chunk) * UU);
    e.T2.alloc(static_cast<size_t>(chunk) * UU);
    e.R.alloc(static_cast<size_t>(chunk) * n * q);
    e.grad.alloc(static_cast<size_t>(chunk) * q * dim);
    e.cnt.alloc(static_cast<size_t>(chunk) * U);
    e.start.alloc(static_cast<size_t>(chunk) * U);
    e.order.alloc(static_cast<size_t>(chunk) * num_mc);
  }
  for (int c0 = 0; c0 < nc; c0 += chunk) {
    const int nb = std::min(chunk, nc - c0);
    ei_large_chunk(gp, w, e, candidates + static_cast<size_t>(c0) * q * dim, nb, q, Xp, p, num_mc, best_so_far, W,
                   ei_host + c0, want_grad ? grad_host + static_cast<size_t>(c0) * q * dim : nullptr);
  }
}

}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_ei_eval_large(const cmoe_gp* gp, const double* candidates, int num_candidates, int q,
                                  const double* points_being_sampled, int p, int num_mc, double best_so_far,
                                  uint64_t seed, const double* normals_table, double* ei, double* grad_ei, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_candidates >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    CMOE_REQUIRE(q >= 1 && p >= 0 && num_mc >= 1, CMOE_ERR_BOUNDS, "q >= 1, p >= 0, num_mc >= 1 required");
    CMOE_REQUIRE(static_cast<long long>(q) + p <= kMaxSampleQ, CMOE_ERR_BOUNDS, "q + p must be <= 8192");
    require_device(gp->device);
    const int U = q + p;
    DevBuf<double> dtable;
    if (normals_table) dtable.upload(normals_table, static_cast<size_t>(num_mc) * U, gp->stream);
    ei_large_eval_batch(*gp, candidates, num_candidates, q, points_being_sampled, p, num_mc, best_so_far, seed,
                        normals_table ? dtable.p : nullptr, ei, grad_ei);
  });
}

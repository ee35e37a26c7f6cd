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

// out = in^T for batched column-major rows x cols matrices (out: cols x rows), one batch entry per blockIdx.y
__global__ void __launch_bounds__(256) transpose_kernel(int rows, int cols, const double* __restrict__ in,
                                                        double* __restrict__ out) {
  const size_t off = static_cast<size_t>(blockIdx.y) * rows * cols;
  const size_t o = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (o >= static_cast<size_t>(rows) * cols) return;
  const size_t r = o % cols, cc = o / cols;  // out (r, cc) = in (cc, r)
  out[off + o] = in[off + r * rows + cc];
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


// Device pointers of one GP's run: the chunk workspace (chunk candidates)
struct EiLargeBufs {
  int chunk = 0;
  double *P, *V, *A, *mu, *stage, *part_v, *imp, *ei;
  double *T1 = nullptr, *T2 = nullptr, *R = nullptr, *grad = nullptr;
  int *fail, *part_i, *win, *dPs;
  int *cnt = nullptr, *start = nullptr, *order = nullptr;
};

// Lays out one GP's chunk workspace for `chunk` candidates at cv.
void ei_large_carve(int n, int U, int q, int dim, int num_mc, bool want_grad, int chunk, Carve& cv, EiLargeBufs& b) {
  const size_t ch = static_cast<size_t>(chunk), UU = static_cast<size_t>(U) * U, nrb = (U + NB - 1) / NB;
  b.chunk = chunk;
  b.P = cv.take<double>(ch * U * dim);
  b.V = cv.take<double>(ch * U * n);
  b.A = cv.take<double>(ch * UU);
  b.mu = cv.take<double>(ch * U);
  b.stage = cv.take<double>(ch * nrb * NB * NB);
  b.fail = cv.take<int>(ch);
  b.dPs = cv.take<int>(1);
  b.part_v = cv.take<double>(ch * nrb * num_mc);
  b.part_i = cv.take<int>(ch * nrb * num_mc);
  b.imp = cv.take<double>(ch * num_mc);
  b.win = cv.take<int>(ch * num_mc);
  b.ei = cv.take<double>(ch);
  if (want_grad) {
    b.T1 = cv.take<double>(ch * UU);
    b.T2 = cv.take<double>(ch * UU);
    b.R = cv.take<double>(ch * n * q);
    b.grad = cv.take<double>(ch * q * dim);
    b.cnt = cv.take<int>(ch * U);
    b.start = cv.take<int>(ch * U);
    b.order = cv.take<int>(ch * num_mc);
  }
}

size_t ei_large_chunk_bytes(int n, int U, int q, int dim, int num_mc, bool want_grad, int chunk) {
  Carve cv;
  EiLargeBufs b;
  ei_large_carve(n, U, q, dim, num_mc, want_grad, chunk, cv, b);
  return cv.off;
}

void ei_large_run(const cmoe_gp& gp, const EiLargeBufs& b, const double* cand, const double* Xp, int nc, int q, int p,
                  int num_mc, double best_so_far, const double* W, cudaStream_t s, double* ei_out, double* grad_out,
                  int* fail_out) {
  const int U = q + p, dim = gp.spec.dim, n = gp.n;
  const bool want_grad = grad_out != nullptr;
  const int nrb = (U + NB - 1) / NB, nsb = (num_mc + NB - 1) / NB;
  const size_t UU = static_cast<size_t>(U) * U;
  const unsigned gUU = static_cast<unsigned>((UU + 255) / 256);
  for (int c0 = 0; c0 < nc; c0 += b.chunk) {
    const int nb = std::min(b.chunk, nc - c0);
    const double* P = b.P;
    build_union_sets(cand + static_cast<size_t>(c0) * q * dim, Xp, nb, q, p, dim, b.P, s);
    // mu, Var + 1e-6 I (gpp_math.cpp:2000-2002) and its factor C, upper triangle zero
    posterior_cov_large(gp, P, b.dPs, b.V, b.mu, b.A, nb, U, 0, 1.0e-6, s);
    CMOE_CUDA(cudaMemsetAsync(b.fail, 0, nb * sizeof(int), s));
    potrf_batched(b.A, U, nb, b.fail, b.stage, s);
    CMOE_CUDA(cudaMemcpyAsync(fail_out + c0, b.fail, nb * sizeof(int), cudaMemcpyDeviceToDevice, s));
    zero_upper(nb, U, b.A, s);
    // forward
    CMOE_CUDA(cudaFuncSetAttribute(ei_mc_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(kTileSmem)));
    ei_mc_tile_kernel<<<dim3(nsb, nrb, nb), kTileThreads, kTileSmem, s>>>(U, num_mc, best_so_far, W, b.mu, b.A,
                                                                          b.part_v, b.part_i);
    ei_winner_kernel<<<dim3((num_mc + 255) / 256, nb), 256, 0, s>>>(num_mc, nrb, b.part_v, b.part_i, b.imp, b.win);
    ei_value_kernel<<<nb, 256, 0, s>>>(num_mc, b.imp, b.ei);
    count_launch(3);
    CMOE_CUDA(cudaGetLastError());
    CMOE_CUDA(cudaMemcpyAsync(ei_out + c0, b.ei, nb * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if (want_grad) {
      // B = K^-1 K(X, P) = L^-T V in place of V (cov_tile_kernel has consumed V)
      trsm_lower_blocked(gp.dK.p, n, b.V, n, nb * U, true, s);
      const size_t smem_bucket = static_cast<size_t>(U) * sizeof(int);
      CMOE_CUDA(cudaFuncSetAttribute(ei_bucket_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(smem_bucket)));
      ei_bucket_kernel<<<nb, kBucketThreads, smem_bucket, s>>>(U, num_mc, b.win, b.cnt, b.start, b.order);
      ei_cbar_kernel<<<dim3(gUU, nb), 256, 0, s>>>(U, num_mc, W, b.cnt, b.start, b.order, b.T1);
      count_launch(2);
      cholesky_adjoint(b.A, U, nb, b.T1, b.T2, s);
      // R = B T[:, :q]
      gemm_nn(n, q, U, b.V, n, static_cast<size_t>(n) * U, b.T1, U, UU, b.R, n, static_cast<size_t>(n) * q, nb, s);
      ei_grad_kernel<<<dim3(q, nb), kGradThreads, 0, s>>>(gp.spec, gp.N, gp.dX.p, gp.dKinvY.p, P, U, q, num_mc, b.T1,
                                                          b.R, b.cnt, b.grad);
      count_launch();
      CMOE_CUDA(cudaGetLastError());
      CMOE_CUDA(cudaMemcpyAsync(grad_out + static_cast<size_t>(c0) * q * dim, b.grad,
                                static_cast<size_t>(nb) * q * dim * sizeof(double), cudaMemcpyDeviceToDevice, s));
    }
  }
}

void check_ei_large_sizes(int q, int p, int num_mc) {
  CMOE_REQUIRE(q >= 1 && p >= 0 && num_mc >= 1, CMOE_ERR_BOUNDS, "q >= 1, p >= 0, num_mc >= 1 required");
  CMOE_REQUIRE(static_cast<long long>(q) + p <= kMaxSampleQ, CMOE_ERR_BOUNDS, "q + p must be <= 8192");
  CMOE_REQUIRE(static_cast<size_t>(num_mc) * (q + p) <= kSampleWorkspaceBytes / sizeof(double), CMOE_ERR_BOUNDS,
               "num_mc * (q + p) normals must fit in 2 GiB");
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
  const int t = (U + NB - 1) / NB;
  CMOE_CUDA(cudaFuncSetAttribute(ei_ctc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(kTileSmem)));
  ei_ctc_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kTileThreads, kTileSmem, s>>>(U, C, T1, T2);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
  mirror_lower(nc, U, T2, s);  // S = Phi(M) + Phi(M)^T
  for (int c = 0; c < nc; ++c)  // X = C^-T S
    trsm_lower_blocked(C + c * UU, U, T2 + c * UU, U, U, true, s);
  transpose_batched(U, U, T2, T1, nc, s);
  for (int c = 0; c < nc; ++c)  // T = C^-T X^T = C^-T S C^-1 = 2 Sigmabar
    trsm_lower_blocked(C + c * UU, U, T1 + c * UU, U, U, true, s);
}

void transpose_batched(int rows, int cols, const double* in, double* out, int batch, cudaStream_t s) {
  transpose_kernel<<<dim3(static_cast<unsigned>((static_cast<size_t>(rows) * cols + 255) / 256), batch), 256, 0, s>>>(
      rows, cols, in, out);
  count_launch();
}

void ei_large_eval(const cmoe_gp* const* gps, int num_gp, const double* candidates, int nc, int q, const double* Xp,
                   int p, int num_mc, const double* best_so_far, uint64_t seed, const double* dtable, double* values,
                   double* grads) {
  check_ei_large_sizes(q, p, num_mc);
  require_device(gps[0]->device);
  const int U = q + p, dim = gps[0]->spec.dim;
  const bool want_grad = grads != nullptr;
  // the normals are counted once, whether drawn here or passed in; the members in flight share the rest of the 2 GiB.
  // A candidate that alone needs more is not refused: it runs alone, one member at a time.
  const size_t w_count = static_cast<size_t>(num_mc) * U;
  size_t per = 0;
  for (int m = 0; m < num_gp; ++m)
    per = std::max(per, ei_large_chunk_bytes(gps[m]->n, U, q, dim, num_mc, want_grad, 1));
  const MemberSchedule ms = schedule_members(num_gp, nc, kSampleWorkspaceBytes - w_count * sizeof(double), per);
  size_t slot_bytes = 0;
  for (int m = 0; m < num_gp; ++m)
    slot_bytes = std::max(slot_bytes, ei_large_chunk_bytes(gps[m]->n, U, q, dim, num_mc, want_grad, ms.chunk));
  slot_bytes = slot_stride(slot_bytes);
  // one region on the first member's handle: the normals (unless passed in), the candidates and pending points, every
  // member's results, the slots
  const size_t ps = static_cast<size_t>(q) * dim;
  double *Wd = nullptr, *dcand = nullptr, *dXp = nullptr, *dval = nullptr, *dgrad = nullptr;
  int* dfail = nullptr;
  char* slots = nullptr;
  LargeUnionWork& w = carve_large_union_work(*gps[0], [&](Carve& cv) {
    Wd = dtable ? nullptr : cv.take<double>(w_count);
    dcand = cv.take<double>(static_cast<size_t>(nc) * ps);
    dXp = cv.take<double>(static_cast<size_t>(std::max(1, p)) * dim);
    dval = cv.take<double>(static_cast<size_t>(num_gp) * nc);
    dgrad = want_grad ? cv.take<double>(static_cast<size_t>(num_gp) * nc * ps) : nullptr;
    dfail = cv.take<int>(static_cast<size_t>(num_gp) * nc);
    slots = cv.take<char>(slot_bytes * ms.width);
  });
  cudaStream_t s0 = gps[0]->stream;
  const double* W = dtable;
  if (W == nullptr) {
    philox_normals_device(seed, 0, num_mc, U, Wd, s0);
    W = Wd;
  }
  CMOE_CUDA(cudaMemcpyAsync(dcand, candidates, static_cast<size_t>(nc) * ps * sizeof(double), cudaMemcpyHostToDevice,
                            s0));
  if (p) CMOE_CUDA(cudaMemcpyAsync(dXp, Xp, static_cast<size_t>(p) * dim * sizeof(double), cudaMemcpyHostToDevice, s0));
  CMOE_CUDA(cudaStreamSynchronize(s0));
  run_members(gps, num_gp, ms.width, w, [&](int m, int slot) {
    EiLargeBufs b;
    Carve sc{slots + slot * slot_bytes};
    ei_large_carve(gps[m]->n, U, q, dim, num_mc, want_grad, ms.chunk, sc, b);
    ei_large_run(*gps[m], b, dcand, dXp, nc, q, p, num_mc, best_so_far[m], W, gps[m]->stream, dval + m * nc,
                 want_grad ? dgrad + m * nc * ps : nullptr, dfail + m * nc);
  });
  drain_members(s0, num_gp, nc, ps, dval, dgrad, dfail, values, grads);
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
    // the table is uploaded once, beside the evaluation's workspace
    DevBuf<double> dtable;
    if (normals_table) dtable.upload(normals_table, static_cast<size_t>(num_mc) * (q + p), gp->stream);
    ei_large_eval(&gp, 1, candidates, num_candidates, q, points_being_sampled, p, num_mc, &best_so_far, seed,
                  normals_table ? dtable.p : nullptr, ei, grad_ei);
  });
}

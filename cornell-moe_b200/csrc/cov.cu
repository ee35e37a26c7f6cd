// Covariance-matrix builders (HBM-write-bound kernels).
//
// Replaces (reference, moe/optimal_learning/cpp/):
//   BuildCovarianceMatrixWithNoiseVariance   gpp_math.cpp:426-455   (lower triangle + noise by observation type)
//   BuildMixCovarianceMatrix                 gpp_math.cpp:309-335
//   SquareExponential / MaternNu2p5 ::Covariance   gpp_covariance.cpp:121-164, 339-387
//
// Tiling: one CTA per 128x64 block of point pairs in the lower-triangular tile grid; the two point slabs are staged
// through shared memory once and every thread produces a 4x4 register block (4 consecutive rows of 4 columns), so a
// lane's stores are 32 contiguous bytes and a warp store covers 8 lanes x 32 B = 256 contiguous bytes per column.  Only lower-triangular tiles are visited: the algorithmic traffic
// is 4*n*(n+1) bytes written + 8*N*dim read.
#include <algorithm>

#include "device_math.cuh"
#include "internal.cuh"
#include "linalg_dev.cuh"
#include "ptx_util.cuh"

namespace cmoe {

namespace {

constexpr int TR = 128;  // point rows per CTA tile
constexpr int TCW = 64;  // point cols per CTA tile
constexpr int kCovUnroll = 2;
constexpr int RB = 4;                  // rows per thread, 4 columns per thread
constexpr int WR = TR / (8 * RB);      // warps along the rows (a warp covers 8*RB rows x 16 cols)
constexpr int WC = 8 / WR;             // warps along the columns
constexpr int TC = WC * 16;            // columns per pass over the staged slabs

// 2^(i/64), the table of the reduced-range exp exp_tab_cov (device_math.cuh)
__device__ const double kCovExp2Table[64] = {
#include "exp2_table64.inc"
};

// g == 0 fast path: K[i + j*n] for i >= j (tile granularity), noise[0] on the diagonal.
// Works on length-scaled coordinates Xs = X / l with the expanded distance
//     -r^2/2 = x_i . x_j - |x_i|^2/2 - |x_j|^2/2
// (one FMA per dimension and entry; the absolute error of the expanded form is ~1e-16 (|x_i|^2 + |x_j|^2), a relative
// perturbation of k of that size — far below the noise term).  The half-norms are accumulated in the same FMA order as
// the dot product and scaled by the exact factor -1/2, so for coincident points the three terms cancel EXACTLY and
// k = alpha exp(0) = alpha bit-for-bit, as in the reference: duplicate points with zero noise must make the Cholesky
// fail at the same leading minor (tests/test_gpu_gp.py::test_gp_singular_reports_leading_minor).
template <int KERNEL>
__global__ void __launch_bounds__(256, 3)
    cov_build_g0_kernel(const __grid_constant__ KernelSpec spec, const double* __restrict__ Xs, int N,
                        const double* __restrict__ noise, double* __restrict__ K) {
  extern __shared__ double sm[];
  const int dim = spec.dim;
  double* Xr = sm;                 // [dim][TR]   coordinate-major: a lane's RB rows are contiguous
  double* Xc = sm + TR * dim;      // [dim][TCW]  (a warp shares its columns: broadcast reads)
  double* Hr = Xc + TCW * dim;     // [TR]   -|x_i|^2/2
  double* Hc = Hr + TR;            // [TCW]  -|x_j|^2/2
  double* tab = Hc + TCW;          // [64]
  if (threadIdx.x < 64) tab[threadIdx.x] = kCovExp2Table[threadIdx.x];
  // linear block index -> (tile row tr, tile col tc) of the lower-triangular tile grid: tc*TCW <= tr*TR + TR - 1
  constexpr int kColsPerRow = TR / TCW;  // col tiles that fit under one row tile's diagonal extent
  int tr = static_cast<int>((sqrt(8.0 * (blockIdx.x / kColsPerRow) + 1.0) - 1.0) * 0.5);
  while (tr * (tr + 1) / 2 * kColsPerRow > static_cast<int>(blockIdx.x)) --tr;
  while ((tr + 1) * (tr + 2) / 2 * kColsPerRow <= static_cast<int>(blockIdx.x)) ++tr;
  const int tc = blockIdx.x - tr * (tr + 1) / 2 * kColsPerRow;
  const int row0 = tr * TR, colbase = tc * TCW;
  if (colbase >= N) return;
  // coalesced, asynchronous (LDGSTS) slab loads, transposed on the fly into the coordinate-major shared layout
  for (int e = threadIdx.x; e < TR * dim; e += blockDim.x) {
    const int r = e / dim, k = e - r * dim;
    const bool ok = row0 + r < N;
    cp_async8(Xr + k * TR + r, ok ? Xs + static_cast<size_t>(row0) * dim + e : Xs, ok);
  }
  for (int e = threadIdx.x; e < TCW * dim; e += blockDim.x) {
    const int c = e / dim, k = e - c * dim;
    const bool ok = colbase + c < N;
    cp_async8(Xc + k * TCW + c, ok ? Xs + static_cast<size_t>(colbase) * dim + e : Xs, ok);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  if (threadIdx.x < TR + TCW) {
    const bool is_row = threadIdx.x < TR;
    const double* src = is_row ? Xr + threadIdx.x : Xc + (threadIdx.x - TR);
    const int stride = is_row ? TR : TCW;
    double h = 0.0;
    for (int k = 0; k < dim; ++k) h = fma(src[k * stride], src[k * stride], h);
    h *= -0.5;
    (is_row ? Hr : Hc)[is_row ? threadIdx.x : threadIdx.x - TR] = h;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int rloc = (warp % WR) * (8 * RB) + (lane & 7) * RB;  // first of this lane's RB rows inside the tile
  const double nz = noise[0];
  double hr[RB];
#pragma unroll
  for (int rr = 0; rr < RB; ++rr) hr[rr] = Hr[rloc + rr];
  for (int sub = 0; sub < TCW / TC; ++sub) {
    const int cloc = sub * TC + (warp / WR) * 16 + (lane >> 3) * 4;  // first of this lane's 4 cols inside the tile
    const int col0 = colbase + sub * TC;
    if (col0 > row0 + TR - 1 || col0 >= N) break;  // pass entirely above the diagonal
    // 2-D register blocking inside a warp: lane = (lr, lc) owns RB rows x 4 cols of an (8 RB) x 16 warp tile, so an
    // LDS.128 of the row slab touches 8 distinct 16-byte chunks (1 wavefront) and the column slab is a 4-way broadcast
    double t[RB][4];
#pragma unroll
    for (int rr = 0; rr < RB; ++rr)
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) t[rr][cc] = 0.0;
#pragma unroll kCovUnroll
    for (int k = 0; k < dim; ++k) {
      double xr[RB], xc[4];
#pragma unroll
      for (int rr = 0; rr < RB; rr += 2) {
        const double2 v = *reinterpret_cast<const double2*>(Xr + k * TR + rloc + rr);
        xr[rr] = v.x;
        xr[rr + 1] = v.y;
      }
#pragma unroll
      for (int cc = 0; cc < 4; cc += 2) {
        const double2 v = *reinterpret_cast<const double2*>(Xc + k * TCW + cloc + cc);
        xc[cc] = v.x;
        xc[cc + 1] = v.y;
      }
#pragma unroll
      for (int rr = 0; rr < RB; ++rr)
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) t[rr][cc] = fma(xr[rr], xc[cc], t[rr][cc]);
    }
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      const int gc = colbase + cloc + cc;
      if (gc >= N) continue;
      const double hcc = Hc[cloc + cc];
      double v[RB];
#pragma unroll
      for (int rr = 0; rr < RB; ++rr) {
        const double e = t[rr][cc] + (hr[rr] + hcc);  // = -r^2/2, exactly 0 for coincident points
        if (KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL) {
          v[rr] = spec.alpha * exp_tab_cov(e, tab);
        } else {
          const double r2 = fmax(0.0, -2.0 * e);
          const double arg = kSqrt5 * sqrt(r2);
          v[rr] = spec.alpha * exp_fast(-arg) * (1.0 + arg + 5.0 / 3.0 * r2);
        }
        if (row0 + rloc + rr == gc) v[rr] = spec.alpha + nz;  // exact diagonal: k(x, x) = alpha
      }
      const int gr = row0 + rloc;
      double* dst = K + static_cast<size_t>(gc) * N + gr;
      if (gr + RB - 1 < N && (N % 2 == 0)) {
        // 16-byte aligned when N is even (gr is a multiple of 4)
#pragma unroll
        for (int rr = 0; rr < RB; rr += 2) reinterpret_cast<double2*>(dst)[rr / 2] = make_double2(v[rr], v[rr + 1]);
      } else {
#pragma unroll
        for (int rr = 0; rr < RB; ++rr)
          if (gr + rr < N) dst[rr] = v[rr];
      }
    }
  }  // passes
}

// --------------------------------------------------------------------------------------------------------------
// g == 0, even N: persistent TMA version.  Per 128 x 64 tile of the lower-triangular tile grid:
//   * the two point slabs (rows of the length-scaled Xs, contiguous in global memory) arrive by TMA bulk copies
//     (cp.async.bulk -> UBLKCP) on an mbarrier — no transposing per-element staging, no bank-conflicted LDGSTS;
//   * the scaled dot products x_i . x_j run on the FP64 tensor pipe (DMMA m8n8k4, K = dim padded to a multiple of 4):
//     it has the FP64 units' throughput but 1/8 of the issue slots and no per-FMA operand traffic;
//   * -|x|^2/2 comes from the SAME instruction sequence applied to the 8 x 8 diagonal blocks of each slab, so
//     t_ij + (h_i + h_j) cancels exactly for coincident points and k = alpha bit-for-bit (see cov_build_g0_kernel);
//   * exp in the accumulator-fragment layout, results staged as a dense [64][128] tile in shared memory and written by
//     ONE TMA tensor store per tile (cp.async.bulk.tensor.2d.global.shared -> UTMASTG); the store drains while the other
//     resident CTA of the SM computes (2 CTAs / SM), and rows / columns beyond N are clipped by the tensor map.
// Contract: Xs readable for ceil(N/128)*128 rows (the slabs are copied whole; rows >= N only feed clipped outputs).
// --------------------------------------------------------------------------------------------------------------
constexpr int kTmaThreads = 256;

template <int KERNEL>
__global__ void __launch_bounds__(kTmaThreads, 2)
    cov_build_tma_kernel(const __grid_constant__ CUtensorMap mapK, const __grid_constant__ KernelSpec spec,
                         const double* __restrict__ Xs, int N, const double* __restrict__ noise, int ntiles) {
  extern __shared__ __align__(128) unsigned char cov_smem_raw[];
  double* stage = reinterpret_cast<double*>(smem_align128(cov_smem_raw));
  const int dim = spec.dim;
  double* slabR = stage + TCW * TR;      // [TR][dim]  rows of Xs as they lie in global memory
  double* slabC = slabR + TR * dim;      // [TCW][dim]
  double* Hr = slabC + TCW * dim;        // [TR]   -|x_i|^2/2
  double* Hc = Hr + TR;                  // [TCW]
  double* tab = Hc + TCW;                // [64]
  __shared__ __align__(8) uint64_t bar;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int lr = lane >> 2, lc = lane & 3;
  if (tid < 64) tab[tid] = kCovExp2Table[tid];
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_proxy_async();
  }
  __syncthreads();
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 32;
  const int ksteps = (dim + 3) >> 2;
  const double nz = noise[0];
  uint32_t phase = 0;
  constexpr int kColsPerRow = TR / TCW;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int tr = static_cast<int>((sqrt(8.0 * (tile / kColsPerRow) + 1.0) - 1.0) * 0.5);
    while (tr * (tr + 1) / 2 * kColsPerRow > tile) --tr;
    while ((tr + 1) * (tr + 2) / 2 * kColsPerRow <= tile) ++tr;
    const int tc = tile - tr * (tr + 1) / 2 * kColsPerRow;
    const int row0 = tr * TR, col0 = tc * TCW;
    if (col0 >= N) continue;
    if (tid == 0) {
      tma_store_wait_read<0>();  // the previous tile's store has finished reading the staging buffer
      mbar_expect_tx(&bar, static_cast<uint32_t>((TR + TCW) * dim * sizeof(double)));
      tma_bulk_g2s(slabR, Xs + static_cast<size_t>(row0) * dim, static_cast<uint32_t>(TR * dim * sizeof(double)), &bar);
      tma_bulk_g2s(slabC, Xs + static_cast<size_t>(col0) * dim, static_cast<uint32_t>(TCW * dim * sizeof(double)), &bar);
    }
    __syncthreads();  // staging buffer free, previous tile's readers of slabs / H done
    while (!mbar_try_wait(&bar, phase)) {
    }
    phase ^= 1;
    // half norms from 8 x 8 diagonal blocks, same DMMA chain as the tile product
    for (int blk = warp; blk < (TR + TCW) / 8; blk += kTmaThreads / 32) {
      const double* src = (blk < TR / 8) ? slabR + blk * 8 * dim : slabC + (blk - TR / 8) * 8 * dim;
      double c0 = 0.0, c1 = 0.0;
      for (int ks = 0; ks < ksteps; ++ks) {
        const int kk = ks * 4 + lc;
        const double a = (kk < dim) ? src[lr * dim + kk] : 0.0;
        dmma_m8n8k4(c0, c1, a, a);
      }
      if ((lr >> 1) == lc) {
        const double d = (lr & 1) ? c1 : c0;
        ((blk < TR / 8) ? Hr + blk * 8 : Hc + (blk - TR / 8) * 8)[lr] = -0.5 * d;
      }
    }
    __syncthreads();
    // a warp sub-tile entirely above the diagonal is skipped (its staging area keeps stale values; the strictly
    // upper triangle of K is unspecified, as in the reference)
    if (col0 + wn <= row0 + wm + 31) {
      double acc[4][4][2];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
      for (int ks = 0; ks < ksteps; ++ks) {
        const int kk = ks * 4 + lc;
        const bool ok = kk < dim;
        double a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = ok ? slabR[(wm + i * 8 + lr) * dim + kk] : 0.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = ok ? slabC[(wn + j * 8 + lr) * dim + kk] : 0.0;
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
      }
      double hrv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) hrv[i] = Hr[wm + i * 8 + lr];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int col = wn + j * 8 + lc * 2 + h;
          const double hcv = Hc[col];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = wm + i * 8 + lr;
            const double e = acc[i][j][h] + (hrv[i] + hcv);  // = -r^2/2, exactly 0 for coincident points
            double v;
            if (KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL) {
              v = spec.alpha * exp_tab_cov(e, tab);
            } else {
              const double r2 = fmax(0.0, -2.0 * e);
              const double arg = kSqrt5 * sqrt(r2);
              v = spec.alpha * exp_fast(-arg) * (1.0 + arg + 5.0 / 3.0 * r2);
            }
            if (row0 + row == col0 + col) v = spec.alpha + nz;  // exact diagonal: k(x, x) = alpha
            stage[col * TR + row] = v;
          }
        }
      }
    }
    fence_proxy_async();  // generic-proxy writes of the staging tile -> visible to the TMA store
    __syncthreads();
    if (tid == 0) {
      tma_store_2d(&mapK, stage, row0, col0);
      tma_store_commit();
    }
  }
  if (tid == 0) tma_store_wait<0>();
}

// generic path (derivative observations): one thread per point pair, writes the (1+g)x(1+g) block
__global__ void __launch_bounds__(256) cov_build_generic_kernel(const __grid_constant__ KernelSpec spec,
                                                                const double* __restrict__ X, int N,
                                                                const double* __restrict__ noise,
                                                                double* __restrict__ K) {
  const int dim = spec.dim, b = 1 + spec.g, n = N * b;
  const int i = blockIdx.x * 32 + (threadIdx.x & 31);  // row point (fast)
  const int j = blockIdx.y * 8 + (threadIdx.x >> 5);   // col point
  if (i >= N || j >= N || i < j) return;
  const double* p1 = X + static_cast<size_t>(i) * dim;
  const double* p2 = X + static_cast<size_t>(j) * dim;
  const KParts kp = kernel_parts(spec, weighted_sqdist(spec, p1, p2));
  for (int cn = 0; cn < b; ++cn) {
    const int a2 = cn ? spec.derivs[cn - 1] : -1;
    for (int m = 0; m < b; ++m) {
      const int a1 = m ? spec.derivs[m - 1] : -1;
      const int row = i * b + m, col = j * b + cn;
      if (row >= col) {
        double v = cov_entry(spec, kp, p1, p2, a1, a2);
        if (row == col) v += noise[m];
        K[static_cast<size_t>(col) * n + row] = v;
      }
    }
  }
}

// K(X, P): thread per (sampled point i, P point j), writes the (1+g)x(1+gs) block; rows fastest.  The P points run
// along grid.x (8 per CTA), so their number is not bounded by grid.y's 65535; the training rows take grid.y.
__global__ void __launch_bounds__(256) mix_cov_kernel(const __grid_constant__ KernelSpec spec,
                                                      const double* __restrict__ X, int N,
                                                      const double* __restrict__ P, int num,
                                                      const int* __restrict__ dPs, int gs,
                                                      double* __restrict__ out) {
  const int dim = spec.dim, b = 1 + spec.g, bs = 1 + gs, n = N * b;
  const int i = blockIdx.y * 32 + (threadIdx.x & 31);
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= N || j >= num) return;
  const double* p1 = X + static_cast<size_t>(i) * dim;
  const double* p2 = P + static_cast<size_t>(j) * dim;
  const KParts kp = kernel_parts(spec, weighted_sqdist(spec, p1, p2));
  for (int cn = 0; cn < bs; ++cn) {
    const int a2 = cn ? dPs[cn - 1] : -1;
    for (int m = 0; m < b; ++m) {
      const int a1 = m ? spec.derivs[m - 1] : -1;
      out[static_cast<size_t>(j * bs + cn) * n + i * b + m] = cov_entry(spec, kp, p1, p2, a1, a2);
    }
  }
}

__global__ void philox_table_kernel(uint64_t seed, uint64_t first_draw, int num_draws, int per_draw,
                                    double* __restrict__ out) {
  const int pairs = (per_draw + 1) / 2;
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<size_t>(num_draws) * pairs) return;
  const int i = static_cast<int>(idx / pairs), k = static_cast<int>(idx % pairs);
  double a, b;
  philox_normal_pair(seed, first_draw + i, k, a, b);
  out[static_cast<size_t>(i) * per_draw + 2 * k] = a;
  if (2 * k + 1 < per_draw) out[static_cast<size_t>(i) * per_draw + 2 * k + 1] = b;
}

}  // namespace

void build_covariance(const KernelSpec& spec, const double* X, const double* Xs, int N, const double* noise,
                      double* K, cudaStream_t s) {
  if (cov_tma_enabled() && spec.g == 0 && N >= 256 && (N & 1) == 0 && (reinterpret_cast<uintptr_t>(K) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(Xs) & 15) == 0) {
    CUtensorMap mapK;
    if (make_tensor_map_2d(&mapK, K, N, N, N, TR, TCW)) {
      const int trows = (N + TR - 1) / TR;
      const int ntiles = trows * (trows + 1) / 2 * (TR / TCW);
      int dev = 0, sms = 132;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      const size_t smem = (static_cast<size_t>(TCW) * TR + static_cast<size_t>(TR + TCW) * (spec.dim + 1) + 64) *
                              sizeof(double) + 128;
      const int grid = std::min(ntiles, 2 * sms);
      if (spec.kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL) {
        CMOE_CUDA(cudaFuncSetAttribute(cov_build_tma_kernel<CMOE_KERNEL_SQUARE_EXPONENTIAL>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        cov_build_tma_kernel<CMOE_KERNEL_SQUARE_EXPONENTIAL><<<grid, kTmaThreads, smem, s>>>(mapK, spec, Xs, N, noise,
                                                                                            ntiles);
      } else {
        CMOE_CUDA(cudaFuncSetAttribute(cov_build_tma_kernel<CMOE_KERNEL_MATERN_NU_2P5>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        cov_build_tma_kernel<CMOE_KERNEL_MATERN_NU_2P5><<<grid, kTmaThreads, smem, s>>>(mapK, spec, Xs, N, noise, ntiles);
      }
      count_launch();
      CMOE_CUDA(cudaGetLastError());
      return;
    }
  }
  if (spec.g == 0) {
    const int trows = (N + TR - 1) / TR;
    dim3 grid(trows * (trows + 1) / 2 * (TR / TCW));
    // the staged slabs take (TR + TCW)(dim + 1) + 64 doubles: past the default 48 KiB for dim >= 31
    const size_t smem = (static_cast<size_t>(TR + TCW) * (spec.dim + 1) + 64) * sizeof(double);
    constexpr int kMaxSmem = ((TR + TCW) * (CMOE_MAX_DIM + 1) + 64) * sizeof(double);
    if (spec.kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL) {
      CMOE_CUDA(cudaFuncSetAttribute(cov_build_g0_kernel<CMOE_KERNEL_SQUARE_EXPONENTIAL>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
      cov_build_g0_kernel<CMOE_KERNEL_SQUARE_EXPONENTIAL><<<grid, 256, smem, s>>>(spec, Xs, N, noise, K);
    } else {
      CMOE_CUDA(cudaFuncSetAttribute(cov_build_g0_kernel<CMOE_KERNEL_MATERN_NU_2P5>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
      cov_build_g0_kernel<CMOE_KERNEL_MATERN_NU_2P5><<<grid, 256, smem, s>>>(spec, Xs, N, noise, K);
    }
  } else {
    dim3 grid((N + 31) / 32, (N + 7) / 8);
    cov_build_generic_kernel<<<grid, 256, 0, s>>>(spec, X, N, noise, K);
  }
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

void build_mix_covariance(const KernelSpec& spec, const double* X, int N, const double* P, int num, const int* dPs,
                          int gs, double* out, cudaStream_t s) {
  if (num == 0 || N == 0) return;
  dim3 grid((num + 7) / 8, (N + 31) / 32);
  mix_cov_kernel<<<grid, 256, 0, s>>>(spec, X, N, P, num, dPs, gs, out);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

void philox_normals_device(uint64_t seed, uint64_t first_draw, int num_draws, int per_draw, double* out,
                           cudaStream_t s) {
  const size_t total = static_cast<size_t>(num_draws) * ((per_draw + 1) / 2);
  if (!total) return;
  philox_table_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(seed, first_draw, num_draws, per_draw,
                                                                               out);
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

}  // namespace cmoe

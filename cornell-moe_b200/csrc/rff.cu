// Random-feature Thompson sampling of the global minimum (DESIGN.md K14), batched over samples.
//
// Replaces (reference, moe/optimal_learning/python/random_features.py):
//   sample_gp_with_random_features            :29-133  (features, design matrix, posterior of the weights)
//   global_optimization_of_GP_approximation   :144-168 (grid argmin + local optimisation)
//   sample_from_global_optima                 :171-175 (one sample at a time)
//
// Per chunk of samples (the contract is in cmoe_b200.h, next to cmoe_gp_sample_rff_optima):
//   W = Omega / l, b = 2 pi u                         rff_features_kernel
//   Phi (M < F) or the column-reversed Phi^T (M >= F) rff_design_kernel
//   I + Phi^T Phi  or  reversed I + Phi Phi^T         rff_gram_kernel: DMMA m16n8k4 (gram_tile_accumulate)
//   L L^T = Gram                                      potrf_batched
//   theta                                             rff_theta_kernel: one CTA per sample, fixed-order GEMVs and
//                                                     blocked substitutions (cta_forward_subst / cta_backward_subst)
//   f on the grid, per-CTA argmin partials           rff_grid_kernel, best_of_parts_kernel
//   projected Newton from the grid argmin            rff_opt_kernel: one warp per sample
// Every kernel treats the samples of a chunk independently and every reduction has a fixed order, so a sample's result
// is a pure function of its randomness, not of num_points or the chunking.  cmoe_gp_sample_rff_functions stops after
// theta; cmoe_rff_evaluate runs rff_eval_kernel, the grid kernel's per-point arithmetic (rff_accumulate) without the
// argmin.  The kernel-matched (Matern-5/2) draw rescales W's rows in rff_features_kernel (rff_chi2_at).
//
// The M >= F branch factors the order-reversed B = I_F + Phi Phi^T: with J the reversal, J B J = L L^T gives the upper
// factor U = J L J of B = U U^T.  The design kernel stores the columns of Phi^T in reversed feature order, so the Gram
// kernel's ordinary product is J B J.  In the reversed coordinates theta_rev = L^-T (L^-1 (J Phi y') + J z).
#include <algorithm>
#include <climits>
#include <cmath>

#include "device_math.cuh"
#include "internal.cuh"
#include "linalg_dev.cuh"

namespace cmoe {

namespace {

constexpr int kRffThreads = 256;      // design, theta, grid kernels
constexpr int kRffTileThreads = 128;  // rff_gram_kernel: 4 warps over a 64 x 64 tile (tile_mma64)
constexpr int kRffGridTile = 128;     // features staged in shared memory per round of rff_grid_kernel
constexpr int kRffGridCtas = 1024;    // grid-kernel CTAs per sample at most (the rest is a grid-stride loop)
constexpr int kRffOptWarps = 2;       // samples per CTA of rff_opt_kernel
constexpr int kRffMaxIter = 100;      // SLSQP's default iteration limit
constexpr int kRffMaxHalvings = 60;
constexpr double kRffKktTol = 1e-9;   // stop: ||x - P(x - grad)||_inf <= kRffKktTol (1 + |f|)
constexpr double kRffArmijo = 1e-4;
constexpr double kRffSlack = 1e-13;   // Armijo rounding slack, relative to 1 + |f|
constexpr double kRffEpsActive = 1e-3;  // epsilon-active set margin, relative to the box's width
constexpr double kTwoPi = 6.283185307179586476925286766559;

struct RffBox {
  double lo[CMOE_MAX_DIM];
  double hi[CMOE_MAX_DIM];
};

struct RffShape {
  int F, M, N, d, g, woodbury;  // woodbury = M < F
  double c;                     // sqrt(2 alpha / F)
  double len[CMOE_MAX_DIM];
  double sqrt_nu[CMOE_MAX_DIM + 1];  // sqrt(nu_t): the design divides by it, as the reference does
  int derivs[CMOE_MAX_DIM];
  int matern;  // kernel-matched Matern-5/2 draw: W = (Omega / l) sqrt(5 / g), g ~ chi^2_5 per feature
};

// sin and cos of the sample functions' arguments: rff_sincos (device_math.cuh)
__device__ __forceinline__ double rff_cos(double a) {
  double sn, cs;
  rff_sincos(a, sn, cs);
  return cs;
}

__device__ __forceinline__ double rff_sin(double a) {
  double sn, cs;
  rff_sincos(a, sn, cs);
  return sn;
}

// The features' share of one point's sample-function sums, in ascending feature order: acc += theta_f cos(W_f x + b_f)
// and, with G, g[k] += theta_f sin(W_f x + b_f) W_fk, for the nf features staged at Wt [nf][d], bt, tt.  The grid
// stage and the evaluator both run it, so the evaluator's values are the grid stage's bits at the same point.
template <bool G>
__device__ __forceinline__ void rff_accumulate(const double* Wt, const double* bt, const double* tt, int nf, int d,
                                               const double* x, double& acc, double* g) {
  for (int f = 0; f < nf; ++f) {
    const double* w = Wt + f * d;
    double a = 0.0;
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k)
      if (k < d) a = fma(w[k], x[k], a);
    if (G) {
      double sn, cs;
      rff_sincos(a + bt[f], sn, cs);
      acc = fma(tt[f], cs, acc);
      const double ws = tt[f] * sn;
#pragma unroll
      for (int k = 0; k < CMOE_MAX_DIM; ++k)
        if (k < d) g[k] = fma(ws, w[k], g[k]);
    } else {
      acc = fma(tt[f], rff_cos(a + bt[f]), acc);
    }
  }
}

// 53-bit uniform in (0, 1] from one 64-bit Philox output word pair, as philox_normal_pair forms it
__device__ __forceinline__ double rff_u53(uint32_t hi, uint32_t lo) {
  const uint64_t w = (static_cast<uint64_t>(hi) << 32) | lo;
  return __dmul_rn(__dadd_rn(static_cast<double>(w >> 11), 0.5), 0x1.0p-53);
}

// g_f ~ chi^2_5 of the kernel-matched (Matern-5/2) draw: the sum of squares of five Box-Muller normals from the Philox
// calls (draw, 2f) and (draw, 2f + 1) with counter word 3 = 3.  Call 2f gives the radial uniforms u0, u1 of two full
// pairs, whose squares sum to -2 ln u whatever their angle; call 2f + 1 gives (u2, v2) and the fifth normal
// sqrt(-2 ln u2) cos(2 pi v2).  g = -2 ln u0 - 2 ln u1 + (-2 ln u2) cos^2(2 pi v2), in that order.
__device__ __forceinline__ double rff_chi2_at(uint64_t seed, uint64_t draw, int f) {
  const uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  uint32_t c[4] = {static_cast<uint32_t>(draw), static_cast<uint32_t>(draw >> 32), 2u * static_cast<uint32_t>(f), 3u};
  philox4x32_10(c, k0, k1);
  const double u0 = rff_u53(c[0], c[1]), u1 = rff_u53(c[2], c[3]);
  uint32_t e[4] = {static_cast<uint32_t>(draw), static_cast<uint32_t>(draw >> 32), 2u * static_cast<uint32_t>(f) + 1u,
                   3u};
  philox4x32_10(e, k0, k1);
  const double u2 = rff_u53(e[0], e[1]), v2 = rff_u53(e[2], e[3]);
  const double cs = rff_cos(__dmul_rn(kTwoPi, v2));
  const double t = __dmul_rn(-2.0, log(u2));
  return __dadd_rn(__dadd_rn(__dmul_rn(-2.0, log(u0)), __dmul_rn(-2.0, log(u1))), __dmul_rn(__dmul_rn(t, cs), cs));
}

__device__ __forceinline__ double philox_normal_at(uint64_t seed, uint64_t draw, size_t k) {
  double a, b;
  philox_normal_pair(seed, draw, static_cast<uint32_t>(k >> 1), a, b);
  return (k & 1) ? b : a;
}

__device__ __forceinline__ double philox_uniform_at(uint64_t seed, uint64_t draw, int f) {
  uint32_t c[4] = {static_cast<uint32_t>(draw), static_cast<uint32_t>(draw >> 32), static_cast<uint32_t>(f >> 1), 2u};
  philox4x32_10(c, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  const uint64_t w = (f & 1) ? ((static_cast<uint64_t>(c[2]) << 32) | c[3]) : ((static_cast<uint64_t>(c[0]) << 32) | c[1]);
  return __dmul_rn(__dadd_rn(static_cast<double>(w >> 11), 0.5), 0x1.0p-53);
}

// W[s][f][k] = Omega / l_k and b[s][f]; grid (ceil(max(F, M) / 256), samples).  Omega and b come from row s of the
// table, or from Philox draw draw0 + s; in Philox mode the kernel also writes z[s][F] and, when M < F, eps[s][M] (the
// table mode uploads them).  The Box-Muller step is philox_normal_pair's, so the numbers are cmoe_philox_normals'.
// With sh.matern each row is scaled by sqrt(5 / g_f), g_f from rff_chi2_at or from t_chi2[s][f] in table mode; the other
// numbers are those of the reference mode.
__global__ void __launch_bounds__(kRffThreads) rff_features_kernel(const __grid_constant__ RffShape sh, uint64_t seed,
                                                                   uint64_t draw0, const double* __restrict__ t_omega,
                                                                   const double* __restrict__ t_b,
                                                                   const double* __restrict__ t_chi2,
                                                                   double* __restrict__ W, double* __restrict__ b,
                                                                   double* __restrict__ z, double* __restrict__ eps) {
  const int s = blockIdx.y, f = blockIdx.x * blockDim.x + threadIdx.x, F = sh.F, d = sh.d;
  const uint64_t draw = draw0 + s;
  const size_t zoff = static_cast<size_t>(F) * d;
  if (!t_omega && sh.woodbury && f < sh.M)
    eps[static_cast<size_t>(s) * sh.M + f] = philox_normal_at(seed, draw, zoff + F + f);
  if (f >= F) return;
  const size_t row = (static_cast<size_t>(s) * F + f) * d;
  double scale = 1.0;
  if (sh.matern) {
    const double g = t_omega ? t_chi2[static_cast<size_t>(s) * F + f] : rff_chi2_at(seed, draw, f);
    scale = __dsqrt_rn(__ddiv_rn(5.0, g));
  }
  double n0 = 0.0, n1 = 0.0;  // the Philox pair holding normal f d + k (one Philox call per pair)
  for (int k = 0; k < d; ++k) {
    const size_t i = static_cast<size_t>(f) * d + k;
    if (!t_omega && (k == 0 || (i & 1) == 0)) philox_normal_pair(seed, draw, static_cast<uint32_t>(i >> 1), n0, n1);
    const double om = t_omega ? t_omega[row + k] : ((i & 1) ? n1 : n0);
    const double w = __ddiv_rn(om, sh.len[k]);
    W[row + k] = sh.matern ? __dmul_rn(w, scale) : w;
  }
  if (t_omega) {
    b[static_cast<size_t>(s) * F + f] = t_b[static_cast<size_t>(s) * F + f];
  } else {
    b[static_cast<size_t>(s) * F + f] = __dmul_rn(kTwoPi, philox_uniform_at(seed, draw, f));
    z[static_cast<size_t>(s) * F + f] = philox_normal_at(seed, draw, zoff + f);
  }
}

// The design matrix of every sample, one element per thread: grid (fast blocks, samples, slow splits); the thread's
// fast index is fixed and it steps over the slow index.  M < F: Phi column-major (fast = feature f, slow = column).
// M >= F: Phi^T with reversed features (fast = column, slow = F - 1 - f).  Consecutive threads write consecutive
// addresses in both layouts.
__global__ void __launch_bounds__(kRffThreads) rff_design_kernel(const __grid_constant__ RffShape sh,
                                                                 const double* __restrict__ X,
                                                                 const double* __restrict__ W,
                                                                 const double* __restrict__ b,
                                                                 double* __restrict__ Phi) {
  const int s = blockIdx.y, F = sh.F, M = sh.M, N = sh.N, d = sh.d;
  const int nfast = sh.woodbury ? F : M, nslow = sh.woodbury ? M : F;
  const int fast = blockIdx.x * blockDim.x + threadIdx.x;
  if (fast >= nfast) return;
  const double* Ws = W + static_cast<size_t>(s) * F * d;
  const double* bs = b + static_cast<size_t>(s) * F;
  double* Ps = Phi + static_cast<size_t>(s) * F * M;
  for (int slow = blockIdx.z; slow < nslow; slow += gridDim.z) {
    const int f = sh.woodbury ? fast : F - 1 - slow, col = sh.woodbury ? slow : fast;
    const int t = col / N, i = col % N;
    const double* w = Ws + static_cast<size_t>(f) * d;
    const double* x = X + static_cast<size_t>(i) * d;
    double a = 0.0;
    for (int k = 0; k < d; ++k) a = fma(w[k], x[k], a);
    a += bs[f];
    const double v = (t == 0) ? sh.c * rff_cos(a) / sh.sqrt_nu[0] : -sh.c * w[sh.derivs[t - 1]] * rff_sin(a) / sh.sqrt_nu[t];
    Ps[static_cast<size_t>(slow) * nfast + fast] = v;
  }
}

// Gram_s = I + V_s^T V_s on the lower 64 x 64 tiles; V_s is K x Q column-major (Phi for M < F: K = F, Q = M; the
// reversed Phi^T for M >= F: K = M, Q = F).  grid (tiles, 1, samples).  Only the lower triangle is written.
__global__ void __launch_bounds__(kRffTileThreads) rff_gram_kernel(const double* __restrict__ V, int K, int Q,
                                                                   double* __restrict__ A) {
  extern __shared__ double smem[];
  double* As = smem;           // [NB][LDT]
  double* Bs = As + NB * LDT;  // [NB][LDT]
  const int s = blockIdx.z, tid = threadIdx.x;
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int row0 = ti * NB, col0 = tj * NB;
  const int rows = min(NB, Q - row0), cols = min(NB, Q - col0);
  const double* Vs = V + static_cast<size_t>(s) * K * Q;
  const int warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  gram_tile_accumulate(Vs + static_cast<size_t>(row0) * K, Vs + static_cast<size_t>(col0) * K, K, rows, cols, As, Bs,
                       acc, wm, wn, lr, lc);
  double* Ab = A + static_cast<size_t>(s) * Q * Q;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr, gr = row0 + r;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h, gc = col0 + c;
        if (r < rows && c < cols && gr >= gc) Ab[static_cast<size_t>(gc) * Q + gr] = acc[i][j][h] + (gr == gc ? 1.0 : 0.0);
      }
  }
}

// theta of one sample per CTA (the header's two branches), z[s][F] and eps[s][M] as rff_features_kernel or the table
// left them.  A sample whose factorisation failed is skipped (the host reports it).  Dot products
// over F are lane-strided in one warp and combined by the warp_sum butterfly; those over M run serially in ascending
// order; theta doubles as the F-vector r of the Woodbury branch.
__global__ void __launch_bounds__(kRffThreads) rff_theta_kernel(const __grid_constant__ RffShape sh,
                                                                const double* __restrict__ Phi,
                                                                const double* __restrict__ yp,
                                                                const double* __restrict__ L,
                                                                const int* __restrict__ fail,
                                                                const double* __restrict__ z,
                                                                const double* __restrict__ eps, double* theta) {
  extern __shared__ double rff_v[];  // [Q] right-hand side -> solution
  const int s = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
  if (fail[s] != 0) return;
  const int F = sh.F, M = sh.M, Q = sh.woodbury ? M : F;
  double* D = rff_v + Q;  // [NB][NB + 1]
  const double* Ps = Phi + static_cast<size_t>(s) * F * M;
  const double* Ls = L + static_cast<size_t>(s) * Q * Q;
  double* th = theta + static_cast<size_t>(s) * F;
  const double* zs = z + static_cast<size_t>(s) * F;
  if (sh.woodbury) {
    for (int f = tid; f < F; f += blockDim.x) {  // r = Phi y' + z
      double acc = 0.0;
      for (int i = 0; i < M; ++i) acc = fma(Ps[static_cast<size_t>(i) * F + f], yp[i], acc);
      th[f] = acc + zs[f];
    }
    __syncthreads();
    for (int i = warp; i < M; i += nw) {  // v = Phi^T r + eps
      const double* col = Ps + static_cast<size_t>(i) * F;
      double acc = 0.0;
      for (int f = lane; f < F; f += 32) acc = fma(col[f], th[f], acc);
      acc = warp_sum(acc);
      if (lane == 0) rff_v[i] = acc + eps[static_cast<size_t>(s) * M + i];
    }
  } else {
    for (int c = warp; c < F; c += nw) {  // v = J Phi y'
      const double* col = Ps + static_cast<size_t>(c) * M;
      double acc = 0.0;
      for (int i = lane; i < M; i += 32) acc = fma(col[i], yp[i], acc);
      acc = warp_sum(acc);
      if (lane == 0) rff_v[c] = acc;
    }
  }
  cta_forward_subst(Ls, Q, rff_v, D);
  if (!sh.woodbury)
    for (int c = tid; c < F; c += blockDim.x) rff_v[c] += zs[F - 1 - c];
  cta_backward_subst(Ls, Q, rff_v, D);
  if (sh.woodbury) {
    for (int f = tid; f < F; f += blockDim.x) {  // theta = r - Phi A^-1 v
      double acc = 0.0;
      for (int i = 0; i < M; ++i) acc = fma(Ps[static_cast<size_t>(i) * F + f], rff_v[i], acc);
      th[f] -= acc;
    }
  } else {
    for (int f = tid; f < F; f += blockDim.x) th[f] = rff_v[F - 1 - f];
  }
}

// f at the grid points of one sample (grid.y), a grid-stride loop over the points; features staged kRffGridTile at a
// time in shared memory.  Each thread keeps the first minimum of its points (ascending), each CTA the first minimum of
// its threads: (part_v, part_i)[s][blockIdx.x].
__global__ void __launch_bounds__(kRffThreads) rff_grid_kernel(const __grid_constant__ RffShape sh,
                                                               const double* __restrict__ grid, int G,
                                                               const double* __restrict__ W,
                                                               const double* __restrict__ b,
                                                               const double* __restrict__ theta,
                                                               double* __restrict__ part_v, int* __restrict__ part_i) {
  extern __shared__ double gs[];  // [kRffGridTile][d] W, [kRffGridTile] b, [kRffGridTile] theta
  __shared__ double bv[kRffThreads / 32];
  __shared__ int bi[kRffThreads / 32];
  const int s = blockIdx.y, tid = threadIdx.x, F = sh.F, d = sh.d;
  double* Wt = gs;
  double* bt = Wt + kRffGridTile * d;
  double* tt = bt + kRffGridTile;
  const double* Ws = W + static_cast<size_t>(s) * F * d;
  const double* bs = b + static_cast<size_t>(s) * F;
  const double* ts = theta + static_cast<size_t>(s) * F;
  double best = INFINITY;
  int bidx = INT_MAX;
  for (int base = blockIdx.x * blockDim.x; base < G; base += gridDim.x * blockDim.x) {  // uniform over the CTA
    const int j = base + tid;
    const bool valid = j < G;
    double x[CMOE_MAX_DIM];
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k) x[k] = (valid && k < d) ? grid[static_cast<size_t>(j) * d + k] : 0.0;
    double acc = 0.0;
    for (int f0 = 0; f0 < F; f0 += kRffGridTile) {
      const int nf = min(kRffGridTile, F - f0);
      __syncthreads();
      for (int e = tid; e < nf * d; e += blockDim.x) Wt[e] = Ws[static_cast<size_t>(f0) * d + e];
      for (int e = tid; e < nf; e += blockDim.x) {
        bt[e] = bs[f0 + e];
        tt[e] = ts[f0 + e];
      }
      __syncthreads();
      if (valid) rff_accumulate<false>(Wt, bt, tt, nf, d, x, acc, nullptr);
    }
    const double v = sh.c * acc;
    if (valid && v < best) {
      best = v;
      bidx = j;
    }
  }
  block_best<false>(best, bidx, bv, bi);
  if (tid == 0) {
    part_v[static_cast<size_t>(s) * gridDim.x + blockIdx.x] = best;
    part_i[static_cast<size_t>(s) * gridDim.x + blockIdx.x] = bidx;
  }
}

// f (and with G, the gradient, into gout: shared, d values) of one sample at x (shared, d values), lanes striding over the features and combined by
// the warp_sum butterfly, so every lane holds the same bits.  With wc, wc[f] = c theta_f cos(W_f x + b_f) is stored
// for the Hessian.
template <bool G>
__device__ __forceinline__ double rff_eval(const RffShape& sh, const double* Ws, const double* bs, const double* ts,
                                           const double* x, int lane, double* gout, double* wc) {
  const int F = sh.F, d = sh.d;
  double fv = 0.0;
  double g[CMOE_MAX_DIM];
  if (G) {
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k) g[k] = 0.0;
  }
  for (int f = lane; f < F; f += 32) {
    const double* w = Ws + static_cast<size_t>(f) * d;
    double a = 0.0;
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k)
      if (k < d) a = fma(w[k], x[k], a);
    a += bs[f];
    if (G) {
      double sn, cs;
      rff_sincos(a, sn, cs);
      fv = fma(ts[f], cs, fv);
      const double ws = ts[f] * sn;
#pragma unroll
      for (int k = 0; k < CMOE_MAX_DIM; ++k)
        if (k < d) g[k] = fma(ws, w[k], g[k]);
      wc[f] = sh.c * ts[f] * cs;
    } else {
      fv = fma(ts[f], rff_cos(a), fv);
    }
  }
  if (G) {
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k)
      if (k < d) {
        const double v = -sh.c * warp_sum(g[k]);
        if (lane == k) gout[k] = v;
      }
  }
  const double fsum = sh.c * warp_sum(fv);
  __syncwarp();
  return fsum;
}

// Projected Newton (the header's local step) for one sample per warp, from the clamped grid argmin.  Each warp keeps
// its iterate, trial point, step and Hessian in shared memory; every scalar decision is warp-uniform.
__global__ void __launch_bounds__(kRffOptWarps * 32) rff_opt_kernel(const __grid_constant__ RffShape sh, int ns,
                                                                    const __grid_constant__ RffBox box,
                                                                    const double* __restrict__ grid,
                                                                    const int* __restrict__ amin,
                                                                    const double* __restrict__ vmin,
                                                                    const double* __restrict__ W,
                                                                    const double* __restrict__ b,
                                                                    const double* __restrict__ theta,
                                                                    double* __restrict__ wc_all,
                                                                    double* __restrict__ pts,
                                                                    double* __restrict__ vals) {
  __shared__ double sx[kRffOptWarps][CMOE_MAX_DIM], st[kRffOptWarps][CMOE_MAX_DIM], sp[kRffOptWarps][CMOE_MAX_DIM];
  __shared__ double sH[kRffOptWarps][CMOE_MAX_DIM][CMOE_MAX_DIM + 1];
  __shared__ double sL[kRffOptWarps][CMOE_MAX_DIM][CMOE_MAX_DIM + 1];
  __shared__ double sg[kRffOptWarps][CMOE_MAX_DIM];
  __shared__ int sfree[kRffOptWarps][CMOE_MAX_DIM];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s = blockIdx.x * kRffOptWarps + wid;
  if (s >= ns) return;
  const int F = sh.F, d = sh.d;
  const double* Ws = W + static_cast<size_t>(s) * F * d;
  const double* bs = b + static_cast<size_t>(s) * F;
  const double* ts = theta + static_cast<size_t>(s) * F;
  double* wc = wc_all + static_cast<size_t>(s) * F;
  double* x = sx[wid];
  double* xt = st[wid];
  double* p = sp[wid];
  double* g = sg[wid];
  double (*H)[CMOE_MAX_DIM + 1] = sH[wid];
  double (*Lc)[CMOE_MAX_DIM + 1] = sL[wid];
  int* fr = sfree[wid];
  const double* x0 = grid + static_cast<size_t>(amin[s]) * d;
  if (lane < d) x[lane] = fmin(fmax(x0[lane], box.lo[lane]), box.hi[lane]);
  __syncwarp();
  double fx;
  for (int it = 0;; ++it) {  // one gradient evaluation site: at most kRffMaxIter steps
    fx = rff_eval<true>(sh, Ws, bs, ts, x, lane, g, wc);
    if (it == kRffMaxIter) break;
    // projected-gradient residual, then Bertsekas' epsilon-active set: variable k is held when it lies within
    // eps_k = min(1e-3 (hi_k - lo_k), residual) of a bound and its gradient points out of the box
    double res = 0.0;
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k)
      if (k < d) res = fmax(res, fabs(x[k] - fmin(fmax(x[k] - g[k], box.lo[k]), box.hi[k])));
    if (res <= kRffKktTol * (1.0 + fabs(fx))) break;
    int nf = 0;
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k) {
      if (k < d) {
        const double xk = x[k], ek = fmin(kRffEpsActive * (box.hi[k] - box.lo[k]), res);
        const bool held = (xk <= box.lo[k] + ek && g[k] > 0.0) || (xk >= box.hi[k] - ek && g[k] < 0.0);
        if (!held) {
          if (lane == 0) fr[nf] = k;
          ++nf;
        }
      }
    }
    __syncwarp();
    // Hessian rows of the free variables: H[j][k] = -sum_f wc_f W_fj W_fk, row j over k
    for (int a = 0; a < nf; ++a) {
      const int j = fr[a];
      double h[CMOE_MAX_DIM];
#pragma unroll
      for (int k = 0; k < CMOE_MAX_DIM; ++k) h[k] = 0.0;
      for (int f = lane; f < F; f += 32) {
        const double* w = Ws + static_cast<size_t>(f) * d;
        const double t = wc[f] * w[j];
#pragma unroll
        for (int k = 0; k < CMOE_MAX_DIM; ++k)
          if (k < d) h[k] = fma(t, w[k], h[k]);
      }
#pragma unroll
      for (int k = 0; k < CMOE_MAX_DIM; ++k)
        if (k < d) {
          const double v = -warp_sum(h[k]);
          if (lane == k) H[j][k] = v;
        }
    }
    __syncwarp();
    // shifted Cholesky of the free block (lower triangle from rows a >= b: H[fr[a]][fr[b]])
    double hmax = 0.0, hmin = INFINITY;
    for (int a = 0; a < nf; ++a) {
      hmax = fmax(hmax, fabs(H[fr[a]][fr[a]]));
      hmin = fmin(hmin, H[fr[a]][fr[a]]);
    }
    const double beta = 1e-3 * fmax(hmax, 1e-12);
    double tau = hmin > 0.0 ? 0.0 : beta - hmin;
    bool ok = false;
    for (int tries = 0; tries < 64 && !ok; ++tries) {
      ok = true;
      for (int c = 0; c < nf; ++c) {
        double dg = H[fr[c]][fr[c]] + tau;
        for (int k = 0; k < c; ++k) dg = fma(-Lc[c][k], Lc[c][k], dg);
        if (!(dg > 0.0)) {
          ok = false;
          break;
        }
        const double ri = rsqrt(dg);  // the diagonal slot holds 1 / L_cc: no division in the loop
        if (lane > c && lane < nf) {
          double v = H[fr[lane]][fr[c]];
          for (int k = 0; k < c; ++k) v = fma(-Lc[lane][k], Lc[c][k], v);
          Lc[lane][c] = v * ri;
        }
        if (lane == c) Lc[c][c] = ri;
        __syncwarp();
      }
      if (!ok) tau = fmax(2.0 * tau, beta);
      __syncwarp();
    }
    if (!ok) break;
    // p_free = -(H_ff + tau I)^-1 g_free (lane 0, then shared; xt holds the intermediate vector)
    if (lane == 0) {
      double* y = xt;
      for (int a = 0; a < nf; ++a) {
        double v = -g[fr[a]];
        for (int k = 0; k < a; ++k) v = fma(-Lc[a][k], y[k], v);
        y[a] = v * Lc[a][a];
      }
      for (int a = nf - 1; a >= 0; --a) {
        double v = y[a];
        for (int k = a + 1; k < nf; ++k) v = fma(-Lc[k][a], y[k], v);
        y[a] = v * Lc[a][a];
      }
      // held variables step along -g (onto their bound); a free variable at a bound drops an outward Newton
      // component, so every component of the projected step is a descent direction for small steps
      for (int k = 0; k < d; ++k) p[k] = -g[k];
      for (int a = 0; a < nf; ++a) {
        const int k = fr[a];
        const bool out = (x[k] <= box.lo[k] && y[a] < 0.0) || (x[k] >= box.hi[k] && y[a] > 0.0);
        p[k] = out ? 0.0 : y[a];
      }
    }
    __syncwarp();
    // Armijo backtracking along the projected arc
    double alpha = 1.0, ft = 0.0;
    bool acc = false;
    for (int h = 0; h < kRffMaxHalvings; ++h) {
      if (lane < d) xt[lane] = fmin(fmax(x[lane] + alpha * p[lane], box.lo[lane]), box.hi[lane]);
      __syncwarp();
      double dec = 0.0;
#pragma unroll
      for (int k = 0; k < CMOE_MAX_DIM; ++k)
        if (k < d) dec = fma(g[k], xt[k] - x[k], dec);
      ft = rff_eval<false>(sh, Ws, bs, ts, xt, lane, nullptr, nullptr);
      if (ft <= fx + kRffArmijo * dec + kRffSlack * (1.0 + fabs(fx))) {
        acc = true;
        break;
      }
      alpha *= 0.5;
      __syncwarp();
    }
    if (!acc) break;
    if (lane < d) x[lane] = xt[lane];
    __syncwarp();
  }
  const double gmin = vmin[s];
  const bool keep = fx < gmin;
  if (lane < d) pts[static_cast<size_t>(s) * d + lane] = keep ? x[lane] : x0[lane];
  if (lane == 0) vals[s] = keep ? fx : gmin;
}

// g_f of the kernel-matched draw for (draw0 + s, f): grid (ceil(F / 256), draws)
__global__ void __launch_bounds__(kRffThreads) rff_chi2_kernel(uint64_t seed, uint64_t draw0, int F,
                                                               double* __restrict__ out) {
  const int s = blockIdx.y, f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F) out[static_cast<size_t>(s) * F + f] = rff_chi2_at(seed, draw0 + s, f);
}

// The sample functions f_p(x) = c sum_f theta_pf cos(W_pf x + b_pf) (and with G, grad = -c sum_f theta_pf sin(.) W_pf)
// at points x_j: grid (CTAs, functions of the chunk).  Points are shared ([nx][d]) or per function (pts_stride = nx d);
// each thread owns points (grid-stride) and runs rff_accumulate over the features staged kRffGridTile at a time, so a
// value is a pure function of (function, point): not of the batch, the chunk or the launch shape.
template <bool G>
__global__ void __launch_bounds__(kRffThreads) rff_eval_kernel(int F, int d, double c, const double* __restrict__ W,
                                                               const double* __restrict__ b,
                                                               const double* __restrict__ theta,
                                                               const double* __restrict__ pts, size_t pts_stride,
                                                               int nx, double* __restrict__ vals,
                                                               double* __restrict__ grads) {
  extern __shared__ double gs[];  // [kRffGridTile][d] W, [kRffGridTile] b, [kRffGridTile] theta
  const int p = blockIdx.y, tid = threadIdx.x;
  double* Wt = gs;
  double* bt = Wt + kRffGridTile * d;
  double* tt = bt + kRffGridTile;
  const double* Ws = W + static_cast<size_t>(p) * F * d;
  const double* bs = b + static_cast<size_t>(p) * F;
  const double* ts = theta + static_cast<size_t>(p) * F;
  const double* P = pts + p * pts_stride;
  for (int base = blockIdx.x * blockDim.x; base < nx; base += gridDim.x * blockDim.x) {  // uniform over the CTA
    const int j = base + tid;
    const bool valid = j < nx;
    double x[CMOE_MAX_DIM], g[CMOE_MAX_DIM];
#pragma unroll
    for (int k = 0; k < CMOE_MAX_DIM; ++k) {
      x[k] = (valid && k < d) ? P[static_cast<size_t>(j) * d + k] : 0.0;
      g[k] = 0.0;
    }
    double acc = 0.0;
    for (int f0 = 0; f0 < F; f0 += kRffGridTile) {
      const int nf = min(kRffGridTile, F - f0);
      __syncthreads();
      for (int e = tid; e < nf * d; e += blockDim.x) Wt[e] = Ws[static_cast<size_t>(f0) * d + e];
      for (int e = tid; e < nf; e += blockDim.x) {
        bt[e] = bs[f0 + e];
        tt[e] = ts[f0 + e];
      }
      __syncthreads();
      if (valid) rff_accumulate<G>(Wt, bt, tt, nf, d, x, acc, g);
    }
    if (!valid) continue;
    const size_t o = static_cast<size_t>(p) * nx + j;
    if (vals) vals[o] = c * acc;
    if (G) {
#pragma unroll
      for (int k = 0; k < CMOE_MAX_DIM; ++k)
        if (k < d) grads[o * d + k] = -c * g[k];
    }
  }
}

}  // namespace

}  // namespace cmoe


namespace cmoe {
namespace {

// The matched draw is a Student-t mixture only for Matern-5/2; a SquareExponential handle's matched draw is the
// reference draw.
bool rff_matern(const cmoe_gp& gp, const cmoe_rff_opts* opts) {
  if (!opts) return false;
  CMOE_REQUIRE(opts->spectral == CMOE_RFF_SPECTRAL_REFERENCE || opts->spectral == CMOE_RFF_SPECTRAL_KERNEL,
               CMOE_ERR_INVALID_VALUE, "opts->spectral must be CMOE_RFF_SPECTRAL_REFERENCE or CMOE_RFF_SPECTRAL_KERNEL");
  return opts->spectral == CMOE_RFF_SPECTRAL_KERNEL && gp.spec.kernel == CMOE_KERNEL_MATERN_NU_2P5;
}

// The sample functions of P draws and, with a grid, their minimisers (the header's contract of
// cmoe_gp_sample_rff_optima_ex; without `optima` it stops after theta, as cmoe_gp_sample_rff_functions does).  Arguments
// are checked by the callers, except those common to both.
void rff_sample(const cmoe_gp* gp, int F, int P, bool optima, const double* domain_bounds, const double* grid, int G,
                uint64_t seed, uint64_t first_draw, const cmoe_rff_table* table, const cmoe_rff_opts* opts, double* points,
                double* values, double* omega, double* b, double* theta) {
  const int d = gp->spec.dim, g = gp->spec.g, N = gp->N;
  const int M = gp->n;
  const int Q = std::min(F, M);
  CMOE_REQUIRE(d >= 1 && d <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, 32]");
  CMOE_REQUIRE(Q <= kMaxSampleQ, CMOE_ERR_BOUNDS, "min(num_features, num_sampled (1 + num_derivatives)) must be <= 8192");
  const size_t phi = static_cast<size_t>(F) * M, gram = static_cast<size_t>(Q) * Q;
  CMOE_REQUIRE(phi <= kSampleWorkspaceBytes / sizeof(double) - gram, CMOE_ERR_BOUNDS,
               "one sample's design matrix and Gram matrix must fit in the 2 GiB sampling workspace");
  if (optima)
    CMOE_REQUIRE(domain_bounds != nullptr && grid != nullptr && points != nullptr && values != nullptr, CMOE_ERR_INVALID_VALUE,
                 "domain_bounds, grid, points or values is NULL");
  const bool woodbury = M < F;
  const bool matern = rff_matern(*gp, opts);
  if (table)
    CMOE_REQUIRE(table->omega && table->b && table->z && (table->eps || !woodbury), CMOE_ERR_INVALID_VALUE,
                 "table field is NULL");
  const bool tchi2 = table && matern;
  if (tchi2) {
    CMOE_REQUIRE(opts->chi2 != nullptr, CMOE_ERR_INVALID_VALUE, "opts->chi2 is NULL (kernel-matched table mode)");
    for (size_t e = 0; e < static_cast<size_t>(P) * F; ++e)
      CMOE_REQUIRE(std::isfinite(opts->chi2[e]) && opts->chi2[e] > 0.0, CMOE_ERR_INVALID_VALUE,
                   "opts->chi2 entries must be finite and > 0");
  }
  RffBox box{};
  if (optima) {
    for (int k = 0; k < d; ++k) {
      box.lo[k] = domain_bounds[2 * k];
      box.hi[k] = domain_bounds[2 * k + 1];
      CMOE_REQUIRE(std::isfinite(box.lo[k]) && std::isfinite(box.hi[k]) && box.lo[k] <= box.hi[k],
                   CMOE_ERR_INVALID_VALUE, "domain bounds must be finite with min <= max");
    }
    for (size_t e = 0; e < static_cast<size_t>(G) * d; ++e)
      CMOE_REQUIRE(std::isfinite(grid[e]), CMOE_ERR_INVALID_VALUE, "grid points must be finite");
  }
  for (int t = 0; t <= g; ++t)
    CMOE_REQUIRE(gp->hnoise[t] > 0.0, CMOE_ERR_INVALID_VALUE, "noise variances must be > 0");
  require_device(gp->device);

  RffShape sh{};
  sh.F = F;
  sh.M = M;
  sh.N = N;
  sh.d = d;
  sh.g = g;
  sh.woodbury = woodbury ? 1 : 0;
  sh.matern = matern ? 1 : 0;
  sh.c = std::sqrt(2.0 * gp->spec.alpha / F);
  for (int k = 0; k < d; ++k) sh.len[k] = gp->hlengths[k];
  for (int t = 0; t <= g; ++t) sh.sqrt_nu[t] = std::sqrt(gp->hnoise[t]);
  for (int k = 0; k < g; ++k) sh.derivs[k] = gp->spec.derivs[k];
  // y' = y[:, t] / sqrt(nu_t), type-major (the reference's flatten('F'))
  std::vector<double> hyp(M);
  for (int t = 0; t <= g; ++t)
    for (int i = 0; i < N; ++i) hyp[static_cast<size_t>(t) * N + i] = gp->hy[static_cast<size_t>(i) * (1 + g) + t] / sh.sqrt_nu[t];

  cudaStream_t s = gp->stream;
  const int nsteps = (Q + NB - 1) / NB;
  const int gx = optima ? static_cast<int>(std::min<size_t>(kRffGridCtas, (static_cast<size_t>(G) + kRffThreads - 1) / kRffThreads))
                        : 0;
  const size_t per = sizeof(double) * (phi + gram + static_cast<size_t>(nsteps) * NB * NB +
                                       static_cast<size_t>(F) * (d + 4) + M + static_cast<size_t>(gx) + 2 * d + 1 +
                                       (table ? static_cast<size_t>(F) * (d + 2) + M : 0) +
                                       (tchi2 ? static_cast<size_t>(F) : 0)) +
                     sizeof(int) * (static_cast<size_t>(gx) + 2);
  const int chunk = static_cast<int>(chunk_items(P, kSampleWorkspaceBytes, per, kMaxChunkSets));
  SampleWork& w = sample_work(*gp);
  w.V.ensure(static_cast<size_t>(chunk) * phi);
  w.A.ensure(static_cast<size_t>(chunk) * gram);
  w.fail.ensure(chunk);
  if (optima) {
    w.part_v.ensure(static_cast<size_t>(chunk) * gx);
    w.part_i.ensure(static_cast<size_t>(chunk) * gx);
    w.amin.ensure(chunk);
  }
  DevBuf<double> dX, dyp, dgrid, dW(static_cast<size_t>(chunk) * F * d), db(static_cast<size_t>(chunk) * F),
      dth(static_cast<size_t>(chunk) * F), dwc(optima ? static_cast<size_t>(chunk) * F : 0), dvmin(optima ? chunk : 0),
      dpts(optima ? static_cast<size_t>(chunk) * d : 0), dvals(optima ? chunk : 0), dz(static_cast<size_t>(chunk) * F),
      deps(woodbury ? static_cast<size_t>(chunk) * M : 1), tom, tb, tchi;
  dX.upload(gp->hX.data(), static_cast<size_t>(N) * d, s);
  dyp.upload(hyp.data(), M, s);
  if (optima) dgrid.upload(grid, static_cast<size_t>(G) * d, s);
  const size_t smem_gram = 2 * static_cast<size_t>(NB) * LDT * sizeof(double);
  const size_t smem_theta = (static_cast<size_t>(Q) + NB * (NB + 1)) * sizeof(double);
  const size_t smem_grid = static_cast<size_t>(kRffGridTile) * (d + 2) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(rff_gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_gram)));
  CMOE_CUDA(cudaFuncSetAttribute(rff_theta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_theta)));
  std::vector<int> hfail(chunk);
  for (int c0 = 0; c0 < P; c0 += chunk) {
    const int nc = std::min(chunk, P - c0);
    const uint64_t draw0 = first_draw + c0;
    if (table) {
      tom.upload(table->omega + static_cast<size_t>(c0) * F * d, static_cast<size_t>(nc) * F * d, s);
      tb.upload(table->b + static_cast<size_t>(c0) * F, static_cast<size_t>(nc) * F, s);
      dz.upload(table->z + static_cast<size_t>(c0) * F, static_cast<size_t>(nc) * F, s);
      if (woodbury) deps.upload(table->eps + static_cast<size_t>(c0) * M, static_cast<size_t>(nc) * M, s);
      if (tchi2) tchi.upload(opts->chi2 + static_cast<size_t>(c0) * F, static_cast<size_t>(nc) * F, s);
    }
    rff_features_kernel<<<dim3((std::max(F, M) + kRffThreads - 1) / kRffThreads, nc), kRffThreads, 0, s>>>(
        sh, seed, draw0, table ? tom.p : nullptr, table ? tb.p : nullptr, tchi2 ? tchi.p : nullptr, dW.p, db.p, dz.p,
        deps.p);
    const int nfast = woodbury ? F : M, nslow = woodbury ? M : F, fx = (nfast + kRffThreads - 1) / kRffThreads;
    const int zs = std::max(1, std::min(nslow, 4096 / std::max(1, fx * nc)));
    rff_design_kernel<<<dim3(fx, nc, zs), kRffThreads, 0, s>>>(sh, dX.p, dW.p, db.p, w.V.p);
    const int t = (Q + NB - 1) / NB;
    rff_gram_kernel<<<dim3(t * (t + 1) / 2, 1, nc), kRffTileThreads, smem_gram, s>>>(w.V.p, woodbury ? F : M, Q,
                                                                                     w.A.p);
    count_launch(3);
    CMOE_CUDA(cudaGetLastError());
    CMOE_CUDA(cudaMemsetAsync(w.fail.p, 0, nc * sizeof(int), s));
    potrf_batched(w.A.p, Q, nc, w.fail.p, w.stage, s);
    rff_theta_kernel<<<nc, kRffThreads, smem_theta, s>>>(sh, w.V.p, dyp.p, w.A.p, w.fail.p, dz.p, deps.p, dth.p);
    count_launch(1);
    if (optima) {
      rff_grid_kernel<<<dim3(gx, nc), kRffThreads, smem_grid, s>>>(sh, dgrid.p, G, dW.p, db.p, dth.p, w.part_v.p,
                                                                   w.part_i.p);
      best_of_parts_kernel<false><<<(nc + 127) / 128, 128, 0, s>>>(nc, gx, w.part_v.p, w.part_i.p, w.amin.p, dvmin.p);
      rff_opt_kernel<<<(nc + kRffOptWarps - 1) / kRffOptWarps, kRffOptWarps * 32, 0, s>>>(
          sh, nc, box, dgrid.p, w.amin.p, dvmin.p, dW.p, db.p, dth.p, dwc.p, dpts.p, dvals.p);
      count_launch(3);
    }
    CMOE_CUDA(cudaGetLastError());
    w.fail.download(hfail.data(), nc, s);
    if (optima) {
      dpts.download(points + static_cast<size_t>(c0) * d, static_cast<size_t>(nc) * d, s);
      dvals.download(values + c0, nc, s);
    }
    if (omega) dW.download(omega + static_cast<size_t>(c0) * F * d, static_cast<size_t>(nc) * F * d, s);
    if (b) db.download(b + static_cast<size_t>(c0) * F, static_cast<size_t>(nc) * F, s);
    if (theta) dth.download(theta + static_cast<size_t>(c0) * F, static_cast<size_t>(nc) * F, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    for (int c = 0; c < nc; ++c)
      if (hfail[c] != 0)
        throw Error(CMOE_ERR_SINGULAR, "random-feature Gram matrix singular (non-finite data?)", hfail[c]);
  }
}

}  // namespace
}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_gp_sample_rff_optima(const cmoe_gp* gp, int num_features, int num_points,
                                         const double* domain_bounds, const double* grid, int num_grid,
                                         uint64_t seed, uint64_t first_draw, const cmoe_rff_table* table,
                                         double* points, double* values, double* omega, double* b, double* theta,
                                         int* info) {
  return cmoe_gp_sample_rff_optima_ex(gp, num_features, num_points, domain_bounds, grid, num_grid, seed, first_draw,
                                      table, nullptr, points, values, omega, b, theta, info);
}

extern "C" int cmoe_gp_sample_rff_optima_ex(const cmoe_gp* gp, int num_features, int num_points,
                                            const double* domain_bounds, const double* grid, int num_grid,
                                            uint64_t seed, uint64_t first_draw, const cmoe_rff_table* table,
                                            const cmoe_rff_opts* opts, double* points, double* values, double* omega,
                                            double* b, double* theta, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_features >= 1 && num_points >= 1 && num_grid >= 1, CMOE_ERR_BOUNDS,
                 "num_features, num_points and num_grid must be >= 1");
    CMOE_REQUIRE(gp != nullptr, CMOE_ERR_INVALID_VALUE, "gp is NULL");
    rff_sample(gp, num_features, num_points, true, domain_bounds, grid, num_grid, seed, first_draw, table, opts, points,
               values, omega, b, theta);
  });
}

extern "C" int cmoe_gp_sample_rff_functions(const cmoe_gp* gp, int num_features, int num_points, uint64_t seed,
                                            uint64_t first_draw, const cmoe_rff_table* table,
                                            const cmoe_rff_opts* opts, double* omega, double* b, double* theta,
                                            int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_features >= 1 && num_points >= 1, CMOE_ERR_BOUNDS, "num_features and num_points must be >= 1");
    CMOE_REQUIRE(gp != nullptr, CMOE_ERR_INVALID_VALUE, "gp is NULL");
    CMOE_REQUIRE(omega != nullptr && b != nullptr && theta != nullptr, CMOE_ERR_INVALID_VALUE,
                 "omega, b or theta is NULL");
    rff_sample(gp, num_features, num_points, false, nullptr, nullptr, 0, seed, first_draw, table, opts, nullptr, nullptr,
               omega, b, theta);
  });
}

extern "C" int cmoe_rff_chi2_draws(uint64_t seed, uint64_t first_draw, int num_draws, int num_features, double* out,
                                   int device) {
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(num_draws >= 1 && num_features >= 1, CMOE_ERR_BOUNDS, "num_draws and num_features must be >= 1");
    CMOE_REQUIRE(num_draws <= static_cast<int>(kMaxGridY), CMOE_ERR_BOUNDS, "num_draws must be <= 65535");
    CMOE_REQUIRE(out != nullptr, CMOE_ERR_INVALID_VALUE, "out is NULL");
    require_device(device);
    DevBuf<double> dout(static_cast<size_t>(num_draws) * num_features);
    rff_chi2_kernel<<<dim3((num_features + kRffThreads - 1) / kRffThreads, num_draws), kRffThreads>>>(
        seed, first_draw, num_features, dout.p);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    CMOE_CUDA(cudaMemcpy(out, dout.p, dout.count * sizeof(double), cudaMemcpyDeviceToHost));
  });
}

extern "C" int cmoe_rff_evaluate(int dim, int num_features, int num_functions, const double* omega, const double* b,
                                 const double* theta, double c, const double* points, int num_points, int per_function,
                                 double* values, double* grads, int device, int* info) {
  return guarded(info, [&] {
    const int d = dim, F = num_features, P = num_functions, X = num_points;
    CMOE_REQUIRE(d >= 1 && d <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, 32]");
    CMOE_REQUIRE(F >= 1 && P >= 1 && X >= 1, CMOE_ERR_BOUNDS, "num_features, num_functions and num_points must be >= 1");
    CMOE_REQUIRE(omega != nullptr && b != nullptr && theta != nullptr && points != nullptr, CMOE_ERR_INVALID_VALUE,
                 "omega, b, theta or points is NULL");
    CMOE_REQUIRE(values != nullptr || grads != nullptr, CMOE_ERR_INVALID_VALUE, "values and grads are both NULL");
    const bool pf = per_function != 0;
    // doubles of one function's features, and per point of one function (its outputs and, per function, its point)
    const size_t fdbl = static_cast<size_t>(F) * (d + 2);
    const size_t pdbl = (values ? 1 : 0) + (grads ? static_cast<size_t>(d) : 0) + (pf ? static_cast<size_t>(d) : 0);
    const size_t sdbl = pf ? 0 : static_cast<size_t>(d);  // per shared point
    const size_t budget = kSampleWorkspaceBytes / sizeof(double);
    CMOE_REQUIRE(fdbl + pdbl + sdbl <= budget, CMOE_ERR_BOUNDS,
                 "one function's features and one point must fit in the 2 GiB workspace");
    CMOE_REQUIRE(std::isfinite(c), CMOE_ERR_INVALID_VALUE, "c must be finite");
    const size_t nf = static_cast<size_t>(P) * F;
    for (size_t e = 0; e < nf * d; ++e)
      CMOE_REQUIRE(std::isfinite(omega[e]), CMOE_ERR_INVALID_VALUE, "omega must be finite");
    for (size_t e = 0; e < nf; ++e)
      CMOE_REQUIRE(std::isfinite(b[e]) && std::isfinite(theta[e]), CMOE_ERR_INVALID_VALUE, "b and theta must be finite");
    const size_t npts = (pf ? static_cast<size_t>(P) : 1) * X * d;
    for (size_t e = 0; e < npts; ++e)
      CMOE_REQUIRE(std::isfinite(points[e]), CMOE_ERR_INVALID_VALUE, "points must be finite");
    require_device(device);

    // chunk: xc points of pc functions; points first (all of them for one function if they fit), then functions
    const size_t xc = std::min<size_t>(X, (budget - fdbl) / (pdbl + sdbl));
    const size_t pc = std::min<size_t>({static_cast<size_t>(P), (budget - xc * sdbl) / (fdbl + xc * pdbl), kMaxGridY});
    cudaStream_t s;
    CMOE_CUDA(cudaStreamCreate(&s));
    struct StreamGuard {
      cudaStream_t s;
      ~StreamGuard() { cudaStreamDestroy(s); }
    } sg{s};
    DevBuf<double> dW(pc * F * d), db(pc * F), dth(pc * F), dp((pf ? pc : 1) * xc * d), dv(values ? pc * xc : 0),
        dg(grads ? pc * xc * d : 0);
    const size_t smem = static_cast<size_t>(kRffGridTile) * (d + 2) * sizeof(double);
    for (size_t p0 = 0; p0 < static_cast<size_t>(P); p0 += pc) {
      const size_t np = std::min(pc, P - p0);
      dW.upload(omega + p0 * F * d, np * F * d, s);
      db.upload(b + p0 * F, np * F, s);
      dth.upload(theta + p0 * F, np * F, s);
      for (size_t x0 = 0; x0 < static_cast<size_t>(X); x0 += xc) {
        const size_t nx = std::min(xc, X - x0);
        const bool whole = nx == static_cast<size_t>(X);  // the chunk's rows are contiguous on the host
        if (pf && whole) {
          dp.upload(points + p0 * X * d, np * X * d, s);
        } else if (pf) {
          // rows of the chunk's functions, each nx points from x0 on, packed at stride nx d
          for (size_t q = 0; q < np; ++q)
            CMOE_CUDA(cudaMemcpyAsync(dp.p + q * nx * d, points + ((p0 + q) * X + x0) * d, nx * d * sizeof(double),
                                      cudaMemcpyHostToDevice, s));
        } else {
          dp.upload(points + x0 * d, nx * d, s);
        }
        const int gx = static_cast<int>(std::min<size_t>(kRffGridCtas, (nx + kRffThreads - 1) / kRffThreads));
        const dim3 grid_dim(gx, static_cast<unsigned>(np));
        if (grads)
          rff_eval_kernel<true><<<grid_dim, kRffThreads, smem, s>>>(F, d, c, dW.p, db.p, dth.p, dp.p, pf ? nx * d : 0,
                                                                    static_cast<int>(nx), dv.p, dg.p);
        else
          rff_eval_kernel<false><<<grid_dim, kRffThreads, smem, s>>>(F, d, c, dW.p, db.p, dth.p, dp.p, pf ? nx * d : 0,
                                                                     static_cast<int>(nx), dv.p, nullptr);
        count_launch();
        CMOE_CUDA(cudaGetLastError());
        if (whole) {
          dv.download(values ? values + p0 * X : nullptr, values ? np * X : 0, s);
          dg.download(grads ? grads + p0 * X * d : nullptr, grads ? np * X * d : 0, s);
        }
        for (size_t q = 0; q < np && !whole; ++q) {
          if (values)
            CMOE_CUDA(cudaMemcpyAsync(values + (p0 + q) * X + x0, dv.p + q * nx, nx * sizeof(double),
                                      cudaMemcpyDeviceToHost, s));
          if (grads)
            CMOE_CUDA(cudaMemcpyAsync(grads + ((p0 + q) * X + x0) * d, dg.p + q * nx * d, nx * d * sizeof(double),
                                      cudaMemcpyDeviceToHost, s));
        }
        CMOE_CUDA(cudaStreamSynchronize(s));
      }
    }
  });
}

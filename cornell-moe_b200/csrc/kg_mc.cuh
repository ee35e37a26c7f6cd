// Fused q-KG Monte-Carlo kernels (the north-star hot path).
//
// One MC sample-evaluation of the reference = fantasise y = mu + L z at the q candidate points, re-solve K^-1 y on the
// (N+q) system, scan the discretisation set for the arg-min of the new posterior mean and run a line-search gradient
// descent from it (gpp_knowledge_gradient_optimization.cpp:87-113, 420-472; gpp_optimization.hpp:708-828).
// Here the re-solve is replaced by the algebraically identical rank-q update (SURVEY.md Appendix B)
//     mu+(x) = m + sum_j (beta_j - B_j . c) k(x, X_j) + sum_u c_u k(x, Xu_u),      c = L^-T z,  B = K^-1 K*
// so a sample touches no HBM at all: the per-candidate operands (scaled X, beta, B) are staged once per CTA into shared
// memory with TMA bulk copies and every lane runs one sample's whole inner optimisation out of registers.
//
// Mapping: one thread per MC sample; grid = (sample chunks, candidates).  Lanes that finish fetch the next sample of
// the chunk from a shared counter, so a warp only idles at the very end of a chunk although the line search has
// data-dependent trip counts.  The line search is a per-lane state machine around two warp-uniform routines:
// "evaluate mu+ and its gradient at my query point" (POINT round) and "evaluate all backtracking trials of this step
// along my gradient" (LINE round: eval_line / eval_line_gen for the SquareExponential kernel, eval_line_matern for
// Matern-5/2 without derivative observations); a warp vote picks the kind of round, see kg_mc_body.
// With derivative observations (kg_mc_gen_kernel) the per-sample weights are formed once per sample and streamed back
// through a per-lane cp.async ring (fill_*_weights, stream_point_weights).
#pragma once

#include <algorithm>
#include <initializer_list>
#include <type_traits>

#include "device_math.cuh"
#include "internal.cuh"

#include "linalg_dev.cuh"
#include "ptx_util.cuh"

namespace cmoe {

// Range contract of the shared-memory fast path.  Its exp (exp_tab, no per-call guard) needs |t| < 2^31 ln2 / 64 =
// 2.3e7, t = -|x~ - X~_j|^2 / 2 + ln(alpha).  All operands of these kernels (training, union, start points, inner
// bounds, minimisers) share the centred frame of the GP's covariance build, x~ = (x - centre) / l (kg.cu), because the
// expanded form x~.X~ - |x~|^2/2 - |X~|^2/2 loses ~eps |x~|^2 absolute; the radii below are measured in that frame.  The
// host only selects the fast path while every scaled operand (training, union, discrete points, inner-domain corners)
// lies within kFastPathRadius of the origin; a query point farther than kFarRadius is then at least kFarRadius -
// kFastPathRadius = 2000 length scales from every operand, so all its kernel values are exactly 0 and the evaluation is
// short-circuited; any other query point has |t| <= 6000^2 / 2 = 1.8e7.
#ifndef CMOE_MC_THREADS
#define CMOE_MC_THREADS 128
#endif
#ifndef CMOE_MC_MINBLOCKS
#define CMOE_MC_MINBLOCKS 3
#endif
constexpr int kMcThreads = CMOE_MC_THREADS;

constexpr double kFastPathRadius = 2000.0;
constexpr double kFarRadius = 4000.0;

struct KgMcParams {
  int N;        // training points
  int U;        // union points (= rows, g == 0)
  int ps;       // free coordinates (dim - num_fidelity)
  int dim;
  int M;        // discretisation set size (U + num_pts)
  int num_mc;
  int chunk;    // samples per CTA
  int use_smem;
  int g;          // derivative observations per point (0 on the fast path)
  int Q;          // rows of the union block = U * (1 + g)
  int pk_stride;  // doubles per training point in Pk: QP + 2 (g == 0) or 2 (g > 0: e_j only, the weights live in Wt)
  int derivs[CMOE_MAX_DIM];  // observed partial-derivative indices (g <= 8 on the narrow general path, <= 31 wide)
  int drow[CMOE_MAX_DIM];    // wide general path: row 1 + m of coordinate d = derivs[m] in a point's block, else 0
  int max_steps, max_restarts;
  double mean, mrc, tol, step_tol, alpha;
  const double* Xt;      // [N][DIM] scaled training points (zero padded)
  const double* Pk;      // [nc][N][QP+2]  (e_j, beta_j, B_j[0..QP))
  const double* Xu;      // [nc][U][DIM+2] (scaled union point, e_u, pad)
  const double* A;       // [nc][M][DIM]   unscaled start points minus the centre (fidelity coords = 1, padding = 0)
  const double* recC;    // [nc][num_mc][QP]
  const int* recStart;   // [nc][num_mc]
  const double* Start;   // g == 0: [nc][M][1+QP][DIM+2] start-point table (kg_start_kernel)
  const double* alpha0;  // [max_steps]  pre_mult * (i+1)^-gamma
  double* outVal;        // [nc][num_mc]   -mu+(x*)  (the reference's best_function_value)
  double* outX;          // [nc][num_mc][DIM] scaled minimiser
  double* outH;          // [nc][num_mc]      -|scaled minimiser|^2 / 2 (consumed by kg_acc_kernel)
  unsigned long long* stats;  // [4]: posterior evaluations, accepted steps, point rounds, line batches (per lane)
  // general path (derivative observations): per-candidate weight table and the per-lane weight columns
  const double* Wt;  // [nc][1 + QP][N * (1+g)]: row 0 = beta~, row 1+u = B~[:, u]  (~: derivative rows divided by l_t)
  double* aw;        // [aw_slots][N * (1+g)][kMcThreads]: a = beta~ - B~ c of the sample each lane is working on
  int* work;         // work-item counter of the persistent grid (zeroed before the launch)
  int aw_slots;      // resident CTAs the scratch was sized for
  int chunks;        // work items per candidate
  int work_total;    // chunks * candidates of this launch
  int stage_ops;     // general path: scaled training points and e_j fit next to the ring in shared memory
  double lo[CMOE_MAX_DIM], hi[CMOE_MAX_DIM], inv_len[CMOE_MAX_DIM];  // lo, hi: minus the centre
};

struct KgAccParams {
  int N, U, dim, num_mc;
  int fast_exp;  // 1: the range contract of the table exp holds (see kFastPathRadius)
  int g;          // derivative observations per point (general path: rows = (N + U) * (1 + g))
  int derivs[CMOE_MAX_DIM];
  double inv_len[CMOE_MAX_DIM];
  double alpha;
  const double* Xt;     // [N][DIM]
  const double* Xu;     // [nc][U][DIM+2]
  const double* recC;   // [nc][num_mc][QP]
  const double* outX;   // [nc][num_mc][DIM]
  const double* outH;   // [nc][num_mc]  -|x*|^2/2
  double* R;            // [nc][QP][N+U]   R[a][row] = sum_i c_ia k(row, x*_i)
  double* Gu;           // [nc][U][DIM]    sum_i c_iu Bpart(Xu_u, x*_i) x~*_i
  double* GkB;          // [nc][U]         sum_i c_iu Bpart(Xu_u, x*_i)
};

// exp(t) = 2^k * 2^(i/64) * e^r with |r| <= ln2/128: 64-entry table in shared memory + degree-5 Taylor polynomial
// (truncation r^6/720 <= 3.5e-17 relative).  10 FP64-pipe instructions instead of 15 for exp_fast; same integer-side
// clamp of the exponent, NO guard for |t| >= 2.3e7 (see kFastPathRadius).  Used by the shared-memory fast path of the
// fused q-KG kernel (+11 % throughput on the north-star shape).  Arguments: t <= 700 down to -(2 kFastPathRadius)^2 / 2
// and on to -2.3e7.  Max relative error 4.0e-16 over [-1000 ln2, 700], below that a result in [0, 2^-999]; exp(0) = 1
// exactly.  An empirical bound ~20 % above the 3.30e-16 measured on the device (tests/test_gpu_fast_math.py): the table
// entry (0.5 u, u = 2^-53), the polynomial (~1.2 u, as exp_fast's) and the product p * 2^(i/64) (0.5 u) add up to ~2.5 u,
// the truncation r^6/720 adds 0.3 u.
__device__ const double kExp2Table[64] = {
#include "exp2_table64.inc"
};
__shared__ double g_exp_tab[64];
__device__ __forceinline__ void exp_table_stage() {
  if (threadIdx.x < 64) g_exp_tab[threadIdx.x] = kExp2Table[threadIdx.x];
  __syncthreads();
}
__device__ __forceinline__ double exp_tab(double t) { return exp_tab64(t, g_exp_tab); }
// exp(t) = 2^k * 2^(i/2048) * e^r with |r| <= ln2/4096: 2048-entry table (16 KB of shared memory) + degree-3 Taylor
// polynomial (truncation r^4/24 <= 3.4e-17 relative).  8 FP64-pipe instructions.  Same range contract as exp_tab
// (kFastPathRadius), no per-call guard: n = round(t 2048 / ln2) no longer fits the low word for |t| >= 7.3e5, so the
// exponent k = n >> 11 is taken from both words of the shifted double with one funnel shift (the shift's bias
// 2^51 >> 11 = 2^40 vanishes mod 2^32); k is exact for |t| < 2^31 ln2 = 1.5e9 and clamped on the integer side like
// exp_tab's.  Used by the union rows of kg_acc_tile_kernel; the tile rows of that kernel and of the BIG build of
// kg_mc_kernel<SE,8,8> take the same table through exp2k_shifted below.  Arguments and error as exp_tab's: max relative
// error 4.0e-16 over [-1000 ln2, 700] (tests/test_gpu_fast_math.py), exp(0) = 1 exactly.
__device__ const double kExp2Table2k[2048] = {
#include "exp2_table2048.inc"
};
__shared__ double g_exp_tab2k[2048];
__device__ __forceinline__ void exp_table2k_stage() {
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) g_exp_tab2k[i] = kExp2Table2k[i];
  __syncthreads();
}
constexpr double kExp2kShift = 6755399441055744.0;  // 1.5 2^52: t + kExp2kShift rounds t to an integer in the low bits
constexpr double kKappa = 2048.0 * 1.4426950408889634;  // 2048 log2(e): natural units -> 2048ths of a binary exponent
// exponent n (of 2^(n/2048)) from the shifted double nfs = n + 1.5 2^52: table index from the low word, k = n >> 11 from
// both words with one funnel shift, clamped on the integer side
__device__ __forceinline__ int exp2k_index(double nfs) { return __double2loint(nfs) & 2047; }
__device__ __forceinline__ int exp2k_exponent(double nfs) {
  const unsigned lo = static_cast<unsigned>(__double2loint(nfs)), hi = static_cast<unsigned>(__double2hiint(nfs));
  return max(static_cast<int>(__funnelshift_r(lo, hi, 11)), -1000);
}
// 2^(n/2048) (1 + c1 r + c2 r^2 + c3 r^3): the polynomial, the table multiply and the exponent patch of the 2048-entry
// exps
__device__ __forceinline__ double exp2k_tail(double r, double c1, double c2, double c3, double nfs) {
  double p = c3;
  p = fma(p, r, c2);
  p = fma(p, r, c1);
  p = fma(p, r, 1.0);
  p *= g_exp_tab2k[exp2k_index(nfs)];
  return __hiloint2double(__double2hiint(p) + (exp2k_exponent(nfs) << 20), __double2loint(p));
}
__device__ __forceinline__ double exp_tab2k_round(double t) { return fma(t, kKappa, kExp2kShift); }
__device__ __forceinline__ double exp_tab2k(double t) {
  const double nfs = exp_tab2k_round(t);
  const double nf = nfs - kExp2kShift;
  double r = fma(nf, -6.93147180369123816490e-01 / 2048.0, t);
  r = fma(nf, -1.90821492927058770002e-10 / 2048.0, r);
  return exp2k_tail(r, 1.0, 0.5, 1.6666666666666666e-01, nfs);
}
// 2^((t + H) / 2048) for an integer H, |H| < 2^51, passed as the rounding constant C = 1.5 2^52 + H (exp2k_split): the
// same table, polynomial and exponent patch as exp_tab2k, with the argument already in 2048ths of a binary exponent
// (t = kKappa x the natural one).  nfs = t + C rounds t + H to the integer n in the low bits; m = nfs - C = n - H and
// r = t - m (|r| <= 1/2) are exact, so there is no Cody-Waite pair: 7 FP64-pipe instructions.  Arguments: t + H down to
// kKappa x the range contract of exp_tab2k (|t + H| < 2^31 x 2048 keeps k exact); t alone may be anything below 2^51.
// Max relative error 4.0e-16 (exp_tab2k's bound) over t + H in kKappa x [-1000 ln2, 700], against 2^((t + H) / 2048)
// (tests/test_gpu_fast_math_exp2k.py), exactly 1 at t = 0, H = 0.  Relative to exp((t + H) / kKappa) the result carries
// the rounding of kKappa (1.4e-17 relative) times |t + H| / kKappa: an argument error of the order of rounding the
// argument itself.
constexpr double kExp2kC1 = 6.93147180559945309417e-01 / 2048.0;  // (ln2 / 2048)^k / k!
constexpr double kExp2kC2 = kExp2kC1 * kExp2kC1 / 2.0;
constexpr double kExp2kC3 = kExp2kC1 * kExp2kC1 * kExp2kC1 / 6.0;
__device__ __forceinline__ double exp2k_shifted(double t, double C) {
  const double nfs = t + C;
  const double r = t - (nfs - C);
  return exp2k_tail(r, kExp2kC1, kExp2kC2, kExp2kC3, nfs);
}
// A per-sample exponent term h (natural units) as exp2k_shifted's rounding constant C = 1.5 2^52 + rint(kKappa h) and the
// factor f = 2^((kKappa h - rint(kKappa h)) / 2048) that the rounding leaves, |kKappa h - rint| <= 1/2 (exact):
// exp2k_shifted(kKappa t, C) f = exp(t + h), and no partial exponent can overflow.
__device__ __forceinline__ void exp2k_split(double h, double& C, double& f) {
  const double H = kKappa * h, Hi = rint(H);
  C = kExp2kShift + Hi;
  const double r = H - Hi;
  f = fma(fma(fma(kExp2kC3, r, kExp2kC2), r, kExp2kC1), r, 1.0);
}
// The exp of the tile rounds, exp(t + h) for a row's exponent t and a sample's h (hs: the sample's term as the tile
// rounds pass it).  BIG (the kernel staged the 2048-entry table): t comes from kKappa-scaled operands and hs is
// exp2k_split's rounding constant, and the caller applies the split's factor f to its sums; else exp_tab(t + h).
template <bool BIG>
__device__ __forceinline__ double exp_row(double t, double hs) {
  if (BIG) return exp2k_shifted(t, hs);
  return exp_tab(t + hs);
}
template <bool TAB>
__device__ __forceinline__ double exp_sel(double t) {
  if (TAB) return exp_tab(t);
  return exp_fast(t);
}

// Kernel-specific pieces.  pk0 holds e_j = ln(alpha) - |x~_j|^2/2 for SE and |x~_j|^2 for Matern; hq = -|x~|^2/2.
// Returns the value weight kv (k(x, X_j)) and the gradient weight kb (d k / d x_d = kb * (x~_jd - x~_d) / l_d).
template <int KERNEL, bool TAB = false>
__device__ __forceinline__ void kernel_pair(double dot, double pk0, double hq, double alpha, double& kv, double& kb) {
  if (KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL) {
    kv = exp_sel<TAB>(dot + (pk0 + hq));
    kb = kv;
  } else {
    const double r2 = fmax(0.0, pk0 - 2.0 * (hq + dot));
    const double ar = kSqrt5 * sqrt(r2);
    const double ee = alpha * exp_fast(-ar);
    kv = ee * (1.0 + ar + (5.0 / 3.0) * r2);
    kb = (5.0 / 3.0) * ee * (1.0 + ar);
  }
}

// 16-byte loads of the staged operands: LDS.128 when the pointer is known to be shared, LDG.128 (read-only path) else
template <bool SMEM>
__device__ __forceinline__ double2 ld2(const double* p) {
  if (SMEM) {
    return *reinterpret_cast<const double2*>(p);
  } else {
    return __ldg(reinterpret_cast<const double2*>(p));
  }
}

template <bool SMEM>
__device__ __forceinline__ double ld1(const double* p) {
  if (SMEM) return *p;
  return __ldg(p);
}

// a row's DIM scaled coordinates, as 16-byte pairs
template <int DIM, bool SMEM>
__device__ __forceinline__ void load_row(const double* p, double (&xv)[DIM]) {
#pragma unroll
  for (int d = 0; d < DIM; d += 2) {
    const double2 v = ld2<SMEM>(p + d);
    xv[d] = v.x;
    xv[d + 1] = v.y;
  }
}

// c[u], the weight of union row u, selected with compile-time register indices so that c stays in registers
template <int QP>
__device__ __forceinline__ double union_coef(const double (&c)[QP], int u) {
  double cu = 0.0;
#pragma unroll
  for (int v = 0; v < QP; ++v)
    if (v == u) cu = c[v];
  return cu;
}

// x . y and beta - B . c over the staged operands (one dependent DFMA chain each; splitting them into even / odd
// half chains measured 4 % slower: more instructions, no latency win).
template <int DIM>
__device__ __forceinline__ double dot_dim(const double (&x)[DIM], const double (&y)[DIM], double init) {
  double dot = init;
#pragma unroll
  for (int d = 0; d < DIM; ++d) dot = fma(x[d], y[d], dot);
  return dot;
}

template <int QP, bool SMEM>
__device__ __forceinline__ double weight_row(const double* __restrict__ pk, double beta, const double (&c)[QP]) {
  double a = beta;
#pragma unroll
  for (int u = 0; u < QP; u += 2) {
    const double2 b = ld2<SMEM>(pk + 2 + u);
    a = fma(-b.x, c[u], a);
    a = fma(-b.y, c[u + 1], a);
  }
  return a;
}

// ---------------------------------------------------------------------------------------------------------------
// Tile evaluation of the training rows (shared-memory fast path, DESIGN.md K6).  A round is warp-uniform, so the
// three small contractions of a round — x~ . X~_j (and a_min g~ . X~_j on LINE rounds), a_j = beta_j - B_j . c and, on
// POINT rounds, the gradient sums s_d = sum_j w_j X~_jd — are, for one block of 8 training rows, products of shape
// 32 samples x 8 rows x K.  They run on FP64 DMMA m16n8k4 (M = 16 samples: the warp's lanes in two halves, both in
// one row sweep on POINT rounds and one after the other on LINE rounds, N = 8 rows, K = DIM or QP in steps of 4, K
// tails zero-filled); only the exps and the trial arithmetic stay
// element-wise, in the accumulator layout.  Fragment layout (PTX ISA, f64, lane = 4 g + t):
//   A: a0 = A[g][t], a1 = A[g+8][t];   B: b = B[t][g];   C: c0 = C[g][2t], c1 = C[g][2t+1], c2 = C[g+8][2t], c3 = C[g+8][2t+1]
// A sample's row of every product depends on that sample's operands only, and its partial sums over the 8 columns of a
// block are reduced across the quad in a fixed order, so a result does not depend on which lane holds the sample.
// Columns past N (last block) read row N-1 and get weight 0 (and p_j = 0 on LINE rounds): exact zeros, never 0 x inf.
// ---------------------------------------------------------------------------------------------------------------

// Which instantiations run the tile path: the ones measured to gain, SquareExponential at DIM = 8, QP = 8.  All the
// others keep the scalar row loops (DESIGN.md K6 lists both groups).  The tile rounds need ~240 registers per thread
// (kg_mc_min_blocks); with the 168 that 3 CTAs of 128 threads leave, the spill code grows with DIM and QP, and
// Matern-5/2's LINE rounds are dominated by the per-trial sqrt and exp.
template <int KERNEL, int DIM, int QP>
constexpr bool kg_tile_path() {
  return KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL && DIM == 8 && QP == 8;
}

// Trial step sizes per LINE batch of the SquareExponential kernel (eval_line, eval_line_gen).  Each trial costs one
// squaring and one accumulating FMA per row, and a step whose accepted trial lies past the batch costs its lane a
// second LINE round (and, out of phase with its warp, an idle POINT round).  The scalar row loops and the d-KG path
// keep 8.  The tile rounds of <SE,8,8>, where the chain is half of a LINE row's FP64 instructions, take 6: at the
// bench shape no step accepted a trial past index 5 (the accepted-trial histogram in DESIGN.md K6).
constexpr int kLineBatch = 8;
#ifndef CMOE_LINE_BATCH_TILE
#define CMOE_LINE_BATCH_TILE 6
#endif
template <int KERNEL, int DIM, int QP>
constexpr int kg_line_batch() {
  return kg_tile_path<KERNEL, DIM, QP>() ? CMOE_LINE_BATCH_TILE : kLineBatch;
}
static_assert(CMOE_LINE_BATCH_TILE >= 1 && CMOE_LINE_BATCH_TILE <= kLineBatch, "1 <= tile LINE batch <= kLineBatch");

// CTAs of kMcThreads per SM that kg_mc_kernel's launch bounds ask for.  The tile instantiation takes 2, so that it gets
// up to 255 registers (it uses 240 and spills nothing; the 168 that 3 CTAs leave spilled its round-level state).  Its
// operands (72.6 KB at N = 500) leave room for 2 CTAs.  Every other instantiation keeps 3 CTAs (168 registers).
#ifndef CMOE_MC_TILE_MINBLOCKS
#define CMOE_MC_TILE_MINBLOCKS 2
#endif
template <int KERNEL, int DIM, int QP>
constexpr int kg_mc_min_blocks() {
  return kg_tile_path<KERNEL, DIM, QP>() ? CMOE_MC_TILE_MINBLOCKS : CMOE_MC_MINBLOCKS;
}

// A fragments of the half h (samples 16h .. 16h+15) from the lanes' own rows v[0..W): element k is -v[k] (NEG),
// v[k] * scale[k] or, with row factors r0 / r1 (rows g / g+8), r * (v[k] * scale[k]) — the scaling is done after the
// shuffle, so that the lanes keep only their state arrays live, and in the order the scalar path rounds it.
template <int W, bool NEG, bool ROWF = false>
__device__ __forceinline__ void tile_frag(const double (&v)[W], const double* scale, int h, double (&f)[(W + 3) / 4][2],
                                          double r0 = 1.0, double r1 = 1.0) {
  const int lane = threadIdx.x & 31, src = 16 * h + (lane >> 2), t = lane & 3;
#pragma unroll
  for (int ks = 0; ks < (W + 3) / 4; ++ks) {
    f[ks][0] = 0.0;
    f[ks][1] = 0.0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = 4 * ks + e;
      if (k < W) {
        double x0 = __shfl_sync(0xffffffffu, v[k], src);
        double x1 = __shfl_sync(0xffffffffu, v[k], src + 8);
        if (t == e) {
          if (NEG) {
            x0 = -x0;
            x1 = -x1;
          } else if (scale != nullptr) {
            x0 *= scale[k];
            x1 *= scale[k];
          }
          if (ROWF) {
            x0 *= r0;
            x1 *= r1;
          }
          f[ks][0] = x0;
          f[ks][1] = x1;
        }
      }
    }
  }
}

// per-sample scalar of the half h in the C layout: rows g (lo) and g + 8 (hi)
__device__ __forceinline__ void tile_rows(double v, int h, double& lo, double& hi) {
  const int src = 16 * h + ((threadIdx.x & 31) >> 2);
  lo = __shfl_sync(0xffffffffu, v, src);
  hi = __shfl_sync(0xffffffffu, v, src + 8);
}

// fixed-order sum over the quad (the butterfly gives the same bits on all four lanes)
__device__ __forceinline__ double quad_sum(double v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// hands the quad-uniform values of rows (g, g + 8) of half h to the owning lanes 16h + g and 16h + g + 8 (ADD: added
// to the owner's value)
template <bool ADD = false>
__device__ __forceinline__ double tile_to_owner(double lo, double hi, int h, double mine) {
  const int lane = threadIdx.x & 31, src = 4 * (lane & 7);
  const double vl = __shfl_sync(0xffffffffu, lo, src), vh = __shfl_sync(0xffffffffu, hi, src);
  const double v = (lane & 8) ? vh : vl;
  return (lane >> 4) != h ? mine : (ADD ? mine + v : v);
}

// Row operands of one block, shared by all tile rounds: the B-operand row of the dot / weight products (jb = j0 + g)
// and the two C columns of this lane (je0 = j0 + 2t, je1 = j0 + 2t + 1) with their (e_j, beta_j).
template <int QP, bool TAIL>
struct TileRows {
  int jb, je0, je1;
  bool v0, v1;  // columns inside [0, N)
  double2 h0, h1;
  __device__ __forceinline__ TileRows(const double* __restrict__ Pk, int N, int j0) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    jb = j0 + g;
    je0 = j0 + 2 * t;
    je1 = je0 + 1;
    v0 = !TAIL || je0 < N;
    v1 = !TAIL || je1 < N;
    if (TAIL) {
      jb = min(jb, N - 1);
      je0 = min(je0, N - 1);
      je1 = min(je1, N - 1);
    }
    h0 = *reinterpret_cast<const double2*>(Pk + je0 * (QP + 2));
    h1 = *reinterpret_cast<const double2*>(Pk + je1 * (QP + 2));
  }
};

// B fragments of one block (K = W): b[ks] = B[4 ks + t][g] = row[4 ks + t] of the lane's row jb, zero past W
template <int W>
__device__ __forceinline__ void tile_bfrag(const double* row, double (&b)[(W + 3) / 4]) {
  const int t = threadIdx.x & 3;
#pragma unroll
  for (int ks = 0; ks < (W + 3) / 4; ++ks) b[ks] = (4 * ks + t < W) ? row[4 * ks + t] : 0.0;
}

// acc[4] (C layout) += A (K = W, fragments f) x B (fragments b): pairs of k-steps as one m16n8k8 product (half the
// DMMA instructions, which is what they cost when interleaved with the element-wise FP64 work, DESIGN.md K6)
template <int W>
__device__ __forceinline__ void tile_mma(double (&acc)[4], const double (&f)[(W + 3) / 4][2],
                                         const double (&b)[(W + 3) / 4]) {
  constexpr int KS = (W + 3) / 4;
#pragma unroll
  for (int ks = 0; ks + 1 < KS; ks += 2)
    dmma_m16n8k8(acc[0], acc[1], acc[2], acc[3], f[ks][0], f[ks][1], f[ks + 1][0], f[ks + 1][1], b[ks], b[ks + 1]);
  if (KS % 2) dmma_m16n8k4(acc[0], acc[1], acc[2], acc[3], f[KS - 1][0], f[KS - 1][1], b[KS - 1]);
}

// POINT round (SquareExponential) over the training rows: S0 = sum_j a_j k_j and s_d = sum_j a_j k_j X~_jd of every
// lane's query point xq (hq = -|xq|^2 / 2).  One sweep over the rows serves both halves: a block's B fragments and
// (e_j, beta_j) are loaded once and feed the products of samples 0-15 and 16-31.
template <int DIM, int QP, bool BIG>
__device__ __forceinline__ void tile_posterior(const double* __restrict__ Xt, const double* __restrict__ Pk, int N,
                                               const double (&xq)[DIM], const double (&c)[QP], double hq, double& S0,
                                               double (&s)[DIM]) {
  constexpr int KD = (DIM + 3) / 4, KQ = (QP + 3) / 4, ND = (DIM + 7) / 8;
  const int lane = threadIdx.x & 31, g = lane >> 2;
  double xa[2][KD][2], ca[2][KQ][2], hqr[2][2];
  // BIG: exponents in kKappa units (e_j staged scaled, x~ scaled here); hq enters as exp2k_split's (C, f)
  double hs = hq, f = 1.0;
  if (BIG) exp2k_split(hq, hs, f);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    tile_frag<DIM, false, BIG>(xq, nullptr, h, xa[h], kKappa, kKappa);
    // a = beta + (-c) . B: the negation is exact, each product is the scalar one
    tile_frag<QP, true>(c, nullptr, h, ca[h]);
    tile_rows(hs, h, hqr[h][0], hqr[h][1]);
  }
  double s0[2][2], sacc[2][ND][4];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    s0[h][0] = s0[h][1] = 0.0;
#pragma unroll
    for (int n = 0; n < ND; ++n) sacc[h][n][0] = sacc[h][n][1] = sacc[h][n][2] = sacc[h][n][3] = 0.0;
  }
  auto block = [&](int j0, auto tail) {
    constexpr bool TAIL = decltype(tail)::value;
    const TileRows<QP, TAIL> r(Pk, N, j0);
    double bx[KD], bq[KQ], b0[ND], b1[ND];
    tile_bfrag<DIM>(Xt + r.jb * DIM, bx);
    tile_bfrag<QP>(Pk + r.jb * (QP + 2) + 2, bq);
#pragma unroll
    for (int n = 0; n < ND; ++n) {
      const int d = 8 * n + g;
      b0[n] = (d < DIM) ? Xt[r.je0 * DIM + d] : 0.0;
      b1[n] = (d < DIM) ? Xt[r.je1 * DIM + d] : 0.0;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // the exponent's e_j enters as the accumulator seed
      double dot[4] = {r.h0.x, r.h1.x, r.h0.x, r.h1.x};
      double a[4] = {r.h0.y, r.h1.y, r.h0.y, r.h1.y};
      tile_mma<DIM>(dot, xa[h], bx);
      tile_mma<QP>(a, ca[h], bq);
      double w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const double ai = ((i & 1) ? r.v1 : r.v0) ? a[i] : 0.0;
        const double kv = exp_row<BIG>(dot[i], hqr[h][i >> 1]);
        s0[h][i >> 1] = fma(ai, kv, s0[h][i >> 1]);
        w[i] = ai * kv;
      }
      // s += W X~: k-step 0 takes the even columns (rows je0: A = (w0, w2)), k-step 1 the odd ones (rows je1)
#pragma unroll
      for (int n = 0; n < ND; ++n)
        dmma_m16n8k8(sacc[h][n][0], sacc[h][n][1], sacc[h][n][2], sacc[h][n][3], w[0], w[2], w[1], w[3], b0[n], b1[n]);
    }
  };
  const int nfull = N & ~7;
#pragma unroll 1
  for (int j0 = 0; j0 < nfull; j0 += 8) block(j0, std::false_type());
  if (nfull < N) block(nfull, std::true_type());
  S0 = 0.0;
#pragma unroll
  for (int h = 0; h < 2; ++h) S0 = tile_to_owner(quad_sum(s0[h][0]), quad_sum(s0[h][1]), h, S0);
#pragma unroll
  for (int d = 0; d < DIM; ++d) {
    // s[row][d] sits in lane 4 (row & 7) + ((d & 7) >> 1) of the row's quad, register (d & 1) (+ 2 for rows 8..15)
    const int src = 4 * (lane & 7) + ((d & 7) >> 1);
    double v[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const double vl = __shfl_sync(0xffffffffu, sacc[h][d / 8][d & 1], src);
      const double vh = __shfl_sync(0xffffffffu, sacc[h][d / 8][2 + (d & 1)], src);
      v[h] = (lane & 8) ? vh : vl;
    }
    s[d] = (lane >> 4) ? v[1] : v[0];
  }
  if (BIG) {
    // the factor exp2k_split left out of every kv of this lane (before eval_posterior adds the union rows)
    S0 *= f;
#pragma unroll
    for (int d = 0; d < DIM; ++d) s[d] *= f;
  }
}

// mu+(xq) - m  and  the scaled-gradient accumulators, for one query point (scaled coordinates xq).
template <int KERNEL, int DIM, int QP, bool SMEM, bool TILE = false, bool BIG = false>
__device__ __forceinline__ void eval_posterior(const double* __restrict__ Xt, const double* __restrict__ Pk,
                                               const double* __restrict__ Xu, int N, int U, double alpha,
                                               const double (&xq)[DIM], const double (&c)[QP], double& S0, double& SB,
                                               double (&s)[DIM]) {
  static_assert(DIM % 2 == 0 && QP % 2 == 0, "operands are moved as 16-byte pairs");
  double nq = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) nq = fma(xq[d], xq[d], nq);
  const double hq = -0.5 * nq;
  S0 = 0.0;
  SB = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) s[d] = 0.0;
  static_assert(!TILE || KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL, "the tile path is SquareExponential only");
  if (TILE) tile_posterior<DIM, QP, BIG>(Xt, Pk, N, xq, c, hq, S0, s);
  // one row: scaled coordinates xv, exponent term e, weight weight(), taken before the kernel values (the training rows'
  // weight_row loads) or, with late, after them (the union rows' register select)
  auto row = [&](const double (&xv)[DIM], double e, auto weight, auto late) {
    const double dot = dot_dim<DIM>(xq, xv, 0.0);
    double a = 0.0;
    if constexpr (!decltype(late)::value) a = weight();
    double kv, kb;
    kernel_pair<KERNEL, SMEM>(dot, e, hq, alpha, kv, kb);
    if constexpr (decltype(late)::value) a = weight();
    S0 = fma(a, kv, S0);
    const double wb = a * kb;
    if (KERNEL != CMOE_KERNEL_SQUARE_EXPONENTIAL) SB += wb;
#pragma unroll
    for (int d = 0; d < DIM; ++d) s[d] = fma(wb, xv[d], s[d]);
  };
#pragma unroll 2
  for (int j = 0; j < (TILE ? 0 : N); ++j) {
    const double* xj = Xt + j * DIM;
    const double* pk = Pk + j * (QP + 2);
    double xv[DIM];
    load_row<DIM, SMEM>(xj, xv);
    const double2 h = ld2<SMEM>(pk);  // (e_j, beta_j)
    row(xv, h.x, [&] { return weight_row<QP, SMEM>(pk, h.y, c); }, std::false_type());
  }
  for (int u = 0; u < U; ++u) {
    const double* xu = Xu + u * (DIM + 2);
    double xv[DIM];
    load_row<DIM, SMEM>(xu, xv);
    row(xv, ld2<SMEM>(xu + DIM).x, [&] { return union_coef<QP>(c, u); }, std::true_type());
  }
  if (KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL) SB = S0;
  if (SMEM && nq > kFarRadius * kFarRadius) {
    // farther than kFarRadius length scales from everything: every kernel value is exactly 0 (see kFastPathRadius)
    S0 = 0.0;
    SB = 0.0;
#pragma unroll
    for (int d = 0; d < DIM; ++d) s[d] = 0.0;
  }
}

// Batched backtracking for the SquareExponential kernel.  The reference's line search tries x + a_k g for
// a_k = a_0 2^-k one value-evaluation at a time (gpp_optimization.hpp:750-765).  Along a line the SE kernel factorises:
//     ln k(x + a g, X_j) = ln k(x, X_j) + a p_j - a^2 |g~|^2 / 2 ,   p_j = g~ . (X~_j - x~)
// so with F_j = exp(a_min p_j) the kernel at every trial point is k(x, X_j) F_j^(2^m) times a j-independent factor:
// two exps per training point give all KB trial values by repeated squaring (1 mul + 1 fma per trial) instead of one
// full evaluation (dot + weights + exp) per trial.  S[k] = sum_j a_j k(x, X_j) exp(a_k p_j) for a_k = a_min 2^(KB-1-k'),
// returned in trial order (S[0] <-> largest step); pmax_hi (high word of max_j |a_min p_j|) lets the caller reject
// batches whose factors could leave the double range (it then falls back to one-at-a-time evaluations).  KB is the
// instantiation's kg_line_batch.

// LINE round (SquareExponential) over the training rows, added to S[k] and pmax_hi as eval_line computes them.  The
// lanes' operands come from their unscaled state: base point xr, gradient gr (x~ = xr / l, a_min g~ = a_min (gr / l)),
// with hq = -|x~|^2 / 2 and xga = -a_min x~ . g~.  Unlike tile_posterior, the halves sweep the rows one after the other:
// one sweep for both (twice the 16 trial sums and the fragments live) measured slower on the H100, by 1.8 % per bench
// step even with the lane state parked in shared memory to keep it from spilling (DESIGN.md K6).
template <int DIM, int QP, int KB, bool BIG>
__device__ __forceinline__ void tile_line(const double* __restrict__ Xt, const double* __restrict__ Pk, int N,
                                          const double (&xr)[DIM], const double (&gr)[DIM], const double* inv_len,
                                          double alpha_min, const double (&c)[QP], double hq, double xga,
                                          double (&S)[KB], int& pmax_hi) {
  constexpr int KD = (DIM + 3) / 4, KQ = (QP + 3) / 4;
  // BIG: exponents and slopes in kKappa units (e_j staged scaled; x~, a_min and xga scaled here, so p_j and pmax_hi
  // are kKappa a_min p_j); hq enters as exp2k_split's (C, f)
  double hs = hq, f = 1.0;
  if (BIG) exp2k_split(hq, hs, f);
  const double am = BIG ? kKappa * alpha_min : alpha_min, xgs = BIG ? kKappa * xga : xga;
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    double xa[KD][2], gf[KD][2], ca[KQ][2];
    double hq0, hq1, xg0, xg1, am0, am1;
    tile_rows(hs, h, hq0, hq1);
    tile_rows(xgs, h, xg0, xg1);
    tile_rows(am, h, am0, am1);
    tile_frag<DIM, false, BIG>(xr, inv_len, h, xa, kKappa, kKappa);
    tile_frag<DIM, false, true>(gr, inv_len, h, gf, am0, am1);
    tile_frag<QP, true>(c, nullptr, h, ca);
    double Sp[2][KB];
#pragma unroll
    for (int k = 0; k < KB; ++k) Sp[0][k] = Sp[1][k] = 0.0;
    int pm[2] = {0, 0};
    auto block = [&](int j0, auto tail) {
      constexpr bool TAIL = decltype(tail)::value;
      const TileRows<QP, TAIL> r(Pk, N, j0);
      double dot[4] = {r.h0.x, r.h1.x, r.h0.x, r.h1.x};
      double p[4] = {xg0, xg0, xg1, xg1};
      double a[4] = {r.h0.y, r.h1.y, r.h0.y, r.h1.y};
      double bx[KD], bq[KQ];
      tile_bfrag<DIM>(Xt + r.jb * DIM, bx);
      tile_bfrag<QP>(Pk + r.jb * (QP + 2) + 2, bq);
      tile_mma<DIM>(dot, xa, bx);
      tile_mma<DIM>(p, gf, bx);
      tile_mma<QP>(a, ca, bq);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const bool v = (i & 1) ? r.v1 : r.v0;
        const double pj = v ? p[i] : 0.0;
        pm[i >> 1] = max(pm[i >> 1], __double2hiint(pj) & 0x7fffffff);
        const double w = (v ? a[i] : 0.0) * exp_row<BIG>(dot[i], (i < 2) ? hq0 : hq1);
        double G = BIG ? exp2k_shifted(pj, kExp2kShift) : exp_tab(pj);
#pragma unroll
        for (int k = KB - 1; k >= 0; --k) {
          Sp[i >> 1][k] = fma(w, G, Sp[i >> 1][k]);
          if (k > 0) G *= G;
        }
      }
    };
    const int nfull = N & ~7;
#pragma unroll 1
    for (int j0 = 0; j0 < nfull; j0 += 8) block(j0, std::false_type());
    if (nfull < N) block(nfull, std::true_type());
    if (BIG) {
      // the owner's factor exp2k_split left out of its w's, applied before the sums join the union rows' (natural)
#pragma unroll
      for (int k = 0; k < KB; ++k) S[k] = fma(f, tile_to_owner(quad_sum(Sp[0][k]), quad_sum(Sp[1][k]), h, 0.0), S[k]);
    } else {
#pragma unroll
      for (int k = 0; k < KB; ++k) S[k] = tile_to_owner<true>(quad_sum(Sp[0][k]), quad_sum(Sp[1][k]), h, S[k]);
    }
#pragma unroll
    for (int m = 1; m < 4; m <<= 1) {
      pm[0] = max(pm[0], __shfl_xor_sync(0xffffffffu, pm[0], m));
      pm[1] = max(pm[1], __shfl_xor_sync(0xffffffffu, pm[1], m));
    }
    const int lane = threadIdx.x & 31, src = 4 * (lane & 7);
    const int vl = __shfl_sync(0xffffffffu, pm[0], src), vh = __shfl_sync(0xffffffffu, pm[1], src);
    if ((lane >> 4) == h) pmax_hi = max(pmax_hi, (lane & 8) ? vh : vl);
  }
}

template <int DIM, int QP, int KB, bool SMEM, bool TILE = false, bool BIG = false>
__device__ __forceinline__ void eval_line(const double* __restrict__ Xt, const double* __restrict__ Pk,
                                          const double* __restrict__ Xu, int N, int U, const double (&xb)[DIM],
                                          const double (&gt)[DIM], const double (&c)[QP], double alpha_min,
                                          double (&S)[KB], int& pmax_hi, const double (&xr)[DIM],
                                          const double (&gr)[DIM], const double* inv_len) {
  double nq = 0.0, xg = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) {
    nq = fma(xb[d], xb[d], nq);
    xg = fma(xb[d], gt[d], xg);
  }
  const double hq = -0.5 * nq;
  double ga[DIM];  // a_min g~ : p_j is only ever used scaled by a_min
#pragma unroll
  for (int d = 0; d < DIM; ++d) ga[d] = alpha_min * gt[d];
  const double xga = -alpha_min * xg;
#pragma unroll
  for (int k = 0; k < KB; ++k) S[k] = 0.0;
  pmax_hi = 0;  // max over rows of the high word of |a_min p_j| (integer ALU; monotone in |p|, NaN/inf sort last)
  // one row: scaled coordinates xv, exponent term e, weight weight()
  auto row = [&](const double (&xv)[DIM], double e, auto weight) {
    double dot = 0.0, pj = xga;
#pragma unroll
    for (int d = 0; d < DIM; ++d) {
      dot = fma(xb[d], xv[d], dot);
      pj = fma(ga[d], xv[d], pj);
    }
    // BIG: pmax_hi is kept in the tile rows' kKappa units (BIG implies TILE, so only union rows come here)
    const double a = weight();
    pmax_hi = max(pmax_hi, __double2hiint(BIG ? kKappa * pj : pj) & 0x7fffffff);
    const double w = a * exp_sel<SMEM>(dot + (e + hq));
    double G = exp_sel<SMEM>(pj);
#pragma unroll
    for (int k = KB - 1; k >= 0; --k) {
      S[k] = fma(w, G, S[k]);
      if (k > 0) G *= G;
    }
  };
#pragma unroll 2
  for (int j = 0; j < (TILE ? 0 : N); ++j) {
    const double* xj = Xt + j * DIM;
    const double* pk = Pk + j * (QP + 2);
    double xv[DIM];
    load_row<DIM, SMEM>(xj, xv);
    const double2 h = ld2<SMEM>(pk);  // (e_j, beta_j)
    row(xv, h.x, [&] { return weight_row<QP, SMEM>(pk, h.y, c); });
  }
  for (int u = 0; u < U; ++u) {
    const double* xu = Xu + u * (DIM + 2);
    double xv[DIM];
    load_row<DIM, SMEM>(xu, xv);
    row(xv, ld2<SMEM>(xu + DIM).x, [&] { return union_coef<QP>(c, u); });
  }
  // tile path: the training rows last, so that the scaled operands above are dead during the row loop
  if (TILE) tile_line<DIM, QP, KB, BIG>(Xt, Pk, N, xr, gr, inv_len, alpha_min, c, hq, xga, S, pmax_hi);
}

// Batched backtracking for the Matern-5/2 kernel.  No factorisation along the line here, but the trial points
// x + a_k g share everything that depends on the training point only: with r0^2 = |x~ - X~_j|^2 and
// p_j = g~ . (X~_j - x~),   |x~ + a g~ - X~_j|^2 = r0^2 - 2 a p_j + a^2 |g~|^2 ,
// so the operand loads, the two dot products and the Q weight FMAs are paid once per step and each trial costs one
// sqrt, one exp and a handful of FMAs, value only (a one-at-a-time trial also accumulates the DIM gradient sums it
// almost never uses).  S[k] <-> a_k = a0 2^-k, k < KB.
#ifndef CMOE_LINE_BATCH_M
#define CMOE_LINE_BATCH_M 6
#endif
constexpr int kLineBatchM = CMOE_LINE_BATCH_M;
static_assert(kLineBatchM <= kLineBatch, "S is sized for the SquareExponential batch");

template <int DIM, int QP, bool SMEM>
__device__ __forceinline__ void eval_line_matern(const double* __restrict__ Xt, const double* __restrict__ Pk,
                                                 const double* __restrict__ Xu, int N, int U, double alpha,
                                                 const double (&xb)[DIM], const double (&gt)[DIM],
                                                 const double (&c)[QP], double a0, double (&S)[kLineBatch]) {
  constexpr int KB = kLineBatchM;
  double nq = 0.0, xg = 0.0, gg = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) {
    nq = fma(xb[d], xb[d], nq);
    xg = fma(xb[d], gt[d], xg);
    gg = fma(gt[d], gt[d], gg);
  }
  const double hq = -0.5 * nq;
  double m2a[KB], aag[KB];
  {
    double ak = a0;
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      m2a[k] = -2.0 * ak;
      aag[k] = ak * ak * gg;
      ak *= 0.5;
      S[k] = 0.0;
    }
  }
  // one row: scaled coordinates xv, |X~|^2 term e, weight weight()
  auto row = [&](const double (&xv)[DIM], double e, auto weight) {
    const double dot = dot_dim<DIM>(xb, xv, 0.0);
    const double pj = dot_dim<DIM>(gt, xv, -xg);
    const double a = weight();
    const double r2b = fmax(0.0, e - 2.0 * (hq + dot)), w = a * alpha;
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      // clamped away from 0 for the seed (Matern-5/2 is flat at r = 0: the value is unchanged to the last bit) and,
      // on the table-exp path, from above so that the argument stays inside the table exp's range contract
      const double r2 = fmax(1.0e-280, fma(m2a[k], pj, r2b) + aag[k]);
      double sr, rsr;  // sqrt_rsqrt (device_math.cuh); the unused 1/sqrt(r2) is dead code
      sqrt_rsqrt(r2, sr, rsr);
      double ar = kSqrt5 * sr;
      if (SMEM) ar = fmin(ar, 1.0e6);
      const double we = w * exp_sel<SMEM>(-ar);
      S[k] = fma(we, fma(5.0 / 3.0, r2, 1.0 + ar), S[k]);
    }
  };
#pragma unroll 1
  for (int j = 0; j < N; ++j) {
    const double* xj = Xt + j * DIM;
    const double* pk = Pk + j * (QP + 2);
    double xv[DIM];
    load_row<DIM, SMEM>(xj, xv);
    const double2 h = ld2<SMEM>(pk);  // (|X~_j|^2, beta_j)
    row(xv, h.x, [&] { return weight_row<QP, SMEM>(pk, h.y, c); });
  }
  for (int u = 0; u < U; ++u) {
    const double* xu = Xu + u * (DIM + 2);
    double xv[DIM];
    load_row<DIM, SMEM>(xu, xv);
    row(xv, ld2<SMEM>(xu + DIM).x, [&] { return union_coef<QP>(c, u); });
  }
}

// Kernel pieces for the general path: kv = k(x, X_j) (value row), kb = factor of the first-derivative rows,
// kc = factor of d kb / d x  (SE: all three equal k; Matern-5/2: cov0, first_derivative_part, alpha_exp_part of
// gpp_covariance.cpp:353-355).
template <int KERNEL>
__device__ __forceinline__ void kernel_triple(double dot, double pk0, double hq, double alpha, double& kv, double& kb,
                                              double& kc) {
  if (KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL) {
    kv = exp_fast(dot + (pk0 + hq));
    kb = kv;
    kc = kv;
  } else {
    const double r2 = fmax(0.0, pk0 - 2.0 * (hq + dot));
    const double ar = kSqrt5 * sqrt(r2);
    const double ee = alpha * exp_fast(-ar);
    kv = ee * (1.0 + ar + (5.0 / 3.0) * r2);
    kb = (5.0 / 3.0) * ee * (1.0 + ar);
    kc = (25.0 / 3.0) * ee;
  }
}

constexpr int kMaxG = 8;
// points per trip of the general path's row loops: the loop body is one long dependent chain per point (weight loads
// from L2/HBM, dot, exp), so independent points are interleaved to cover the latencies
#ifndef CMOE_GEN_UNROLL
#define CMOE_GEN_UNROLL 4
#endif
constexpr int kGenUnroll = CMOE_GEN_UNROLL;

// Weight stream of the general path.  Each lane re-reads its weight column (N(1+g) doubles, global memory) on every
// evaluation; a plain load loop leaves the warp waiting on L2/HBM for most of its time (ncu: 74 % of the issue
// slots stalled on the long scoreboard with 8 warps per SM).  The column is therefore pulled through a per-lane ring in
// shared memory with LDGSTS (cp.async, 8 bytes per lane = 256 bytes per warp and row), kRingDepth stages of `P` points
// deep, and the arithmetic reads the ring.  Every lane copies and reads only its own slots, so cp.async.wait_group is
// the only synchronisation.  body(j, w): w[m * kMcThreads] is weight m of point j.
constexpr int kRingRows = 80;   // ring slots per lane (rows of the weight column)
constexpr int kRingDepth = 8;   // stages in flight
template <typename F>
__device__ __forceinline__ void stream_point_weights(const double* aw, double* ring, int N, int b1, F&& body) {
  constexpr int T = kMcThreads;
  const int P = max(1, kRingRows / (kRingDepth * b1));  // points per stage
  const int SR = P * b1, R = N * b1;
  const int nst = (N + P - 1) / P;
  auto issue = [&](int st) {
    if (st < nst) {
      const int r0 = st * SR;
      const int cnt = min(SR, R - r0);
      double* dst = ring + (st & (kRingDepth - 1)) * SR * T;
      const double* src = aw + static_cast<size_t>(r0) * T;
      for (int k = 0; k < cnt; ++k) cp_async8(dst + k * T, src + static_cast<size_t>(k) * T, true);
    }
    cp_async_commit();
  };
  for (int st = 0; st < kRingDepth - 1; ++st) issue(st);
  for (int st = 0; st < nst; ++st) {
    issue(st + kRingDepth - 1);  // refills the slot consumed in the previous trip
    cp_async_wait<kRingDepth - 1>();
    const double* w = ring + (st & (kRingDepth - 1)) * SR * T;
    const int j1 = min(N, (st + 1) * P);
#pragma unroll 2
    for (int j = st * P; j < j1; ++j, w += b1 * T) body(j, w, 0);
  }
  cp_async_wait<0>();
}

// Wide variant (g > 8, up to 32 rows per point): eight stages of whole points no longer fit the kRingRows slots, so the
// same ring is filled in stages of kWideStageRows rows, not tied to point boundaries; row r of the column lives in slot
// r % kRingRows, and a point's rows may wrap around the end of the ring.  kWideLookahead stages are in flight; after
// stage st has landed, every point whose last row it holds is evaluated, then stage st + kWideLookahead is issued into
// the slots of stage st + kWideLookahead - kWideStages.  No point evaluated later starts in those slots: its first row
// is past (st + 1) kWideStageRows - 32 (static_assert below).  body(j, ring, base): weight m of point j is in slot
// (base + m) % kRingRows (ring_weight).
constexpr int kWideStageRows = 8;
constexpr int kWideStages = kRingRows / kWideStageRows;
constexpr int kWideLookahead = 6;
constexpr int kMaxGWide = 31;  // 1 + g <= 32 rows per point (Q = U (1 + g) <= 32)
static_assert(kWideStages * kWideStageRows == kRingRows, "the wide stages tile the ring");
static_assert((kWideStages - kWideLookahead) * kWideStageRows >= kMaxGWide, "a refill never overwrites a live point");
template <typename F>
__device__ __forceinline__ void stream_point_weights_wide(const double* aw, double* ring, int N, int b1, F&& body) {
  constexpr int T = kMcThreads, SR = kWideStageRows, L = kWideLookahead;
  const int R = N * b1;
  const int nst = (R + SR - 1) / SR;
  auto issue = [&](int st) {
    if (st < nst) {
      const int r0 = st * SR;
      const int cnt = min(SR, R - r0);
      double* dst = ring + (st % kWideStages) * SR * T;
      const double* src = aw + static_cast<size_t>(r0) * T;
      for (int k = 0; k < cnt; ++k) cp_async8(dst + k * T, src + static_cast<size_t>(k) * T, true);
    }
    cp_async_commit();
  };
  for (int st = 0; st < L; ++st) issue(st);
  int j = 0, base = 0;
  for (int st = 0; st < nst; ++st) {
    cp_async_wait<L - 1>();
    const int ready = min(R, (st + 1) * SR);
    for (; (j + 1) * b1 <= ready; ++j) {
      body(j, ring, base);
      base += b1;
      if (base >= kRingRows) base -= kRingRows;
    }
    issue(st + L);  // after the evaluations above: it refills slots they may have read
  }
  cp_async_wait<0>();
}

// weight m of a point: narrow ring w = the point's first slot (contiguous rows); wide ring w = the ring, rows from base
template <bool WIDE>
__device__ __forceinline__ double ring_weight(const double* w, int base, int m) {
  if (!WIDE) return w[m * kMcThreads];
  int k = base + m;
  if (k >= kRingRows) k -= kRingRows;
  return w[k * kMcThreads];
}

template <bool WIDE, typename F>
__device__ __forceinline__ void stream_weights(const double* aw, double* ring, int N, int b1, F&& body) {
  if constexpr (WIDE) {
    stream_point_weights_wide(aw, ring, N, b1, body);
  } else {
    stream_point_weights(aw, ring, N, b1, body);
  }
}

// General evaluation with derivative observations (d-KG): every training point owns 1+g rows
//   K((j,0), x) = kv ,  K((j,m), x) = kb (x~_t - X~_jt) / l_t   (t = derivs[m-1]; the 1/l_t is folded into the pack)
//   mu+(x) - m = sum_j [ a_j0 kv + kb sum_m a~_jm (x~_t - X~_jt) ]  with  a_(j,m) = beta_(j,m) - B_(j,m),: . c
//   d/dx~_d   = (X~_jd - x~_d) (a_j0 kb + kc wsum) + kb a~_jm [d == t]
// The weights a_(j,m) come from this lane's ring slots (aj), the point operands from shared memory when they were
// parked there (XS) and through the read-only path otherwise.
// WIDE (g > 8): the derivative rows are visited in coordinate order d (row prm.drow[d]), so the query coordinate and the
// point's coordinate of row m are xq[d] and xv[d] with compile-time d and no per-row register arrays are needed; the
// kb a~_jm terms go straight into s[d] instead of em.
template <int KERNEL, int DIM, int QP, bool XS, bool WIDE = false>
__device__ __forceinline__ void eval_posterior_gen(const KgMcParams& prm, const double* __restrict__ Xt,
                                                   const double* __restrict__ Pk, const double* __restrict__ Xu,
                                                   const double (&xq)[DIM], const double* aw, double* ring,
                                                   const double* __restrict__ cl, double& S0, double& SB,
                                                   double (&s)[DIM], double (&em)[kMaxG]) {
  const int N = prm.N, U = prm.U, g = prm.g, stride = prm.pk_stride;
  double nq = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) nq = fma(xq[d], xq[d], nq);
  const double hq = -0.5 * nq;
  // query coordinates at the derivative indices (compile-time register indexing only)
  double xm[kMaxG];
  if (!WIDE) {
#pragma unroll
    for (int m = 0; m < kMaxG; ++m) {
      xm[m] = 0.0;
      em[m] = 0.0;
      if (m < g) {
#pragma unroll
        for (int d = 0; d < DIM; ++d)
          if (d == prm.derivs[m]) xm[m] = xq[d];
      }
    }
  }
  S0 = 0.0;
  SB = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) s[d] = 0.0;
  stream_weights<WIDE>(aw, ring, N, 1 + g, [&](int j, const double* aj, int base) {
    const double* xj = Xt + static_cast<size_t>(j) * DIM;
    const double* pk = Pk + static_cast<size_t>(j) * stride;
    double xv[DIM];
    load_row<DIM, XS>(xj, xv);
    double dot = 0.0;
#pragma unroll
    for (int d = 0; d < DIM; ++d) dot = fma(xq[d], xv[d], dot);
    double kv, kb, kc;
    kernel_triple<KERNEL>(dot, ld1<XS>(pk), hq, prm.alpha, kv, kb, kc);
    const double a0 = ring_weight<WIDE>(aj, base, 0);  // this lane's weights of point j (ring slots)
    double wsum = 0.0;
    if (WIDE) {
#pragma unroll
      for (int d = 0; d < DIM; ++d) {
        const int r = prm.drow[d];
        if (r > 0) {
          const double am = ring_weight<WIDE>(aj, base, r);
          wsum = fma(am, xq[d] - xv[d], wsum);
          s[d] = fma(kb, am, s[d]);
        }
      }
    } else {
#pragma unroll
      for (int m = 0; m < kMaxG; ++m) {
        if (m < g) {
          const double am = aj[(m + 1) * kMcThreads];
          wsum = fma(am, xm[m] - ld1<XS>(xj + prm.derivs[m]), wsum);
          em[m] = fma(kb, am, em[m]);
        }
      }
    }
    S0 = fma(a0, kv, S0);
    S0 = fma(kb, wsum, S0);
    const double wb = fma(kc, wsum, a0 * kb);
    SB += wb;
#pragma unroll
    for (int d = 0; d < DIM; ++d) s[d] = fma(wb, xv[d], s[d]);
  });
  const int bs = 1 + g;
  for (int u = 0; u < U; ++u) {
    const double* xu = Xu + static_cast<size_t>(u) * (DIM + 2);
    double xv[DIM];
    load_row<DIM, false>(xu, xv);
    double dot = 0.0;
#pragma unroll
    for (int d = 0; d < DIM; ++d) dot = fma(xq[d], xv[d], dot);
    double kv, kb, kc;
    kernel_triple<KERNEL>(dot, __ldg(xu + DIM), hq, prm.alpha, kv, kb, kc);
    const double a0 = cl[u * bs];
    double wsum = 0.0;
    if (WIDE) {
#pragma unroll
      for (int d = 0; d < DIM; ++d) {
        const int r = prm.drow[d];
        if (r > 0) {
          const double am = cl[u * bs + r] * prm.inv_len[d];
          wsum = fma(am, xq[d] - xv[d], wsum);
          s[d] = fma(kb, am, s[d]);
        }
      }
    } else {
#pragma unroll
      for (int m = 0; m < kMaxG; ++m) {
        if (m < g) {
          const double am = cl[u * bs + 1 + m] * prm.inv_len[prm.derivs[m]];
          wsum = fma(am, xm[m] - __ldg(xu + prm.derivs[m]), wsum);
          em[m] = fma(kb, am, em[m]);
        }
      }
    }
    S0 = fma(a0, kv, S0);
    S0 = fma(kb, wsum, S0);
    const double wb = fma(kc, wsum, a0 * kb);
    SB += wb;
#pragma unroll
    for (int d = 0; d < DIM; ++d) s[d] = fma(wb, xv[d], s[d]);
  }
}

// Batched backtracking with derivative observations (SquareExponential): along x + a g the value rows scale as in
// eval_line and the derivative rows' factor (x~_t - X~_jt) is linear in a, so with
//     u_j = sum_m a~_jm (x~_t - X~_jt),  v_j = sum_m a~_jm g~_t,  k0_j = k(x, X_j),  G_jk = exp(a_k p_j)
// the trial values are  E_k [ sum_j k0_j G_jk (a_j0 + u_j) + a_k sum_j k0_j G_jk v_j ]:  S[k] and T[k] below.
// The (1+g) Q weight FMAs per point — the dominant cost of this path — are paid once per step instead of once per trial.
// WIDE: the derivative rows in coordinate order, as in eval_posterior_gen.
template <int DIM, int QP, bool XS, bool WIDE = false>
__device__ __forceinline__ void eval_line_gen(const KgMcParams& prm, const double* __restrict__ Xt,
                                              const double* __restrict__ Pk, const double* __restrict__ Xu,
                                              const double (&xb)[DIM], const double (&gt)[DIM], const double* aw,
                                              double* ring, const double* __restrict__ cl, double alpha_min,
                                              double (&S)[kLineBatch], double (&T)[kLineBatch], int& pmax_hi) {
  const int N = prm.N, U = prm.U, g = prm.g, stride = prm.pk_stride;
  double nq = 0.0, xg = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) {
    nq = fma(xb[d], xb[d], nq);
    xg = fma(xb[d], gt[d], xg);
  }
  const double hq = -0.5 * nq;
  double ga[DIM];
#pragma unroll
  for (int d = 0; d < DIM; ++d) ga[d] = alpha_min * gt[d];
  const double xga = -alpha_min * xg;
  // base coordinates and direction at the derivative indices (compile-time register indexing only)
  double xm[kMaxG], gm[kMaxG];
  if (!WIDE) {
#pragma unroll
    for (int m = 0; m < kMaxG; ++m) {
      xm[m] = 0.0;
      gm[m] = 0.0;
      if (m < g) {
#pragma unroll
        for (int d = 0; d < DIM; ++d)
          if (d == prm.derivs[m]) {
            xm[m] = xb[d];
            gm[m] = gt[d];
          }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kLineBatch; ++k) S[k] = T[k] = 0.0;
  pmax_hi = 0;
  stream_weights<WIDE>(aw, ring, N, 1 + g, [&](int j, const double* aj, int base) {
    const double* xj = Xt + static_cast<size_t>(j) * DIM;
    const double* pk = Pk + static_cast<size_t>(j) * stride;
    double xv[DIM];
    load_row<DIM, XS>(xj, xv);
    double dot = 0.0, pj = xga;
#pragma unroll
    for (int d = 0; d < DIM; ++d) {
      dot = fma(xb[d], xv[d], dot);
      pj = fma(ga[d], xv[d], pj);
    }
    const double a0 = ring_weight<WIDE>(aj, base, 0);
    double us = 0.0, vs = 0.0;
    if (WIDE) {
#pragma unroll
      for (int d = 0; d < DIM; ++d) {
        const int r = prm.drow[d];
        if (r > 0) {
          const double am = ring_weight<WIDE>(aj, base, r);
          us = fma(am, xb[d] - xv[d], us);
          vs = fma(am, gt[d], vs);
        }
      }
    } else {
#pragma unroll
      for (int m = 0; m < kMaxG; ++m) {
        if (m < g) {
          const double am = aj[(m + 1) * kMcThreads];
          us = fma(am, xm[m] - ld1<XS>(xj + prm.derivs[m]), us);
          vs = fma(am, gm[m], vs);
        }
      }
    }
    pmax_hi = max(pmax_hi, __double2hiint(pj) & 0x7fffffff);
    const double k0 = exp_fast(dot + (ld1<XS>(pk) + hq));
    const double w = k0 * (a0 + us), wv = k0 * vs;
    double G = exp_fast(pj);
#pragma unroll
    for (int k = kLineBatch - 1; k >= 0; --k) {
      S[k] = fma(w, G, S[k]);
      T[k] = fma(wv, G, T[k]);
      if (k > 0) G *= G;
    }
  });
  const int bs = 1 + g;
  for (int u = 0; u < U; ++u) {
    const double* xu = Xu + static_cast<size_t>(u) * (DIM + 2);
    double xv[DIM];
    load_row<DIM, false>(xu, xv);
    double dot = 0.0, pj = xga;
#pragma unroll
    for (int d = 0; d < DIM; ++d) {
      dot = fma(xb[d], xv[d], dot);
      pj = fma(ga[d], xv[d], pj);
    }
    const double a0 = cl[u * bs];
    double us = 0.0, vs = 0.0;
    if (WIDE) {
#pragma unroll
      for (int d = 0; d < DIM; ++d) {
        const int r = prm.drow[d];
        if (r > 0) {
          const double am = cl[u * bs + r] * prm.inv_len[d];
          us = fma(am, xb[d] - xv[d], us);
          vs = fma(am, gt[d], vs);
        }
      }
    } else {
#pragma unroll
      for (int m = 0; m < kMaxG; ++m) {
        if (m < g) {
          const double am = cl[u * bs + 1 + m] * prm.inv_len[prm.derivs[m]];
          us = fma(am, xm[m] - __ldg(xu + prm.derivs[m]), us);
          vs = fma(am, gm[m], vs);
        }
      }
    }
    pmax_hi = max(pmax_hi, __double2hiint(pj) & 0x7fffffff);
    const double k0 = exp_fast(dot + (__ldg(xu + DIM) + hq));
    const double w = k0 * (a0 + us), wv = k0 * vs;
    double G = exp_fast(pj);
#pragma unroll
    for (int k = kLineBatch - 1; k >= 0; --k) {
      S[k] = fma(w, G, S[k]);
      T[k] = fma(wv, G, T[k]);
      if (k > 0) G *= G;
    }
  }
}


// General path: the weights a = beta~ - B~ c depend on the sample only, not on the query point, so they are formed once
// when a lane takes a new sample and parked in that lane's column of the CTA's scratch (global memory, streamed back
// with L2-only loads by every evaluation of the sample: (1+g) loads per training point instead of (1+g)(Q+1) loads
// and (1+g) Q FMAs).  The warp fills the column of each requesting lane together, rows strided over the lanes, so the
// table reads are coalesced; the FMA order per row (beta first, then u ascending) is the one the per-evaluation code had.
template <int QP>
__device__ __forceinline__ void fill_sample_weights(const double* __restrict__ Wt, int R,
                                                    const double* __restrict__ recC, double* aw_warp, unsigned want,
                                                    int sample, int lane) {
  while (want) {
    const int b = __ffs(want) - 1;
    want &= want - 1;
    const int sb = __shfl_sync(0xffffffffu, sample, b);
    double cb[QP];
#pragma unroll
    for (int u = 0; u < QP; ++u) cb[u] = __ldg(recC + static_cast<size_t>(sb) * QP + u);
    double* col = aw_warp + b;
#pragma unroll 4
    for (int r = lane; r < R; r += 32) {
      double a = __ldg(Wt + r);
#pragma unroll
      for (int u = 0; u < QP; ++u) a = fma(-__ldg(Wt + static_cast<size_t>(1 + u) * R + r), cb[u], a);
      col[static_cast<size_t>(r) * kMcThreads] = a;
    }
  }
  __syncwarp();
}

// The same column formed by its own lane (table loads are warp-uniform).  Costs R Q FMAs per lane however many lanes
// take part, so it is used when at least kOwnFillLanes do; a lone lane is served by the whole warp instead.
constexpr int kOwnFillLanes = 6;
template <int QP>
__device__ __forceinline__ void fill_own_weights(const double* __restrict__ Wt, int R, const double (&c)[QP],
                                                 double* aw) {
#pragma unroll 4
  for (int r = 0; r < R; ++r) {
    double a = __ldg(Wt + r);
#pragma unroll
    for (int u = 0; u < QP; ++u) a = fma(-__ldg(Wt + static_cast<size_t>(1 + u) * R + r), c[u], a);
    aw[static_cast<size_t>(r) * kMcThreads] = a;
  }
}

// Large-union build (PRE): the sample's whole weight column is precomputed (kg_large.cu, [num_mc][R] per candidate), so
// the warp copies the column of each requesting lane into that lane's scratch column, rows strided over the lanes so
// that the reads are coalesced.
__device__ __forceinline__ void copy_sample_weights(const double* __restrict__ Wt, int R, double* aw_warp, unsigned want,
                                                    int sample, int lane) {
  while (want) {
    const int b = __ffs(want) - 1;
    want &= want - 1;
    const int sb = __shfl_sync(0xffffffffu, sample, b);
    const double* src = Wt + static_cast<size_t>(sb) * R;
    double* col = aw_warp + b;
#pragma unroll 4
    for (int r = lane; r < R; r += 32) col[static_cast<size_t>(r) * kMcThreads] = __ldg(src + r);
  }
  __syncwarp();
}

// Value and gradient of mu+ at a sample's start point, from the start-point table instead of a POINT round (g == 0).
// mu+ - m and the POINT round's sums S0, SB, s_d are affine in c, so kg_start_kernel tabulates, per discretisation
// point, row 0 (the beta part) and rows 1+u (the union point u's part: k(a, Xu_u) - sum_j B_ju k(a, X_j)), columns
// (S0, SB, s_0 .. s_DIM-1); a sample combines them with its c in ascending u.  xb is the (unscaled) start point; returns
// f = -mu+ and the gradient the INIT transition forms.
template <int DIM, int QP>
__device__ __forceinline__ void start_from_table(const KgMcParams& prm, const double* __restrict__ row,
                                                 const double (&c)[QP], const double (&xb)[DIM], double& fb,
                                                 double (&gb)[DIM]) {
  constexpr int W = DIM + 2;
  // one pair of columns at a time (S0 and SB first), so that only two sums are live next to the lane's state
  auto pair = [&](int k) {
    double2 t = __ldg(reinterpret_cast<const double2*>(row + k));
#pragma unroll
    for (int u = 0; u < QP; ++u) {
      const double2 v = __ldg(reinterpret_cast<const double2*>(row + (1 + u) * W + k));
      t.x = fma(c[u], v.x, t.x);
      t.y = fma(c[u], v.y, t.y);
    }
    return t;
  };
  const double2 t0 = pair(0);  // (S0, SB)
  fb = -(prm.mean + t0.x);
#pragma unroll
  for (int d = 0; d < DIM; d += 2) {
    const double2 s = pair(2 + d);
    gb[d] = (d < prm.ps) ? -prm.inv_len[d] * (s.x - (xb[d] * prm.inv_len[d]) * t0.y) : 0.0;
    gb[d + 1] = (d + 1 < prm.ps) ? -prm.inv_len[d + 1] * (s.y - (xb[d + 1] * prm.inv_len[d + 1]) * t0.y) : 0.0;
  }
}

enum : int { ST_FETCH = 0, ST_INIT = 1, ST_TRIAL = 2, ST_LIMIT = 3, ST_DONE = 4, ST_LINE = 5 };

#ifdef CMOE_KG_TRIAL_HIST
// Probe build only (profiles/build_variants.sh, read by profiles/kg_trial_hist_probe.py; one translation unit per
// library): how the LINE batches of kg_mc_body end.  Bins [step][index] count accepted trials by the inner step index
// (capped) and the trial index counted from a_0 (search + k); then batches run, batches with no passing trial, range
// fallbacks to ST_TRIAL, warp rounds, warp rounds whose vote left lanes idle, and idle lanes summed over those rounds.
constexpr int kHistSteps = 16, kHistTrials = 32;
enum : int {
  H_BATCHES = kHistSteps * kHistTrials, H_ALL_FAIL, H_RANGE, H_ROUNDS, H_IDLE_ROUNDS, H_IDLE_LANES, kHistSize
};
__device__ unsigned long long kg_trial_hist[kHistSize];
__device__ __forceinline__ void hist_add(int i, unsigned v = 1) { atomicAdd(kg_trial_hist + i, v); }
}  // namespace cmoe
// copies the kHistSize counters to out and, with reset != 0, zeroes them; returns a cudaError_t
extern "C" int cmoe_kg_trial_hist(unsigned long long* out, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out, cmoe::kg_trial_hist, sizeof(cmoe::kg_trial_hist));
  if (e == cudaSuccess && reset) {
    static const unsigned long long zero[cmoe::kHistSize] = {};
    e = cudaMemcpyToSymbol(cmoe::kg_trial_hist, zero, sizeof(zero));
  }
  return static_cast<int>(e);
}
namespace cmoe {
#endif


// The per-lane line-search state machine.  Live across evaluations: c, the base point xb with f and grad f there,
// the step size and a few counters; the start point of the current restart run is parked in the sample's output slot.
//
// A round of the warp is either a POINT round (mu+ and its gradient at one query point per lane: INIT / TRIAL / LIMIT
// lanes) or, for the SquareExponential fast path, a LINE round (all backtracking trials of a step at once, eval_line).
// Which one runs is a warp vote; lanes waiting for the other kind idle for that round and are in phase again after it
// (a sample alternates LINE, POINT, LINE, ... so the vote keeps a warp in lock-step once it is).  Without derivative
// observations a sample's start evaluation comes from the start-point table (start_from_table) when the lane takes the
// sample, so a new sample's first round is a LINE round, in phase with the lanes that continue; only the general path
// (GEN) spends a POINT round on it (ST_INIT).
// PRE (GEN only): the large-union build of kg_mc_large_kernel; Wt holds the precomputed weight columns of the
// candidate's samples (copy_sample_weights) and c is not read.
template <int KERNEL, int DIM, int QP, bool SMEM, bool GEN, bool WIDE = false, bool BIG = false, bool PRE = false>
__device__ __forceinline__ void kg_mc_body(const KgMcParams& prm, const double* __restrict__ Xt,
                                           const double* __restrict__ Pk, const double* __restrict__ Xu, int cand,
                                           int s_begin, int s_end, int* next_sample, double* aw = nullptr,
                                           const double* __restrict__ Wt = nullptr, double* ring = nullptr) {
  constexpr bool SE = (KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL);
  constexpr bool LINE = SE || !GEN;  // Matern-5/2 batches its trials too (eval_line_matern) unless derivative rows exist
  constexpr int KB = !SE ? kLineBatchM : GEN ? kLineBatch : kg_line_batch<KERNEL, DIM, QP>();  // trials per LINE round
  constexpr int ST_SEARCH = LINE ? ST_LINE : ST_TRIAL;  // how a step's backtracking starts
  constexpr bool TILE = SMEM && !GEN && kg_tile_path<KERNEL, DIM, QP>();  // DMMA tiles for the training rows
  const int N = prm.N, U = prm.U;
  const double* A = prm.A + static_cast<size_t>(cand) * prm.M * DIM;
  const double* recC = prm.recC + static_cast<size_t>(cand) * prm.num_mc * QP;
  const int* recStart = prm.recStart + static_cast<size_t>(cand) * prm.num_mc;
  double* outVal = prm.outVal + static_cast<size_t>(cand) * prm.num_mc;
  double* outX = prm.outX + static_cast<size_t>(cand) * prm.num_mc * DIM;
  double* outH = prm.outH + static_cast<size_t>(cand) * prm.num_mc;

  int state = ST_FETCH;
  int sample = s_begin + threadIdx.x;
  double c[QP], xb[DIM], gb[DIM];
  double cl[GEN ? QP : 1];  // general path: run-time indexable copy of c for the union rows (lives in local memory)
  double fb = 0.0, alpha_n = 0.0, gnorm = 0.0;
  int step_i = 0, restart_i = 0, search = 0;
  unsigned n_evals = 0, n_steps = 0, n_point = 0, n_line = 0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) xb[d] = gb[d] = 0.0;
#pragma unroll
  for (int u = 0; u < QP; ++u) c[u] = 0.0;

  while (true) {
    bool took_sample = false;
    bool finish_run = false;
    if (state == ST_FETCH) {
      if (sample < s_end) {
        if (prm.max_restarts > 0) {
          took_sample = true;
          if constexpr (!PRE) {
#pragma unroll
            for (int u = 0; u < QP; ++u) c[u] = recC[static_cast<size_t>(sample) * QP + u];
            if (GEN) {
#pragma unroll
              for (int u = 0; u < QP; ++u) cl[GEN ? u : 0] = c[u];
            }
          }
          const double* a0 = A + static_cast<size_t>(recStart[sample]) * DIM;
#pragma unroll
          for (int d = 0; d < DIM; ++d) {
            xb[d] = a0[d];
            outX[static_cast<size_t>(sample) * DIM + d] = a0[d];  // start of restart run 0
          }
          step_i = 0;
          restart_i = 0;
          if (GEN) {
            state = ST_INIT;
          } else {
            // the start evaluation from the table, then the INIT transition: the sample's first round is a LINE round
            start_from_table<DIM, QP>(prm,
                                      prm.Start + (static_cast<size_t>(cand) * prm.M + recStart[sample]) *
                                                      (1 + QP) * (DIM + 2),
                                      c, xb, fb, gb);
            n_evals += 1;
            if (prm.max_steps <= 0) {
              finish_run = true;  // the lane stays in ST_FETCH, so it sits out this iteration's round
            } else {
              alpha_n = prm.alpha0[0];
              search = 0;
              gnorm = 0.0;
#pragma unroll
              for (int d = 0; d < DIM; ++d) gnorm = fma(gb[d], gb[d], gnorm);
              state = ST_SEARCH;
            }
          }
        } else {
          // ComputeOptimalPosteriorMean returns without touching its outputs (...optimization.cpp:424-426):
          // best_function_value stays 0 and the best point keeps its fill value 1.0
          outVal[sample] = 0.0;
          double nx = 0.0;
#pragma unroll
          for (int d = 0; d < DIM; ++d) {
            outX[static_cast<size_t>(sample) * DIM + d] = 1.0 * prm.inv_len[d];
            nx = fma(prm.inv_len[d], prm.inv_len[d], nx);
          }
          outH[sample] = -0.5 * nx;
          sample = atomicAdd(next_sample, 1);
        }
      } else {
        state = ST_DONE;
      }
    }
    if (__all_sync(0xffffffffu, state == ST_DONE)) break;
    if (GEN) {
      const unsigned want = __ballot_sync(0xffffffffu, took_sample);
      if constexpr (PRE) {
        if (want) copy_sample_weights(Wt, prm.N * (1 + prm.g), aw - (threadIdx.x & 31), want, sample, threadIdx.x & 31);
      } else if (__popc(want) >= kOwnFillLanes) {
        // many lanes at once (samples with equal round counts keep a warp's lanes in cohorts): every requesting lane
        // forms its own column from warp-uniform (broadcast) table loads; the column stores are full lines
        if (took_sample) fill_own_weights<QP>(Wt, prm.N * (1 + prm.g), c, aw);
        __syncwarp();
      } else if (want) {
        fill_sample_weights<QP>(Wt, prm.N * (1 + prm.g), recC, aw - (threadIdx.x & 31), want, sample,
                                threadIdx.x & 31);
      }
    }

    bool line_round = false;
    if (LINE) {
      const unsigned wl = __ballot_sync(0xffffffffu, state == ST_LINE);
      const unsigned wp = __ballot_sync(0xffffffffu, state == ST_INIT || state == ST_TRIAL || state == ST_LIMIT);
      line_round = __popc(wl) > __popc(wp);
#ifdef CMOE_KG_TRIAL_HIST
      if ((threadIdx.x & 31) == 0 && (wl | wp)) {
        const int idle = __popc(line_round ? wp : wl);
        hist_add(H_ROUNDS);
        if (idle) {
          hist_add(H_IDLE_ROUNDS);
          hist_add(H_IDLE_LANES, idle);
        }
      }
#endif
    }

    if (LINE && line_round) {
      // ---- all backtracking trials of this step in one pass (warp-uniform) ----
      double xt[DIM], gt[DIM], S[SE ? KB : kLineBatch];
      int pmax_hi;
      double gg = 0.0;
#pragma unroll
      for (int d = 0; d < DIM; ++d) {
        xt[d] = xb[d] * prm.inv_len[d];
        gt[d] = gb[d] * prm.inv_len[d];
        gg = fma(gt[d], gt[d], gg);
      }
      double nb2 = 0.0;  // tile path: formed before the evaluation, so that xt is dead during it
      if (TILE) {
#pragma unroll
        for (int d = 0; d < DIM; ++d) nb2 = fma(xt[d], xt[d], nb2);
      }
      constexpr double kTop = static_cast<double>(1 << (KB - 1));
      double T[GEN ? kLineBatch : 1];
      if constexpr (!SE) {
        pmax_hi = 0;  // no factor can leave the double range on this path
        eval_line_matern<DIM, QP, SMEM>(Xt, Pk, Xu, N, U, prm.alpha, xt, gt, c, alpha_n, S);
      } else if constexpr (GEN) {
        eval_line_gen<DIM, QP, SMEM, WIDE>(prm, Xt, Pk, Xu, xt, gt, aw, ring, cl, alpha_n * (1.0 / kTop), S,
                               reinterpret_cast<double (&)[kLineBatch]>(T), pmax_hi);
      } else {
        eval_line<DIM, QP, KB, SMEM, TILE, BIG>(Xt, Pk, Xu, N, U, xt, gt, c, alpha_n * (1.0 / kTop), S, pmax_hi, xb,
                                                 gb, prm.inv_len);
      }
      if (state == ST_LINE) {
        n_line += 1;
        // safe iff a_0 |p_j| = 2^(KB-1) |a_min p_j| < 512 for every row: every factor exp(a_k p_j) stays in range
        // (BIG: pmax_hi in kKappa units, so is the bound; the high word of the bound is at most the bound).  a_min
        // and the bound 512 / kTop are a_0 and 512 scaled by the same power of two, which moves both high words by the
        // same exponent step: the test decides a_0 |p_j| < 512 exactly as conservatively whatever KB is.
        if (!TILE) {
#pragma unroll
          for (int d = 0; d < DIM; ++d) nb2 = fma(xt[d], xt[d], nb2);
        }
#ifdef CMOE_KG_TRIAL_HIST
        hist_add(H_BATCHES);
#endif
        if (pmax_hi >= __double2hiint((BIG ? kKappa : 1.0) * 512.0 / kTop) || !(nb2 <= kFarRadius * kFarRadius)) {
          state = ST_TRIAL;  // factors could leave the double range: this step backtracks one evaluation at a time
#ifdef CMOE_KG_TRIAL_HIST
          hist_add(H_RANGE);
#endif
        } else {
          int kacc = -1;
          double ak = alpha_n, a_acc = alpha_n;
#pragma unroll
          for (int k = 0; k < KB; ++k) {
            const double sk = GEN ? fma(ak, T[GEN ? k : 0], S[k]) : S[k];
            const double fq = SE ? -(prm.mean + exp_fast(-0.5 * ak * ak * gg) * sk) : -(prm.mean + sk);
            // Armijo-type test of the reference: f(x + a g) - f(x) > 0.5 a |g|^2   (gpp_optimization.hpp:758)
            const bool ok = (search + k < 30) && ((fq - fb) > 0.5 * ak * gnorm);
            if (kacc < 0 && ok) {
              kacc = k;
              a_acc = ak;
            }
            ak *= 0.5;
          }
#ifdef CMOE_KG_TRIAL_HIST
          hist_add(kacc < 0 ? H_ALL_FAIL
                            : min(step_i, kHistSteps - 1) * kHistTrials + min(search + kacc, kHistTrials - 1));
#endif
          if (kacc >= 0) {
            n_evals += kacc + 1;
            search += kacc;
            alpha_n = a_acc;
            state = ST_LIMIT;  // value and gradient at the domain-limited point decide the step (:767-781)
          } else {
            n_evals += min(KB, 30 - search);
            search += KB;
            alpha_n *= 1.0 / (2.0 * kTop);
            if (search >= 30) finish_run = true;  // exhausted: reject and stop this run (:778-781)
          }
        }
      }
    } else {
      // ---- query point of this lane: base (INIT), base + alpha*grad (TRIAL), base + limited step (LIMIT) ----
      double xq[DIM];
#pragma unroll
      for (int d = 0; d < DIM; ++d) {
        double st = 0.0;
        if (state == ST_TRIAL || state == ST_LIMIT) st = alpha_n * gb[d];
        if (state == ST_LIMIT) st = (d < prm.ps) ? limit_step(st, xb[d], prm.lo[d], prm.hi[d], prm.mrc) : 0.0;
        xq[d] = (xb[d] + st) * prm.inv_len[d];
      }

      // ---- the expensive, warp-uniform part ----
      double S0, SB, s[DIM];
      double em[kMaxG];
      if (GEN) {
        eval_posterior_gen<KERNEL, DIM, QP, SMEM, WIDE>(prm, Xt, Pk, Xu, xq, aw, ring, cl, S0, SB, s, em);
        // kb a~_jm lands on coordinate derivs[m]: fold it into s so that the common gradient formula below holds
        // (grad_d = inv_len_d (s_d - x~_d SB)), using compile-time register indices only (WIDE: already in s)
        if (!WIDE) {
#pragma unroll
          for (int m = 0; m < kMaxG; ++m)
            if (m < prm.g) {
#pragma unroll
              for (int d = 0; d < DIM; ++d)
                if (d == prm.derivs[m]) s[d] += em[m];
            }
        }
      } else {
        eval_posterior<KERNEL, DIM, QP, SMEM, TILE, BIG>(Xt, Pk, Xu, N, U, prm.alpha, xq, c, S0, SB, s);
      }
      if (state == ST_INIT || state == ST_TRIAL || state == ST_LIMIT) {
        n_evals += 1;
        n_point += 1;
      }
      const double fq = -(prm.mean + S0);

      // ---- per-lane transitions (cheap) ----
      bool accept = false;
      if (state == ST_INIT) {
        fb = fq;
#pragma unroll
        for (int d = 0; d < DIM; ++d) gb[d] = (d < prm.ps) ? -prm.inv_len[d] * (s[d] - xq[d] * SB) : 0.0;
        if (prm.max_steps <= 0) {
          finish_run = true;
        } else {
          step_i = -1;  // becomes 0 in the common "start a step" block below
          accept = true;
        }
      } else if (state == ST_TRIAL) {
        // Armijo-type test of the reference: f(x + a g) - f(x) > 0.5 a |g|^2   (gpp_optimization.hpp:758)
        const bool ok = (fq - fb) > 0.5 * alpha_n * gnorm;
        if (!ok) {
          alpha_n *= 0.5;
          search += 1;
          if (search >= 30) finish_run = true;  // exhausted: reject and stop this run (:778-781)
        } else {
          // limit the accepted step to the domain; if unchanged, this evaluation IS the final evaluation of the step
          bool same = true;
#pragma unroll
          for (int d = 0; d < DIM; ++d) {
            const double raw = alpha_n * gb[d];
            const double lim = (d < prm.ps) ? limit_step(raw, xb[d], prm.lo[d], prm.hi[d], prm.mrc) : 0.0;
            same = same && (lim == raw);
          }
          if (same) {
            if (fq <= fb) {
              finish_run = true;
            } else {
              accept = true;
            }
          } else {
            state = ST_LIMIT;  // one more evaluation at the limited point
          }
        }
      } else if (state == ST_LIMIT) {
        if (fq <= fb) {
          finish_run = true;  // no increase: restore the base point and stop (:778-781)
        } else {
          accept = true;
        }
      }
      if (accept) {
        // the evaluated query point becomes the base point; start the next step (or finish the run)
        double ns = 0.0;
        if (state != ST_INIT) {
#pragma unroll
          for (int d = 0; d < DIM; ++d) {
            double st = alpha_n * gb[d];
            if (state == ST_LIMIT) st = (d < prm.ps) ? limit_step(st, xb[d], prm.lo[d], prm.hi[d], prm.mrc) : 0.0;
            xb[d] += st;
            ns = fma(st, st, ns);
          }
#pragma unroll
          for (int d = 0; d < DIM; ++d) gb[d] = (d < prm.ps) ? -prm.inv_len[d] * (s[d] - xq[d] * SB) : 0.0;
          fb = fq;
          n_steps += 1;
        }
        step_i += 1;
        if (state != ST_INIT && (sqrt(ns) < prm.step_tol || step_i >= prm.max_steps)) {
          finish_run = true;
        } else {
          alpha_n = prm.alpha0[step_i];
          search = 0;
          gnorm = 0.0;
#pragma unroll
          for (int d = 0; d < DIM; ++d) gnorm = fma(gb[d], gb[d], gnorm);
          state = ST_SEARCH;
        }
      }
    }
    if (finish_run) {
      // restart logic of GradientDescentOptimizerLineSearch::Optimize (gpp_optimization.hpp:1255-1273)
      double nd2 = 0.0;
#pragma unroll
      for (int d = 0; d < DIM; ++d) {
        const double df = outX[static_cast<size_t>(sample) * DIM + d] - xb[d];
        nd2 = fma(df, df, nd2);
      }
      restart_i += 1;
      if (sqrt(nd2) <= prm.tol || restart_i >= prm.max_restarts || prm.max_steps <= 0) {
        outVal[sample] = fb;
        double nx = 0.0;
#pragma unroll
        for (int d = 0; d < DIM; ++d) {
          const double xs = xb[d] * prm.inv_len[d];
          outX[static_cast<size_t>(sample) * DIM + d] = xs;
          nx = fma(xs, xs, nx);
        }
        outH[sample] = -0.5 * nx;
        sample = atomicAdd(next_sample, 1);
        state = ST_FETCH;
      } else {
#pragma unroll
        for (int d = 0; d < DIM; ++d) outX[static_cast<size_t>(sample) * DIM + d] = xb[d];
        step_i = 0;
        alpha_n = prm.alpha0[0];
        search = 0;
        gnorm = 0.0;
#pragma unroll
        for (int d = 0; d < DIM; ++d) gnorm = fma(gb[d], gb[d], gnorm);
        state = ST_SEARCH;
      }
    }
  }
  // integer counters: atomics keep the totals deterministic
  n_evals = __reduce_add_sync(0xffffffffu, n_evals);
  n_steps = __reduce_add_sync(0xffffffffu, n_steps);
  n_point = __reduce_add_sync(0xffffffffu, n_point);
  n_line = __reduce_add_sync(0xffffffffu, n_line);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(prm.stats + 0, static_cast<unsigned long long>(n_evals));
    atomicAdd(prm.stats + 1, static_cast<unsigned long long>(n_steps));
    atomicAdd(prm.stats + 2, static_cast<unsigned long long>(n_point));
    atomicAdd(prm.stats + 3, static_cast<unsigned long long>(n_line));
  }
}

// BIG: the tile rounds use exp2k_shifted, whose 2048-entry table takes 16 KB of static shared memory next to the
// operands, with their exponents in kKappa units.
// Only the tile instantiation has a BIG build.  The host launches it on the shared-memory path only, where it does not
// lower the residency (cmoe_kg_plan_create), so the BIG build has no global-memory branch.
template <int KERNEL, int DIM, int QP, bool BIG = false>
__global__ void __launch_bounds__(kMcThreads, (kg_mc_min_blocks<KERNEL, DIM, QP>()))
    kg_mc_kernel(const __grid_constant__ KgMcParams prm) {
  static_assert(!BIG || kg_tile_path<KERNEL, DIM, QP>(), "only the tile rounds use the 2048-entry table");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ uint64_t mbar;
  __shared__ int next_sample;
  const int cand = blockIdx.y;
  const int N = prm.N, U = prm.U;
  const int s_begin = blockIdx.x * prm.chunk;
  const int s_end = min(prm.num_mc, s_begin + prm.chunk);
  const double* gXt = prm.Xt;
  const double* gPk = prm.Pk + static_cast<size_t>(cand) * N * (QP + 2);
  const double* gXu = prm.Xu + static_cast<size_t>(cand) * U * (DIM + 2);
  if (threadIdx.x == 0) next_sample = s_begin + blockDim.x;
  exp_table_stage();
  if (BIG) exp_table2k_stage();
  if (BIG || prm.use_smem) {
    // stage the per-candidate operands with TMA bulk copies (UBLKCP) signalled through an mbarrier
    double* sXt = reinterpret_cast<double*>(smem_raw);
    double* sPk = sXt + static_cast<size_t>(N) * DIM;
    double* sXu = sPk + static_cast<size_t>(N) * (QP + 2);
    const uint32_t bX = static_cast<uint32_t>(N) * DIM * 8u, bP = static_cast<uint32_t>(N) * (QP + 2) * 8u,
                   bU = static_cast<uint32_t>(U) * (DIM + 2) * 8u;
    if (threadIdx.x == 0) mbar_init(&mbar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_expect_tx(&mbar, bX + bP + bU);
      tma_bulk_g2s(sXt, gXt, bX, &mbar);
      tma_bulk_g2s(sPk, gPk, bP, &mbar);
      tma_bulk_g2s(sXu, gXu, bU, &mbar);
    }
    mbar_wait(&mbar, 0);
    if (BIG) {
      // the tile rounds' exponents are in kKappa units (exp2k_shifted); tile_posterior and tile_line are the only
      // readers of e_j in this build (the union rows' e_u stay natural)
      for (int j = threadIdx.x; j < N; j += blockDim.x) sPk[j * (QP + 2)] *= kKappa;
      __syncthreads();
    }
    kg_mc_body<KERNEL, DIM, QP, true, false, false, BIG>(prm, sXt, sPk, sXu, cand, s_begin, s_end, &next_sample);
  } else {
    __syncthreads();
    kg_mc_body<KERNEL, DIM, QP, false, false>(prm, gXt, gPk, gXu, cand, s_begin, s_end, &next_sample);
  }
}

// General-path kernel (derivative observations): same state machine; the per-point operands are read through the
// read-only path and the per-sample weights from the lane's scratch column (fill_sample_weights).  Persistent grid: one
// CTA per scratch slot, work items (candidate, sample chunk) handed out by an atomic counter.
#ifndef CMOE_MC_GEN_MINBLOCKS
#define CMOE_MC_GEN_MINBLOCKS 2
#endif
// WIDE: the instantiations for 9 <= g <= 31 (stream_point_weights_wide; derivative rows in coordinate order).
template <int KERNEL, int DIM, int QP, bool WIDE = false>
__global__ void __launch_bounds__(kMcThreads, CMOE_MC_GEN_MINBLOCKS)
    kg_mc_gen_kernel(const __grid_constant__ KgMcParams prm) {
  extern __shared__ __align__(16) double gen_ring[];  // [kRingRows][kMcThreads]
  __shared__ int next_sample;
  __shared__ int work_item;
  const int R = prm.N * (1 + prm.g);
  double* aw = prm.aw + static_cast<size_t>(blockIdx.x) * R * kMcThreads + threadIdx.x;
  // The weight stream passes through L1 on its way into the ring (8-byte cp.async is .ca only) and evicts everything
  // else, so the candidate-independent operands of every point — scaled coordinates and e_j — are parked behind the ring
  // in shared memory when they fit (read as broadcast LDS); e_j is the same for every candidate (candidate 0's pack).
  double* sX = gen_ring + static_cast<size_t>(kRingRows + kRingDepth) * kMcThreads;
  double* sE = sX + static_cast<size_t>(prm.N) * DIM;
  if (prm.stage_ops) {
    for (int e = threadIdx.x; e < prm.N * DIM; e += blockDim.x) sX[e] = prm.Xt[e];
    for (int j = threadIdx.x; j < prm.N; j += blockDim.x) {
      sE[2 * j] = prm.Pk[static_cast<size_t>(j) * prm.pk_stride];
      sE[2 * j + 1] = 0.0;
    }
    __syncthreads();
  }
  while (true) {
    if (threadIdx.x == 0) work_item = atomicAdd(prm.work, 1);
    __syncthreads();
    const int w = work_item;
    if (w >= prm.work_total) break;
    const int cand = w / prm.chunks;
    const int s_begin = (w % prm.chunks) * prm.chunk;
    const int s_end = min(prm.num_mc, s_begin + prm.chunk);
    if (threadIdx.x == 0) next_sample = s_begin + blockDim.x;
    __syncthreads();
    const double* gPk = prm.Pk + static_cast<size_t>(cand) * prm.N * prm.pk_stride;
    const double* gXu = prm.Xu + static_cast<size_t>(cand) * prm.U * (DIM + 2);
    const double* gWt = prm.Wt + static_cast<size_t>(cand) * (1 + QP) * R;
    if (prm.stage_ops) {
      kg_mc_body<KERNEL, DIM, QP, true, true, WIDE>(prm, sX, sE, gXu, cand, s_begin, s_end, &next_sample, aw, gWt,
                                                    gen_ring + threadIdx.x);
    } else {
      kg_mc_body<KERNEL, DIM, QP, false, true, WIDE>(prm, prm.Xt, gPk, gXu, cand, s_begin, s_end, &next_sample, aw,
                                                     gWt, gen_ring + threadIdx.x);
    }
    __syncthreads();  // next_sample / work_item are rewritten by thread 0
  }
}

// Large-union build (kg_large.cu, DESIGN.md K17): the same state machine with the union points as ordinary weighted
// points after the training points (prm.N = N + U, prm.U = 0).  Every point operand is per candidate (prm.Xt
// [nc][N+U][DIM], prm.Pk [nc][N+U][pk_stride]) and the weight columns [beta - B c ; c] (~ convention) of every sample are
// precomputed (prm.Wt [nc][num_mc][(N+U)(1+g)]), so the union size only sizes that table.  g == 0 is one row per point.
template <int KERNEL, int DIM, bool WIDE>
__global__ void __launch_bounds__(kMcThreads, CMOE_MC_GEN_MINBLOCKS)
    kg_mc_large_kernel(const __grid_constant__ KgMcParams prm) {
  extern __shared__ __align__(16) double gen_ring[];  // [kRingRows + kRingDepth][kMcThreads]
  __shared__ int next_sample;
  __shared__ int work_item;
  const int R = prm.N * (1 + prm.g);
  double* aw = prm.aw + static_cast<size_t>(blockIdx.x) * R * kMcThreads + threadIdx.x;
  while (true) {
    if (threadIdx.x == 0) work_item = atomicAdd(prm.work, 1);
    __syncthreads();
    const int w = work_item;
    if (w >= prm.work_total) break;
    const int cand = w / prm.chunks;
    const int s_begin = (w % prm.chunks) * prm.chunk;
    const int s_end = min(prm.num_mc, s_begin + prm.chunk);
    if (threadIdx.x == 0) next_sample = s_begin + blockDim.x;
    __syncthreads();
    const double* gXt = prm.Xt + static_cast<size_t>(cand) * prm.N * DIM;
    const double* gPk = prm.Pk + static_cast<size_t>(cand) * prm.N * prm.pk_stride;
    const double* gWt = prm.Wt + static_cast<size_t>(cand) * prm.num_mc * R;
    kg_mc_body<KERNEL, DIM, 2, false, true, WIDE, false, true>(prm, gXt, gPk, nullptr, cand, s_begin, s_end,
                                                                &next_sample, aw, gWt, gen_ring + threadIdx.x);
    __syncthreads();  // next_sample / work_item are rewritten by thread 0
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Phase 2: per-candidate accumulations over the samples' minimisers for the envelope-theorem gradient
//   R[a][row] = sum_i c_ia k(row, x*_i)   (rows = training points then union points; fixed sample order)
//   Gu[u][d]  = sum_i c_iu kb(Xu_u, x*_i) x~*_id ,  GkB[u] = sum_i c_iu kb(Xu_u, x*_i)
// grid (row blocks, candidates); one thread per row.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kAccTile = 64;  // samples per shared-memory tile of the accumulation kernels

// Streams candidate `cand`'s sample records (minimiser, c, -|x*|^2/2) through shared memory in double-buffered tiles
// of kAccTile samples (LDGSTS, 16-byte chunks) and calls body(sx, sc, sh, cnt) once per tile, in sample order:
// sx = [kAccTile][DIM], sc = [kAccTile][QP], sh = [kAccTile], cnt = valid samples.  Slots past num_mc are zero-filled.
// The body may rewrite the tile in place (kg_acc_tile_rows), behind a barrier of its own.
// sbuf: 2 * kAccTile * (DIM + QP + 1) doubles.  Every thread of the CTA must call it.
template <int DIM, int QP, typename F>
__device__ __forceinline__ void acc_stream_samples(const KgAccParams& prm, int cand, double* __restrict__ sbuf,
                                                   F&& body) {
  const double* xs = prm.outX + static_cast<size_t>(cand) * prm.num_mc * DIM;
  const double* cs = prm.recC + static_cast<size_t>(cand) * prm.num_mc * QP;
  const double* hs = prm.outH + static_cast<size_t>(cand) * prm.num_mc;
  constexpr int TS = kAccTile;
  constexpr int kBuf = TS * (DIM + QP + 1);  // doubles per buffer: [TS][DIM] | [TS][QP] | [TS]
  const int num_mc = prm.num_mc;
  const int ntiles = (num_mc + TS - 1) / TS;
  auto load_tile = [&](int tile, int buf) {
    double* sx = sbuf + buf * kBuf;
    double* sc = sx + TS * DIM;
    double* sh = sc + TS * QP;
    const int i0 = tile * TS;
    for (int e = threadIdx.x; e < TS * DIM / 2; e += blockDim.x) {
      const bool ok = i0 + (2 * e) / DIM < num_mc;
      cp_async16(sx + 2 * e, ok ? xs + static_cast<size_t>(i0) * DIM + 2 * e : xs, ok);
    }
    for (int e = threadIdx.x; e < TS * QP / 2; e += blockDim.x) {
      const bool ok = i0 + (2 * e) / QP < num_mc;
      cp_async16(sc + 2 * e, ok ? cs + static_cast<size_t>(i0) * QP + 2 * e : cs, ok);
    }
    for (int e = threadIdx.x; e < TS; e += blockDim.x) {
      const bool ok = i0 + e < num_mc;
      cp_async8(sh + e, ok ? hs + i0 + e : hs, ok);
    }
  };
  load_tile(0, 0);
  cp_async_commit();
  for (int tile = 0; tile < ntiles; ++tile) {
    const int buf = tile & 1;
    if (tile + 1 < ntiles) load_tile(tile + 1, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    double* sx = sbuf + buf * kBuf;
    double* sc = sx + TS * DIM;
    body(sx, sc, sc + TS * QP, min(TS, num_mc - tile * TS));
    __syncthreads();  // the buffer is refilled two tiles later
  }
}

// One thread per row of [training points; union points]; the samples' records stream through shared memory
// (acc_stream_samples) and are read back as warp-broadcast LDS.128.
// TAB selects the table exp under the fast path's range contract (kFastPathRadius).
// GEN (derivative observations): the rows are (point, m), m = 0..g, training rows first; row (p, m > 0) is the
// derivative of k(p, x*) with respect to coordinate t = derivs[m-1] of p:  kb (x~*_t - p~_t) / l_t.  The union rows'
// own-point gradient sums (Gu, GkB) are only produced for g == 0 (kg_g1_kernel does that part otherwise).
template <int KERNEL, int DIM, int QP, bool TAB, bool GEN = false>
__device__ __forceinline__ void kg_acc_body(const KgAccParams& prm, double* __restrict__ sbuf) {
  const int cand = blockIdx.y;
  const int grow = blockIdx.x * blockDim.x + threadIdx.x;
  const int b1 = GEN ? 1 + prm.g : 1;
  const int N = prm.N, U = prm.U, nrows = (N + U) * b1;
  const bool active = grow < nrows;
  const bool is_u = grow >= N * b1;
  const int row = GEN ? (is_u ? N + (grow - N * b1) / b1 : grow / b1) : grow;  // index into [training ; union] points
  const int mrow = GEN ? (is_u ? (grow - N * b1) % b1 : grow % b1) : 0;
  int tcoord = 0;
  double tscale = 0.0;  // 1 / l_t of a derivative row
  if (GEN && mrow > 0) {
    tcoord = prm.derivs[mrow - 1];
    tscale = prm.inv_len[tcoord];
  }
  double xr[DIM];
  double pk0 = 0.0;
  if (active) {
    const double* src = is_u ? (prm.Xu + (static_cast<size_t>(cand) * U + (row - N)) * (DIM + 2))
                             : (prm.Xt + static_cast<size_t>(row) * DIM);
#pragma unroll
    for (int d = 0; d < DIM; ++d) xr[d] = src[d];
    if (is_u) {
      pk0 = src[DIM];
    } else {
      double nrm = 0.0;
#pragma unroll
      for (int d = 0; d < DIM; ++d) nrm = fma(xr[d], xr[d], nrm);
      pk0 = (KERNEL == CMOE_KERNEL_SQUARE_EXPONENTIAL) ? (log(prm.alpha) - 0.5 * nrm) : nrm;
    }
  } else {
#pragma unroll
    for (int d = 0; d < DIM; ++d) xr[d] = 0.0;
  }
  double acc[QP];
#pragma unroll
  for (int a = 0; a < QP; ++a) acc[a] = 0.0;
  double gu[DIM], gkb = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) gu[d] = 0.0;
  const int uu = is_u ? (row - N) : 0;
  double xrt = 0.0;  // own coordinate along the derivative direction
  if (GEN) {
#pragma unroll
    for (int d = 0; d < DIM; ++d)
      if (d == tcoord) xrt = xr[d];
  }
  acc_stream_samples<DIM, QP>(prm, cand, sbuf, [&](const double* sx, const double* sc, const double* sh, int cnt) {
#pragma unroll 2
    for (int i = 0; i < cnt; ++i) {
      double xi[DIM], ci[QP];
#pragma unroll
      for (int d = 0; d < DIM; d += 2) {
        const double2 v = *reinterpret_cast<const double2*>(sx + i * DIM + d);
        xi[d] = v.x;
        xi[d + 1] = v.y;
      }
#pragma unroll
      for (int a = 0; a < QP; a += 2) {
        const double2 v = *reinterpret_cast<const double2*>(sc + i * QP + a);
        ci[a] = v.x;
        ci[a + 1] = v.y;
      }
      double dot = 0.0;
#pragma unroll
      for (int d = 0; d < DIM; ++d) dot = fma(xi[d], xr[d], dot);
      double kv, kb;
      kernel_pair<KERNEL, TAB>(dot, pk0, sh[i], prm.alpha, kv, kb);
      if (GEN && mrow > 0) kv = kb * (sx[i * DIM + tcoord] - xrt) * tscale;
#pragma unroll
      for (int a = 0; a < QP; ++a) acc[a] = fma(ci[a], kv, acc[a]);
      if (!GEN && is_u) {
        double cu = 0.0;
#pragma unroll
        for (int a = 0; a < QP; ++a)
          if (a == uu) cu = ci[a];
        const double w = cu * kb;
        gkb += w;
#pragma unroll
        for (int d = 0; d < DIM; ++d) gu[d] = fma(w, xi[d], gu[d]);
      }
    }
  });
  if (!active) return;
  double* R = prm.R + static_cast<size_t>(cand) * QP * nrows;
#pragma unroll
  for (int a = 0; a < QP; ++a) R[static_cast<size_t>(a) * nrows + grow] = acc[a];
  if (!GEN && is_u) {
    prm.GkB[static_cast<size_t>(cand) * U + uu] = gkb;
#pragma unroll
    for (int d = 0; d < DIM; ++d) prm.Gu[(static_cast<size_t>(cand) * U + uu) * DIM + d] = gu[d];
  }
}

template <int KERNEL, int DIM, int QP, bool GEN>
__global__ void __launch_bounds__(128) kg_acc_kernel(const __grid_constant__ KgAccParams prm) {
  extern __shared__ __align__(16) double acc_smem[];
  if (prm.fast_exp) {
    exp_table_stage();
    kg_acc_body<KERNEL, DIM, QP, true, GEN>(prm, acc_smem);
    return;
  }
  kg_acc_body<KERNEL, DIM, QP, false, GEN>(prm, acc_smem);
}

// ---------------------------------------------------------------------------------------------------------------
// Tile accumulation of the training rows (kg_tile_path instantiation, shared-memory fast path; DESIGN.md K6).
//   R^T[row][a] = sum_i exp(X~_row . x~*_i + e_row + h_i) c_ia ,   e_row = ln(alpha) - |X~_row|^2 / 2,  h_i = -|x~*_i|^2/2
// is two FP64 DMMA m16n8k4 products per 16 rows x 8 samples: the exponents in kKappa units (M = 16 rows, N = 8 samples,
// K = DIM, A = kKappa X~, accumulator seeded with kKappa e_row; h_i enters the element-wise exp2k_shifted as its
// rounding constant, the factor exp2k_split leaves goes into c_i) and R^T += KV C (K = the 8 samples, N = QP).  The
// second product takes KV's accumulator layout as its A operand, k-step 0 = the even columns, k-step 1 = the odd ones.
// Column n of a sample group s0 is sample s0 + (n >> 1) + 4 (n & 1), so that lane (g, t) holds samples s0 + t and
// s0 + t + 4, and its C operands c[s0 + t][g], c[s0 + t + 4][g] are two conflict-free LDS.  The K order of the exponent
// product is coordinate 2t + ks in k-step ks, so that a lane's x* operands of both k-steps are one LDS.128.
// A warp owns kAccRowTiles tiles of 16 rows: the row operands (A fragments, e_row) and the accumulators stay in
// registers over all samples, and each group's sample operands feed 4 kAccRowTiles DMMAs.  Every lane walks the samples
// in ascending groups, so a candidate's R does not depend on its batch or the launch.  Rows past N read row N - 1 and
// are not stored; samples past num_mc are zero-filled (c = 0, finite exponent): exact zeros.
// The last CTA of each candidate (blockIdx.x = gridDim.x - 1) does the U <= QP union rows instead: their R rows and the
// own-point sums Gu, GkB (kg_acc_body's formulas) with kAccUnionSplit threads per union row, each taking every
// kAccUnionSplit-th sample of a tile, combined by a fixed butterfly.
// ---------------------------------------------------------------------------------------------------------------
#ifndef CMOE_ACC_ROW_TILES
#define CMOE_ACC_ROW_TILES 4
#endif
constexpr int kAccRowTiles = CMOE_ACC_ROW_TILES;   // 16-row tiles per warp
constexpr int kAccTileThreads = 128;
constexpr int kAccTileRowsPerCta = kAccTileThreads / 32 * 16 * kAccRowTiles;
constexpr int kAccUnionSplit = 16;
static_assert(kAccTileThreads / kAccUnionSplit >= 8, "one thread group per union row (U <= QP = 8)");

template <int DIM, int QP>
__device__ __forceinline__ void kg_acc_tile_rows(const KgAccParams& prm, double* __restrict__ sbuf) {
  static_assert(DIM == 8 && QP == 8, "one k-step pair of coordinates and of samples, one n-block of union columns");
  constexpr int T = kAccRowTiles;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int cand = blockIdx.y, N = prm.N, nrows = N + prm.U;
  const int r0 = (blockIdx.x * (kAccTileThreads / 32) + (threadIdx.x >> 5)) * 16 * T;
  const double lna = log(prm.alpha);
  double xa[T][2][2], e[T][2], acc[T][4];  // xa[tile][ks][h] = X~[row g + 8h][2t + ks], e[tile][h] = e_row of row g + 8h
#pragma unroll
  for (int k = 0; k < T; ++k) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const double* x = prm.Xt + static_cast<size_t>(min(r0 + 16 * k + g + 8 * h, N - 1)) * DIM;
      double nrm = 0.0;
#pragma unroll
      for (int d = 0; d < DIM; ++d) nrm = fma(x[d], x[d], nrm);
      // the exponents in kKappa units (exp2k_shifted)
      e[k][h] = kKappa * (lna - 0.5 * nrm);
      xa[k][0][h] = kKappa * x[2 * t];
      xa[k][1][h] = kKappa * x[2 * t + 1];
    }
    acc[k][0] = acc[k][1] = acc[k][2] = acc[k][3] = 0.0;
  }
  acc_stream_samples<DIM, QP>(prm, cand, sbuf, [&](const double* sx, double* sc, double* sh, int cnt) {
    // once per sample and CTA: h_i becomes exp2k_split's rounding constant C_i, and its factor f_i goes into c_i (every
    // slot, so that the zero-filled ones past num_mc get a finite exponent)
    for (int i = threadIdx.x; i < kAccTile; i += blockDim.x) {
      double f;
      exp2k_split(sh[i], sh[i], f);
#pragma unroll
      for (int a = 0; a < QP; ++a) sc[i * QP + a] *= f;
    }
    __syncthreads();
#pragma unroll 1
    for (int s0 = 0; s0 < cnt; s0 += 8) {
      const double2 xb = *reinterpret_cast<const double2*>(sx + (s0 + (g >> 1) + 4 * (g & 1)) * DIM + 2 * t);
      const double h0 = sh[s0 + t], h1 = sh[s0 + t + 4];
      const double c0 = sc[(s0 + t) * QP + g], c1 = sc[(s0 + t + 4) * QP + g];
#pragma unroll
      for (int k = 0; k < T; ++k) {
        double kv[4] = {e[k][0], e[k][0], e[k][1], e[k][1]};
        dmma_m16n8k8(kv[0], kv[1], kv[2], kv[3], xa[k][0][0], xa[k][0][1], xa[k][1][0], xa[k][1][1], xb.x, xb.y);
        kv[0] = exp2k_shifted(kv[0], h0);
        kv[1] = exp2k_shifted(kv[1], h1);
        kv[2] = exp2k_shifted(kv[2], h0);
        kv[3] = exp2k_shifted(kv[3], h1);
        dmma_m16n8k8(acc[k][0], acc[k][1], acc[k][2], acc[k][3], kv[0], kv[2], kv[1], kv[3], c0, c1);
      }
    }
  });
  double* R = prm.R + static_cast<size_t>(cand) * QP * nrows;
#pragma unroll
  for (int k = 0; k < T; ++k) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 16 * k + g + 8 * h;
      if (row < N) {
        R[static_cast<size_t>(2 * t) * nrows + row] = acc[k][2 * h];
        R[static_cast<size_t>(2 * t + 1) * nrows + row] = acc[k][2 * h + 1];
      }
    }
  }
}

template <int DIM, int QP>
__device__ __forceinline__ void kg_acc_tile_union(const KgAccParams& prm, double* __restrict__ sbuf) {
  const int cand = blockIdx.y, N = prm.N, U = prm.U, nrows = N + U;
  const int u = threadIdx.x / kAccUnionSplit, part = threadIdx.x % kAccUnionSplit;
  const int uc = min(u, U - 1);  // groups past U read a valid union row and store nothing
  const double* src = prm.Xu + (static_cast<size_t>(cand) * U + uc) * (DIM + 2);
  double xr[DIM];
#pragma unroll
  for (int d = 0; d < DIM; ++d) xr[d] = src[d];
  const double pk0 = src[DIM];
  double acc[QP], gu[DIM], gkb = 0.0;
#pragma unroll
  for (int a = 0; a < QP; ++a) acc[a] = 0.0;
#pragma unroll
  for (int d = 0; d < DIM; ++d) gu[d] = 0.0;
  acc_stream_samples<DIM, QP>(prm, cand, sbuf, [&](const double* sx, const double* sc, const double* sh, int cnt) {
#pragma unroll 2
    for (int i = part; i < cnt; i += kAccUnionSplit) {
      double xi[DIM], ci[QP];
#pragma unroll
      for (int d = 0; d < DIM; d += 2) {
        const double2 v = *reinterpret_cast<const double2*>(sx + i * DIM + d);
        xi[d] = v.x;
        xi[d + 1] = v.y;
      }
#pragma unroll
      for (int a = 0; a < QP; a += 2) {
        const double2 v = *reinterpret_cast<const double2*>(sc + i * QP + a);
        ci[a] = v.x;
        ci[a + 1] = v.y;
      }
      const double kv = exp_tab2k(dot_dim<DIM>(xi, xr, 0.0) + (pk0 + sh[i]));
      double cu = 0.0;
#pragma unroll
      for (int a = 0; a < QP; ++a) {
        acc[a] = fma(ci[a], kv, acc[a]);
        if (a == uc) cu = ci[a];
      }
      const double w = cu * kv;
      gkb += w;
#pragma unroll
      for (int d = 0; d < DIM; ++d) gu[d] = fma(w, xi[d], gu[d]);
    }
  });
  // fixed butterfly over the group's kAccUnionSplit lanes (the same bits on all of them)
#pragma unroll
  for (int m = 1; m < kAccUnionSplit; m <<= 1) {
#pragma unroll
    for (int a = 0; a < QP; ++a) acc[a] += __shfl_xor_sync(0xffffffffu, acc[a], m);
#pragma unroll
    for (int d = 0; d < DIM; ++d) gu[d] += __shfl_xor_sync(0xffffffffu, gu[d], m);
    gkb += __shfl_xor_sync(0xffffffffu, gkb, m);
  }
  if (part != 0 || u >= U) return;
  double* R = prm.R + static_cast<size_t>(cand) * QP * nrows;
#pragma unroll
  for (int a = 0; a < QP; ++a) R[static_cast<size_t>(a) * nrows + N + u] = acc[a];
  prm.GkB[static_cast<size_t>(cand) * U + u] = gkb;
#pragma unroll
  for (int d = 0; d < DIM; ++d) prm.Gu[(static_cast<size_t>(cand) * U + u) * DIM + d] = gu[d];
}

// grid (row CTAs of kAccTileRowsPerCta training rows + 1 union CTA, candidates); only under the fast path's range
// contract (exp_tab2k)
template <int DIM, int QP>
__global__ void __launch_bounds__(kAccTileThreads) kg_acc_tile_kernel(const __grid_constant__ KgAccParams prm) {
  extern __shared__ __align__(16) double acc_smem[];
  exp_table2k_stage();
  if (blockIdx.x == gridDim.x - 1) {
    kg_acc_tile_union<DIM, QP>(prm, acc_smem);
  } else {
    kg_acc_tile_rows<DIM, QP>(prm, acc_smem);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Host dispatch.  Every launcher works out its own grid and dynamic shared memory from its parameters, the sample
// chunks per candidate (MC launchers) and the candidates of the batch.  kg_select picks an instantiation's launchers
// for a plan's shape; the compiled set is the entry lists at the end of this file.
// ---------------------------------------------------------------------------------------------------------------
using KgMcLaunch = void (*)(const KgMcParams&, int chunks, int nb, cudaStream_t s);
using KgAccLaunch = void (*)(const KgAccParams&, int nb, cudaStream_t s);

// kg_mc_kernel's operands staged in shared memory (the g == 0 fast path)
template <int DIM, int QP>
size_t kg_smem_bytes(int N, int U) {
  return (static_cast<size_t>(N) * (DIM + QP + 2) + static_cast<size_t>(U) * (DIM + 2)) * sizeof(double);
}
// the accumulation kernels' two sample tiles (acc_stream_samples)
template <int DIM, int QP>
constexpr size_t kAccSmemBytes = 2 * static_cast<size_t>(kAccTile) * (DIM + QP + 1) * sizeof(double);

// grid (sample chunks, candidates); the operands go to shared memory when p.use_smem is set
template <int KERNEL, int DIM, int QP, bool BIG = false>
void launch_kg_mc(const KgMcParams& p, int chunks, int nb, cudaStream_t s) {
  const size_t smem = p.use_smem ? kg_smem_bytes<DIM, QP>(p.N, p.U) : 0;
  // function attributes are per device: set on every launch (cheap), never cached process-wide
  cudaFuncSetAttribute(kg_mc_kernel<KERNEL, DIM, QP, BIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  kg_mc_kernel<KERNEL, DIM, QP, BIG><<<dim3(chunks, nb), kMcThreads, smem, s>>>(p);
}
// resident CTAs of kg_mc_kernel per SM on the current device with `smem` bytes of staged operands (0: global memory)
template <int KERNEL, int DIM, int QP, bool BIG = false>
int kg_mc_ctas_per_sm(size_t smem) {
  CMOE_CUDA(cudaFuncSetAttribute(kg_mc_kernel<KERNEL, DIM, QP, BIG>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 200 * 1024));
  int per_sm = 0;
  CMOE_CUDA(
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kg_mc_kernel<KERNEL, DIM, QP, BIG>, kMcThreads, smem));
  return per_sm;
}
// persistent grid over the p.work_total = chunks * candidates work items
template <int KERNEL, int DIM, int QP, bool WIDE = false>
void launch_kg_mc_gen(const KgMcParams& p, int, int, cudaStream_t s) {
  int dev = 0, sms = 1, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t ring_bytes = static_cast<size_t>(kRingRows + kRingDepth) * kMcThreads * sizeof(double) +
                            (p.stage_ops ? static_cast<size_t>(p.N) * (DIM + 2) * sizeof(double) : 0);
  cudaFuncSetAttribute(kg_mc_gen_kernel<KERNEL, DIM, QP, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       static_cast<int>(ring_bytes));
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kg_mc_gen_kernel<KERNEL, DIM, QP, WIDE>, kMcThreads,
                                                ring_bytes);
  const int grid = std::max(1, std::min(std::min(p.aw_slots, p.work_total), sms * std::max(1, per_sm)));
  kg_mc_gen_kernel<KERNEL, DIM, QP, WIDE><<<grid, kMcThreads, ring_bytes, s>>>(p);
}
// persistent grid over the p.work_total work items, at most one CTA per scratch slot
template <int KERNEL, int DIM, bool WIDE>
void launch_kg_mc_large(const KgMcParams& p, cudaStream_t s) {
  int dev = 0, sms = 1, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t ring_bytes = static_cast<size_t>(kRingRows + kRingDepth) * kMcThreads * sizeof(double);
  cudaFuncSetAttribute(kg_mc_large_kernel<KERNEL, DIM, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       static_cast<int>(ring_bytes));
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kg_mc_large_kernel<KERNEL, DIM, WIDE>, kMcThreads, ring_bytes);
  const int grid = std::max(1, std::min(std::min(p.aw_slots, p.work_total), sms * std::max(1, per_sm)));
  kg_mc_large_kernel<KERNEL, DIM, WIDE><<<grid, kMcThreads, ring_bytes, s>>>(p);
}
// grid (128-row CTAs, candidates) over the (N + U) (1 + g) rows
template <int KERNEL, int DIM, int QP, bool GEN>
void launch_kg_acc(const KgAccParams& p, int nb, cudaStream_t s) {
  const int nrows = (p.N + p.U) * (GEN ? 1 + p.g : 1);
  cudaFuncSetAttribute(kg_acc_kernel<KERNEL, DIM, QP, GEN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
  kg_acc_kernel<KERNEL, DIM, QP, GEN><<<dim3((nrows + 127) / 128, nb), 128, kAccSmemBytes<DIM, QP>, s>>>(p);
}
// grid (row CTAs + the union CTA, candidates)
template <int DIM, int QP>
void launch_kg_acc_tile(const KgAccParams& p, int nb, cudaStream_t s) {
  const dim3 grid((p.N + kAccTileRowsPerCta - 1) / kAccTileRowsPerCta + 1, nb);
  kg_acc_tile_kernel<DIM, QP><<<grid, kAccTileThreads, kAccSmemBytes<DIM, QP>, s>>>(p);
}

// A plan's builds for its shape: the MC and accumulation launchers, whether the operands are staged in shared memory
// (the fast path, whose exps rely on kFastPathRadius's range contract) and the resident CTAs per SM that the sample
// chunks are sized for.
struct KgPath {
  KgMcLaunch mc;
  KgAccLaunch acc;
  bool use_smem;
  int ctas_per_sm;
};
using KgSelect = KgPath (*)(int N, int U, int g, bool fast);

// The builds an entry compiles.
enum KgBuilds {
  kKgFast,     // the g == 0 path only
  kKgFastGen,  // that and the general path for derivative observations (g <= 8)
  kKgWide,     // the wide general path only (9 <= g <= 31)
};

// An instantiation's builds for N training points, U union points, g derivative observations per point and whether the
// fast path's range contract holds.  find_kg_entry hands g > 0 only to entries with a general path, g > 8 only to wide
// ones.
//  * The general path hands its work items to a persistent grid and keeps 3 CTAs per SM, the count its scratch slots
//    are sized for; its exps are the guarded ones.
//  * g == 0 stages the operands in shared memory where they fit in 200 KiB and the range contract holds, and sizes the
//    chunks for kg_mc_kernel's residency as the occupancy API reports it.  There the tile instantiation takes its tile
//    accumulation kernel, and the build of kg_mc_kernel whose tile rounds use the 2048-entry exp table (16 KB more
//    shared memory per CTA) wherever that build keeps the residency of the 64-entry one, so that neither the fast
//    path's N range nor its occupancy shrinks.
template <int KERNEL, int DIM, int QP, KgBuilds B>
KgPath kg_select(int N, int U, int g, bool fast) {
  if constexpr (B == kKgWide) {
    return {&launch_kg_mc_gen<KERNEL, DIM, QP, true>, &launch_kg_acc<KERNEL, DIM, QP, true>, false, 3};
  } else {
    if constexpr (B == kKgFastGen) {
      if (g > 0) return {&launch_kg_mc_gen<KERNEL, DIM, QP>, &launch_kg_acc<KERNEL, DIM, QP, true>, false, 3};
    }
    const size_t smem = kg_smem_bytes<DIM, QP>(N, U);
    const bool use_smem = smem <= 200 * 1024 && fast;
    const int per_sm = std::max(1, kg_mc_ctas_per_sm<KERNEL, DIM, QP>(use_smem ? smem : 0));
    if constexpr (kg_tile_path<KERNEL, DIM, QP>()) {
      if (use_smem) {
        const bool big = kg_mc_ctas_per_sm<KERNEL, DIM, QP, true>(smem) >= per_sm;
        return {big ? &launch_kg_mc<KERNEL, DIM, QP, true> : &launch_kg_mc<KERNEL, DIM, QP>,
                &launch_kg_acc_tile<DIM, QP>, true, per_sm};
      }
    }
    return {&launch_kg_mc<KERNEL, DIM, QP>, &launch_kg_acc<KERNEL, DIM, QP, false>, use_smem, per_sm};
  }
}

// One compiled instantiation in the run-time dispatch table of kg.cu.
struct KgDispatchEntry {
  int kernel, dim, qp;
  bool gen;   // has the general path (derivative observations)
  bool wide;  // the general path for 9 <= g <= 31 only
  KgSelect select;
};
template <int KERNEL, int DIM, int QP, KgBuilds B>
constexpr KgDispatchEntry kg_entry() {
  return {KERNEL, DIM, QP, B != kKgFast, B == kKgWide, &kg_select<KERNEL, DIM, QP, B>};
}
bool register_kg_entries(std::initializer_list<KgDispatchEntry> entries);
// g: derivative observations per point; entries with g <= 8 never dispatch to a wide entry, g > 8 only to one
const KgDispatchEntry* find_kg_entry(int kernel, int dim, int Q, int g);

// The compiled set, per padded dimension D (kg_mc_inst_*.cu).  Union-row counts: 2, 4, 8, 16, 24, 32 (24 serves
// config 4: q = 4 with 4 derivative observations -> 20 rows; the 32-wide instantiation spilled ~1.5 KB per thread there)
#define CMOE_KG_ENTRIES_FOR_DIM(D)                                                                                    \
  kg_entry<0, D, 2, kKgFast>(), kg_entry<0, D, 4, kKgFast>(), kg_entry<0, D, 8, kKgFastGen>(),                        \
      kg_entry<0, D, 16, kKgFastGen>(), kg_entry<0, D, 24, kKgFastGen>(), kg_entry<0, D, 32, kKgFastGen>(),           \
      kg_entry<1, D, 2, kKgFast>(), kg_entry<1, D, 4, kKgFast>(), kg_entry<1, D, 8, kKgFastGen>(),                    \
      kg_entry<1, D, 16, kKgFastGen>(), kg_entry<1, D, 24, kKgFastGen>(), kg_entry<1, D, 32, kKgFastGen>()

// Wide general path (9 <= g <= 31, kg_mc_wide_*.cu): only what such a g can reach — dim >= 9 (padded 12, 16, 32) and
// Q = U (1 + g) >= 10 (widths 16, 24, 32).  The accumulation kernel does not depend on g and is the narrow entry's.
#define CMOE_KG_WIDE_ENTRIES_FOR_DIM(D)                                                                    \
  kg_entry<0, D, 16, kKgWide>(), kg_entry<0, D, 24, kKgWide>(), kg_entry<0, D, 32, kKgWide>(),             \
      kg_entry<1, D, 16, kKgWide>(), kg_entry<1, D, 24, kKgWide>(), kg_entry<1, D, 32, kKgWide>()

// The large-union build's run-time dispatch table (kg_large.cu): one entry per kernel, padded dimension and ring kind.
using KgLargeLaunch = void (*)(const KgMcParams&, cudaStream_t);
struct KgLargeEntry {
  int kernel, dim;
  bool wide;  // 9 <= g <= 31 (stream_point_weights_wide)
  KgLargeLaunch mc;
};
bool register_kg_large_entries(std::initializer_list<KgLargeEntry> entries);
const KgLargeEntry* find_kg_large_entry(int kernel, int dim, int g);
#define CMOE_KG_LARGE_ENTRIES_FOR_DIM(D) \
  KgLargeEntry{0, D, false, &launch_kg_mc_large<0, D, false>}, KgLargeEntry{1, D, false, &launch_kg_mc_large<1, D, false>}
#define CMOE_KG_LARGE_WIDE_ENTRIES_FOR_DIM(D) \
  KgLargeEntry{0, D, true, &launch_kg_mc_large<0, D, true>}, KgLargeEntry{1, D, true, &launch_kg_mc_large<1, D, true>}

// The q-KG set-up that cmoe_kg_plan_create (kg.cu) and the large-union stages (kg_large.cu) share.
// The inner optimiser's argument checks, in this order: the num_fidelity range, g <= 31, distinct partials past 8,
// inner steps <= 4096, a non-empty inner box.  Throws CMOE_ERR_BOUNDS.
void kg_check_inner(const KernelSpec& spec, int num_fidelity, const cmoe_gd_params* inner, const double* inner_bounds);
// The inner optimiser's KgMcParams fields that follow from the GP, `inner` and the inner bounds (in the frame of A), for
// ps free coordinates, M discretisation points and num_mc samples; alpha0 = the device step sizes (kg_step_sizes).
// Every other field is zero: the caller sets the row sets (N, U, Q, pk_stride), use_smem, stage_ops, the chunk and the
// buffers.
KgMcParams kg_inner_params(const cmoe_gp& gp, int ps, int M, int num_mc, const cmoe_gd_params& inner,
                           const double* inner_bounds, const double* alpha0);
// pre_mult (i + 1)^-gamma for the inner steps i (at least one entry)
std::vector<double> kg_step_sizes(const cmoe_gd_params& inner);
// discrete_pts [num_pts][ps] -> [max(1, num_pts)][dim] with the fidelity coordinates pinned to 1 (...cpp:259-261, 365)
std::vector<double> kg_pinned_discrete(const double* discrete_pts, int num_pts, int ps, int dim);
// samples per work item of the MC kernel: aim for >= ~8 waves of ctas_per_sm CTAs per SM over `candidates`, between 2
// and 16 samples per lane
int kg_samples_per_item(long long candidates, int num_mc, int sms, int ctas_per_sm);

// kg.cu's per-candidate stages that the large-union path shares (asynchronous on s)
// KG[c] = best_posterior[c] + mean of outVal[c][:], NaN where fail[c] != 0 (kg_value_kernel)
void kg_value(int nb, int num_mc, const double* outVal, const double* best_post, const int* fail, double* kg,
              cudaStream_t s);
// every sample's minimiser <- the max_num_restarts <= 0 fill value, in the operands' frame (kg_fill_point_kernel)
void kg_fill_points(const KernelSpec& spec, const Centre& ctr, int samples, int DIMP, double* outX, double* outH,
                    cudaStream_t s);
// Tp[c][a'][a] = R[c][a'][n + a] - sum_j R[c][a'][j] B[c][a][j]  (kg_tprime_kernel); R [nb][QP][n + Q], B [nb][Q][n]
void kg_tprime(int nb, int n, int Q, int QP, const double* R, const double* B, double* Tp, cudaStream_t s);
// G1[c][p][d] = sum_i sum_m c_i,(p,m) d K(Xu_p row m, x*_i) / d Xu_p,d  (kg_g1_kernel); recC [nb][num_mc][QP]
void kg_g1(const KernelSpec& spec, const Centre& ctr, int nb, int U, int q, int QP, int DIMP, int num_mc,
           const double* P, const double* recC, const double* outX, double* G1, cudaStream_t s);

}  // namespace cmoe

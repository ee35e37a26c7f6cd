// Device-side building blocks of the dense FP64 factorisation shared by linalg.cu (launch-per-step path, small
// systems), potrf_coop.cu (one cooperative launch per outer panel) and sample.cu (batched Cholesky): warp-level register
// Cholesky of a 32x32 block, the 64x64 diagonal-block factorisation built from it, rotating-window triangular
// substitution, the FP64 tensor-pipe instruction.
#pragma once

#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {
namespace {

constexpr int NB = 64;        // Cholesky block size == K depth of one DMMA tile product
constexpr int LDT = NB + 4;   // smem leading dimension: 68 = 4 (mod 16) makes the DMMA fragment loads conflict-free
constexpr double kPivotTol = 1.0e-16;  // gpp_linear_algebra.cpp:118

// linear index of a lower-triangular tile grid -> (ti, tj), tj <= ti
__device__ __forceinline__ void tri_tile(int t, int& ti, int& tj) {
  ti = static_cast<int>((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while (ti * (ti + 1) / 2 > t) --ti;
  while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
  tj = t - ti * (ti + 1) / 2;
}

// --------------------------------------------------------------------------------------------------------------
// Diagonal-block factorisation + panel solve.  The column recurrence sqrt -> scale -> update is the latency-critical
// chain of the whole factorisation (n/64 dependent block steps), so it runs out of REGISTERS: a warp factors a 32x32
// block with lane r holding row r and the pivot / multiplier columns travelling by shuffle — no barriers, no shared
// memory round trips inside the recurrence.
// --------------------------------------------------------------------------------------------------------------
constexpr int PT = 128;  // threads of the panel kernel: one panel row per thread

// The register-resident recurrences below are written as SHORT LOOPS over a rotating register window (after step k
// the window is shifted so that slot 0 is always the pivot column) instead of fully unrolled triangles: straight-line
// code of thousands of instructions that execute once each runs at instruction-fetch speed (measured: 18 us for a
// 64x64 factorisation, 25 us for the panel solve), a loop body of a few hundred instructions stays in the I-cache.
// Slots that rotate past the end of the row compute on padding and are never stored.

// In-register Cholesky of a 32x32 block: on entry a[c] = A[lane][c] (c <= lane meaningful).  The finished column j of
// L is written to LT[(col0 + j) * LTS + col0 + lane] (transposed factor) and rd[col0 + j] = 1/L_jj (FAST) or L_jj.
// Returns 0 or the 1-based index of the first pivot that fails `> 1e-16` (gpp_linear_algebra.cpp:118,141-142); the
// outcome is warp-uniform and only evaluated at the end (the arithmetic after a failed pivot is discarded).
// The finished column is broadcast through a double-buffered shared column (one STS + one __syncwarp per column).
// FAST: sqrt and divide through one reciprocal square root + Newton corrections — the same results as sqrt()/"/" to
// the last bit in all but rare halfway cases (and exactly when the true results are representable) at a third of the
// dependent latency; small systems (known-answer cases) keep IEEE sqrt / divide.
constexpr int LTS = NB + 2;  // row stride of the transposed factor (even: 16-byte aligned rows)

// The FAST pivot step of chol32_warp, in two parts so that the kernels keep their instruction order around the column
// store: l = sqrt(p) and the multiplier q = a / l from the library rsqrt with one correction step each
// (chol_pivot_fast), then r = 1/l from rsqrt and one Newton step (chol_pivot_recip: no divide on the per-column critical
// path).  l and q equal the IEEE sqrt and divide except when the exact value lies within 32 u^2 (relative, u = 2^-53)
// of a rounding midpoint, and exactly when the true result is representable; r is within 0.55 ulp of 1/l (measured 0.50,
// tests/test_gpu_fast_math.py).  Arguments: pivots p > kPivotTol (smaller ones fail the factorisation and their results
// are discarded) and any finite a.
__device__ __forceinline__ void chol_pivot_fast(double p, double a, double& l, double& q) {
  const double y = rsqrt(p);
  l = p * y;
  l = fma(0.5 * y, fma(-l, l, p), l);
  q = a * y;
  q = fma(fma(-q, l, a), y, q);
}
__device__ __forceinline__ double chol_pivot_recip(double p, double l) {
  const double r = rsqrt(p);  // ~ 1/l
  return fma(fma(-l, r, 1.0), r, r);
}

template <bool FAST>
__device__ __forceinline__ int chol32_warp(double (&a)[32], int lane, double* colbuf /* [2][64], [32..63] = 0 */,
                                           double* LT, double* rd, int col0) {
  int fail = 0;
#pragma unroll 1
  for (int j = 0; j < 32; ++j) {
    const double piv = __shfl_sync(0xffffffffu, a[0], j);
    fail = (fail == 0 && !(piv > kPivotTol)) ? j + 1 : fail;
    double l, q;
    if (FAST) {
      chol_pivot_fast(piv, a[0], l, q);
    } else {
      l = sqrt(piv);
      q = a[0] / l;
    }
    const double lj = (lane == j) ? l : q;
    if (lane >= j) LT[(col0 + j) * LTS + col0 + lane] = lj;
    if (FAST) {
      const double r = chol_pivot_recip(piv, l);
      if (lane == j) rd[col0 + j] = r;
    } else {
      if (lane == j) rd[col0 + j] = l;
    }
    double* col = colbuf + (j & 1) * 64;
    col[lane] = lj;
    __syncwarp();
    // window slot k <-> column j + k; multipliers L[j+k][j] = col[j+k] (zero beyond the block)
#pragma unroll
    for (int k = 1; k < 32; ++k) a[k - 1] = fma(-lj, col[j + k], a[k]);
    a[31] = 0.0;
  }
  return fail;
}

// Same factorisation, two columns per round: the 2 x 2 pivot block [l11 0; l21 l22] is formed from three shuffles, both
// multiplier columns travel through ONE shared-memory round trip and the window is updated by a rank-2 step.
// LEAN = false: the arithmetic (operation order and roundings) is exactly that of two successive rounds of
// chol32_warp<true>.  LEAN = true (the cooperative large-n path): pivots through sqrt_rsqrt, multipliers as a * (1/l)
// without the correction step — the column recurrence is the latency-critical chain of the whole factorisation
// (measured per column, one warp alone on the SM: 324 cycles single-column, 270 paired, see microbench_chain.cu).
// colbuf: [2][2][64] with [32..63] of every column zero.
// prog (optional, shared memory): columns finished so far, for follower warps that trail the factorisation.  The
// column data (LT, rd) and the counter are shared-memory stores of the same warp, issued in program order behind a
// __syncwarp(); no fence is placed on the pivot chain (measured: a block fence by one lane costs ~70 cycles there).
template <bool LEAN = false>
__device__ __forceinline__ int chol32_warp_pair(double (&a)[32], int lane, double* colbuf,
                                                double* LT, double* rd, int col0, volatile int* prog = nullptr) {
  int fail = 0;
#pragma unroll 1
  for (int j = 0; j < 32; j += 2) {
    const double p11 = __shfl_sync(0xffffffffu, a[0], j);
    const double p21 = __shfl_sync(0xffffffffu, a[0], j + 1);
    const double p22 = __shfl_sync(0xffffffffu, a[1], j + 1);
    fail = (fail == 0 && !(p11 > kPivotTol)) ? j + 1 : fail;
    if (fail) break;  // warp-uniform: nothing after a failed pivot is used; do not feed 0 / NaN to rsqrt
    double y1, l11, q1, l21;
    if (LEAN) {
      sqrt_rsqrt(p11, l11, y1);
      q1 = a[0] * y1;
      l21 = p21 * y1;
    } else {
      y1 = rsqrt(p11);
      l11 = p11 * y1;
      l11 = fma(0.5 * y1, fma(-l11, l11, p11), l11);
      q1 = a[0] * y1;
      q1 = fma(fma(-q1, l11, a[0]), y1, q1);
      l21 = p21 * y1;  // what lane j+1 computes as its q1 (same operations on the same operands)
      l21 = fma(fma(-l21, l11, p21), y1, l21);
    }
    // column j+1 after the update by column j
    const double d2 = fma(-l21, l21, p22);
    fail = (fail == 0 && !(d2 > kPivotTol)) ? j + 2 : fail;
    if (fail) break;
    const double a1 = fma(-q1, l21, a[1]);
    double y2, l22, q2;
    if (LEAN) {
      sqrt_rsqrt(d2, l22, y2);
      q2 = a1 * y2;
    } else {
      y2 = rsqrt(d2);
      l22 = d2 * y2;
      l22 = fma(0.5 * y2, fma(-l22, l22, d2), l22);
      q2 = a1 * y2;
      q2 = fma(fma(-q2, l22, a1), y2, q2);
    }
    const double lj1 = (lane == j) ? l11 : q1;
    const double lj2 = (lane == j + 1) ? l22 : q2;
    if (lane >= j) LT[(col0 + j) * LTS + col0 + lane] = lj1;
    if (lane >= j + 1) LT[(col0 + j + 1) * LTS + col0 + lane] = lj2;
    if (LEAN) {
      if (lane == j) rd[col0 + j] = y1;
      if (lane == j + 1) rd[col0 + j + 1] = y2;
    } else {
      if (lane == j) rd[col0 + j] = fma(fma(-l11, y1, 1.0), y1, y1);  // one Newton step on 1/l from y ~ 1/l
      if (lane == j + 1) rd[col0 + j + 1] = fma(fma(-l22, y2, 1.0), y2, y2);
    }
    double* c1 = colbuf + ((j >> 1) & 1) * 128;
    double* c2 = c1 + 64;
    c1[lane] = lj1;
    c2[lane] = lj2;
    __syncwarp();
    if (prog && lane == 0) *prog = j + 2;
    // window slot k <-> column j + k
#pragma unroll
    for (int k = 2; k < 32; ++k) a[k - 2] = fma(-lj2, c2[j + k], fma(-lj1, c1[j + k], a[k]));
    a[30] = 0.0;
    a[31] = 0.0;
  }
  if (prog && fail && lane == 0) *prog = 1 << 20;  // release the followers (their results are discarded)
  return fail;
}

// Software-pipelined form of the paired factorisation (lean pivots).  Measured: in chol32_warp_pair half of a round is
// the ISSUE time of the 60 window FMAs + 60 shared-memory loads that sit, in program order, between one round's pivots
// and the next round's shuffles (an in-order warp cannot start the next dependent chain before they have issued).
// Here only the two window slots the next pivots need are updated right away; the rest of round j's rank-2 update is
// carried as "pending" (multipliers in registers, columns in the other parity buffer) and executed inside round j+1,
// in one branch-free basic block together with that round's dependent pivot chain, so the scheduler fills the chain's
// latency gaps with it.  A failed pivot is recorded, not branched on (the raw RSQ64H seed has no slow path).
__device__ __forceinline__ int chol32_warp_pipe(double (&a)[32], int lane, double* colbuf, double* LT, double* rd,
                                                int col0, volatile int* prog = nullptr) {
  int fail = 0;
  double plj1 = 0.0, plj2 = 0.0;            // pending multipliers of the previous round (zero: nothing pending)
  const double* pc1 = colbuf + 128;         // previous round's column buffers (start: zeros)
  const double* pc2 = colbuf + 192;
  double p11 = __shfl_sync(0xffffffffu, a[0], 0);
  double p21 = __shfl_sync(0xffffffffu, a[0], 1);
  double p22 = __shfl_sync(0xffffffffu, a[1], 1);
#pragma unroll 1
  for (int j = 0; j < 32; j += 2) {
    // ---- pivot chain of columns j, j+1 (dependent) ----
    fail = (fail == 0 && !(p11 > kPivotTol)) ? j + 1 : fail;
    double y1, l11, y2, l22;
    sqrt_rsqrt(p11, l11, y1);
    const double q1 = a[0] * y1;
    const double l21 = p21 * y1;
    const double d2 = fma(-l21, l21, p22);
    fail = (fail == 0 && !(d2 > kPivotTol)) ? j + 2 : fail;
    sqrt_rsqrt(d2, l22, y2);
    const double a1 = fma(-q1, l21, a[1]);
    const double q2 = a1 * y2;
    const double lj1 = (lane == j) ? l11 : q1;
    const double lj2 = (lane == j + 1) ? l22 : q2;
    // ---- pending rank-2 update of the previous round on slots 2..31 (independent of the chain above) ----
#pragma unroll
    for (int k = 2; k < 32; ++k) a[k] = fma(-plj2, pc2[j + k], fma(-plj1, pc1[j + k], a[k]));
    // ---- publish the two columns ----
    if (lane >= j) LT[(col0 + j) * LTS + col0 + lane] = lj1;
    if (lane >= j + 1) LT[(col0 + j + 1) * LTS + col0 + lane] = lj2;
    if (lane == j) rd[col0 + j] = y1;
    if (lane == j + 1) rd[col0 + j + 1] = y2;
    double* c1 = colbuf + ((j >> 1) & 1) * 128;
    double* c2 = c1 + 64;
    c1[lane] = lj1;
    c2[lane] = lj2;
    __syncwarp();
    if (prog && lane == 0) *prog = j + 2;
    // ---- the two slots the next pivots need, then their shuffles ----
    const double n0 = fma(-lj2, c2[j + 2], fma(-lj1, c1[j + 2], a[2]));
    const double n1 = fma(-lj2, c2[j + 3], fma(-lj1, c1[j + 3], a[3]));
    p11 = __shfl_sync(0xffffffffu, n0, (j + 2) & 31);
    p21 = __shfl_sync(0xffffffffu, n0, (j + 3) & 31);
    p22 = __shfl_sync(0xffffffffu, n1, (j + 3) & 31);
    // window: slot k <-> column j + 2 + k; slots 2.. still lack this round's update (done in the next round)
    a[0] = n0;
    a[1] = n1;
#pragma unroll
    for (int k = 4; k < 32; ++k) a[k - 2] = a[k];
    a[30] = 0.0;
    a[31] = 0.0;
    plj1 = lj1;
    plj2 = lj2;
    pc1 = c1;
    pc2 = c2;
  }
  if (prog && fail && lane == 0) *prog = 1 << 20;
  return fail;
}

// STEPS steps of  x <- x L^-T  for one row held in a rotating register window of W slots: slot i holds column
// cbase + i on entry and column cbase + STEPS + i on exit.  The solved value of column k is handed to emit(k, value).
// LT[k*LTS + c] = L[c][k]; cbase and UNR are multiples of 2 and LTS is even, so pairs of multipliers come as one
// 16-byte broadcast load; rows of LT must be followed by readable padding (slots past the end of the row read it and
// are never emitted).
template <int W, int STEPS, int UNR, bool FAST, typename Emit>
__device__ __forceinline__ void solve_steps_rot(double (&x)[W], const double* LT,
                                                const double* rd, int cbase, Emit&& emit) {
  static_assert(STEPS % UNR == 0 && UNR % 2 == 0 && W % 2 == 0, "even windows, whole bodies");
#pragma unroll 1
  for (int kb = 0; kb < STEPS; kb += UNR) {
#pragma unroll
    for (int s = 0; s < UNR; ++s) {
      const int k = cbase + kb + s;
      const double xk = FAST ? x[s] * rd[k] : x[s] / rd[k];
      emit(k, xk);
      const double* lt = LT + k * LTS + cbase + kb;  // 16-byte aligned
      if (((s + 1) & 1) != 0) x[s + 1] = fma(-xk, lt[s + 1], x[s + 1]);
#pragma unroll
      for (int i = (s + 2) & ~1; i < W; i += 2) {
        const double2 v = *reinterpret_cast<const double2*>(lt + i);
        x[i] = fma(-xk, v.x, x[i]);
        x[i + 1] = fma(-xk, v.y, x[i + 1]);
      }
    }
#pragma unroll
    for (int i = 0; i + UNR < W; ++i) x[i] = x[i + UNR];
#pragma unroll
    for (int i = W - UNR; i < W; ++i) x[i] = 0.0;
  }
}

// Factor the 64x64 block in shared memory S (row r, col c at S[r][c]; rows/cols beyond the matrix padded with the
// identity): [L11 0; L21 L22] via chol32(A11), L21 = A21 L11^-T, A22 -= L21 L21^T, chol32(A22).  The factor is left
// in LT (transposed) with rd[k] = 1/L_kk (FAST) or L_kk.  Called by all PT threads; returns 0 or the failing 1-based
// pivot index.
template <bool FAST>
__device__ __forceinline__ int factor_block64(double (*S)[NB + 1], double* LT, double* rd,
                                              double* colbuf, volatile int* sfail) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp == 0) {
    double a[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) a[c] = S[lane][c];
    const int f = chol32_warp<FAST>(a, lane, colbuf, LT, rd, 0);
    if (lane == 0) *sfail = f;
    __syncwarp();
    if (!f) {
      // L21 = A21 L11^-T: lane r solves row 32+r; the result goes to S (row access for the SYRK) and LT
      double x[32];
#pragma unroll
      for (int c = 0; c < 32; ++c) x[c] = S[32 + lane][c];
      solve_steps_rot<32, 32, 4, FAST>(x, LT, rd, 0, [&](int k, double v) {
        S[32 + lane][k] = v;
        LT[k * LTS + 32 + lane] = v;
      });
    }
  }
  __syncthreads();
  if (*sfail) return *sfail;
  {
    // A22 -= L21 L21^T: warp w owns columns 8w..8w+7, lane r row 32+r
    constexpr int CW = 32 / (PT / 32);
    double acc[CW];
#pragma unroll
    for (int cc = 0; cc < CW; ++cc) acc[cc] = S[32 + lane][32 + warp * CW + cc];
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
      const double xr = S[32 + lane][k];
#pragma unroll
      for (int cc = 0; cc < CW; ++cc) acc[cc] = fma(-xr, LT[k * LTS + 32 + warp * CW + cc], acc[cc]);
    }
#pragma unroll
    for (int cc = 0; cc < CW; ++cc) S[32 + lane][32 + warp * CW + cc] = acc[cc];
  }
  __syncthreads();
  if (warp == 0) {
    double a[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) a[c] = S[32 + lane][32 + c];
    const int f = chol32_warp<FAST>(a, lane, colbuf, LT, rd, 32);
    if (lane == 0) *sfail = f ? 32 + f : 0;
  }
  __syncthreads();
  return *sfail;
}

__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

// Two m8n8k4 products that share B, stacked along M: rows 0..7 take (a0; d0, d1), rows 8..15 take (a1; d2, d3), each
// with the fragment layout of dmma_m8n8k4.  On sm_90 this is one DMMA.16x8x4, which runs at twice the FP64 rate of
// DMMA.8x8x4 (measured on an H100 80GB HBM3 at 400 W, eight independent accumulators per warp and eight
// 256-thread CTAs per SM: 65.9 against 33.5 TFLOP/s).
__device__ __forceinline__ void dmma_m16n8k4(double& d0, double& d1, double& d2, double& d3, double a0, double a1,
                                             double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
               : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3)
               : "d"(a0), "d"(a1), "d"(b));
}

// Two chained m16n8k4 products in one instruction (DMMA.16x8x8 on sm_90): (a0, a1; b0) is the first k-step in the
// fragment layout of dmma_m16n8k4, (a2, a3; b1) the second.
__device__ __forceinline__ void dmma_m16n8k8(double& d0, double& d1, double& d2, double& d3, double a0, double a1,
                                             double a2, double a3, double b0, double b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};\n"
               : "+d"(d0), "+d"(d1), "+d"(d2), "+d"(d3)
               : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(b0), "d"(b1));
}

// acc += As^T-tile * Bs-tile over one 64-deep chunk: warp (wm, wn) owns a 32 x 32 sub-tile, 2 x 4 m16n8k4 products per
// k-step (the fragment layout of dmma_tile_kernel in linalg.cu).  As / Bs: [k][LDT], element (k, row).  Accumulator
// acc[i][j][h] is element (wm + 8 i + lr, wn + 8 j + 2 lc + h) of the 64 x 64 tile.
__device__ __forceinline__ void tile_mma64(const double* As, const double* Bs, double (&acc)[4][4][2], int wm, int wn,
                                           int lr, int lc) {
#pragma unroll 4
  for (int kk = 0; kk < NB; kk += 4) {
    double a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = As[(kk + lc) * LDT + wm + i * 8 + lr];
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = Bs[(kk + lc) * LDT + wn + j * 8 + lr];
#pragma unroll
    for (int i = 0; i < 4; i += 2)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        dmma_m16n8k4(acc[i][j][0], acc[i][j][1], acc[i + 1][j][0], acc[i + 1][j][1], a[i], a[i + 1], b[j]);
  }
}

// acc += Vr^T Vc for one 64 x 64 Gram tile: Vr / Vc are the tile's first row / column operand, column-major with
// leading dimension (and depth) n; rows / cols of them are valid.  The operands are streamed through As / Bs
// ([NB][LDT] each) in 64-deep cp.async chunks; the CTA has kTileThreads-style 4 warps, (wm, wn, lr, lc) as tile_mma64.
__device__ __forceinline__ void gram_tile_accumulate(const double* Vr, const double* Vc, int n, int rows, int cols,
                                                     double* As, double* Bs, double (&acc)[4][4][2], int wm, int wn,
                                                     int lr, int lc) {
  const int tid = threadIdx.x;
  for (int kc = 0; kc < n; kc += NB) {
    if (kc > 0) __syncthreads();  // everybody is done with the previous chunk
    for (int e = tid; e < NB * NB; e += blockDim.x) {
      const int k = e % NB, r = e / NB;  // consecutive threads read consecutive k of one V column
      const bool okk = kc + k < n;
      const bool oka = okk && r < rows, okb = okk && r < cols;
      cp_async8(As + k * LDT + r, oka ? Vr + static_cast<size_t>(r) * n + kc + k : Vr, oka);
      cp_async8(Bs + k * LDT + r, okb ? Vc + static_cast<size_t>(r) * n + kc + k : Vc, okb);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    tile_mma64(As, Bs, acc, wm, wn, lr, lc);
  }
}

// One CTA solves L x = z (cta_forward_subst) or L^T x = z (cta_backward_subst) in place in shared memory, L the n x n
// column-major lower factor in global memory, by blocked substitution over 64-row blocks: warp 0 solves the diagonal
// block out of shared memory (D: [NB][NB + 1]), then every thread updates its rows, summing the block's products in
// ascending column order.  Every operation has a fixed order, so the result does not depend on the launch.
__device__ __forceinline__ void cta_forward_subst(const double* Ls, int n, double* z, double* D) {
  const int tid = threadIdx.x;
  for (int k0 = 0; k0 < n; k0 += NB) {
    const int nb = min(NB, n - k0);
    __syncthreads();  // the previous block's update of z and its reads of D are done
    for (int e = tid; e < NB * NB; e += blockDim.x) {
      const int rr = e % NB, c = e / NB;
      if (rr < nb && c < nb && rr >= c) D[c * (NB + 1) + rr] = Ls[static_cast<size_t>(k0 + c) * n + k0 + rr];
    }
    __syncthreads();
    if (tid < 32) {  // lane owns rows tid and tid + 32 of the block
      const int r0 = tid, r1 = tid + 32;
      double v0 = r0 < nb ? z[k0 + r0] : 0.0, v1 = r1 < nb ? z[k0 + r1] : 0.0;
      for (int j = 0; j < nb; ++j) {
        const double xj = __shfl_sync(0xffffffffu, j < 32 ? v0 : v1, j & 31) / D[j * (NB + 1) + j];
        if (r0 == j) v0 = xj;
        if (r1 == j) v1 = xj;
        if (r0 > j && r0 < nb) v0 = fma(-D[j * (NB + 1) + r0], xj, v0);
        if (r1 > j && r1 < nb) v1 = fma(-D[j * (NB + 1) + r1], xj, v1);
      }
      if (r0 < nb) z[k0 + r0] = v0;
      if (r1 < nb) z[k0 + r1] = v1;
    }
    __syncthreads();
    for (int i = k0 + nb + tid; i < n; i += blockDim.x) {  // z_i -= sum_c L[i, k0 + c] z[k0 + c]
      const double* Li = Ls + static_cast<size_t>(k0) * n + i;
      double acc = 0.0;
      for (int c = 0; c < nb; ++c) acc = fma(Li[static_cast<size_t>(c) * n], z[k0 + c], acc);
      z[i] -= acc;
    }
  }
  __syncthreads();
}

__device__ __forceinline__ void cta_backward_subst(const double* Ls, int n, double* z, double* D) {
  const int tid = threadIdx.x;
  for (int k0 = ((n - 1) / NB) * NB; k0 >= 0; k0 -= NB) {
    const int nb = min(NB, n - k0);
    __syncthreads();  // the previous block's update of z and its reads of D are done
    for (int e = tid; e < NB * NB; e += blockDim.x) {
      const int rr = e % NB, c = e / NB;
      if (rr < nb && c < nb && rr >= c) D[c * (NB + 1) + rr] = Ls[static_cast<size_t>(k0 + c) * n + k0 + rr];
    }
    __syncthreads();
    if (tid < 32) {  // L_bb^T x = z_b, last row first; lane owns rows tid and tid + 32 of the block
      const int r0 = tid, r1 = tid + 32;
      double v0 = r0 < nb ? z[k0 + r0] : 0.0, v1 = r1 < nb ? z[k0 + r1] : 0.0;
      for (int j = nb - 1; j >= 0; --j) {
        const double xj = __shfl_sync(0xffffffffu, j < 32 ? v0 : v1, j & 31) / D[j * (NB + 1) + j];
        if (r0 == j) v0 = xj;
        if (r1 == j) v1 = xj;
        if (r0 < j) v0 = fma(-D[r0 * (NB + 1) + j], xj, v0);
        if (r1 < j) v1 = fma(-D[r1 * (NB + 1) + j], xj, v1);
      }
      if (r0 < nb) z[k0 + r0] = v0;
      if (r1 < nb) z[k0 + r1] = v1;
    }
    __syncthreads();
    for (int i = tid; i < k0; i += blockDim.x) {  // z_i -= sum_c L[k0 + c, i] z[k0 + c]
      const double* Li = Ls + static_cast<size_t>(i) * n + k0;
      double acc = 0.0;
      for (int c = 0; c < nb; ++c) acc = fma(Li[c], z[k0 + c], acc);
      z[i] -= acc;
    }
  }
  __syncthreads();
}

}  // namespace
}  // namespace cmoe

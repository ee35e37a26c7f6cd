// Dense FP64 linear algebra on sm_90a: blocked right-looking Cholesky (register-resident panel factorisation, trailing
// SYRK/GEMM on the FP64 tensor pipe — mma.sync m16n8k4 DMMA; tcgen05 has no f64 kind — with one-panel look-ahead), blocked
// multi-RHS triangular solves and a single-launch flag-chained solve for one right-hand side.
//
// Replaces (reference, moe/optimal_learning/cpp/):
//   ComputeCholeskyFactorL              gpp_linear_algebra.cpp:109-148  (pivot test `> 1e-16`, returns k+1 on failure)
//   TriangularMatrixVectorSolve         gpp_linear_algebra.cpp:160-193
//   TriangularMatrixMatrixSolve         gpp_linear_algebra.cpp:203-208
//   CholeskyFactorLMatrix{Vector,Matrix}Solve  gpp_linear_algebra.hpp:220,247
//
// Layout: column-major, only the lower triangle of the factor is defined (as in the reference).
#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

#include "device_math.cuh"
#include "internal.cuh"
#include "linalg_dev.cuh"
#include "ptx_util.cuh"

namespace cmoe {

namespace {

// One launch per 64-column block step: CTA 0 factors the diagonal block and writes it back; every other CTA owns PT
// rows of the panel below it (one row per thread, held in registers), factors the (L2-resident) diagonal block
// redundantly in its own shared memory — cheaper than a second dependent launch — and then solves  X L_kk^T = A_ik
// by right-looking substitution in registers.  Failure (pivot <= 1e-16) is detected identically by every CTA; CTA 0
// records k+1 in *flag.
template <bool FAST>
__global__ void __launch_bounds__(PT) potrf_panel_kernel(double* __restrict__ A, int lda, int n, int k0, int nb,
                                                         int* __restrict__ flag, int* __restrict__ loaded) {
  extern __shared__ __align__(16) double panel_smem[];
  double* LT = panel_smem;                                                   // [NB][LTS] + NB padding
  double* colbuf = LT + NB * LTS + NB;                                       // [2][64]
  double* rd = colbuf + 128;                                                 // [NB]
  double (*S)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(rd + NB);       // [NB][NB+1]
  __shared__ int sfail;
  if (*flag != 0) return;
  const int tid = threadIdx.x;
  double* Ab = A + static_cast<size_t>(k0) * lda + k0;
  {
    const int r = tid & (NB - 1);
#pragma unroll 4
    for (int c = tid >> 6; c < NB; c += PT / NB)
      S[r][c] = (r < nb && c < nb && r >= c) ? Ab[static_cast<size_t>(c) * lda + r] : ((r == c && r >= nb) ? 1.0 : 0.0);
    for (int e = tid; e < NB * LTS + NB + 128; e += PT) LT[e] = 0.0;  // factor, its padding and the column buffers
  }
  const int myrow = k0 + nb + (static_cast<int>(blockIdx.x) - 1) * PT + tid;
  const bool valid = blockIdx.x > 0 && myrow < n;
  double x[NB];
  if (blockIdx.x > 0) {
    // issue the panel-row loads before the factorisation: their latency hides behind it
    const double* Ar = A + static_cast<size_t>(k0) * lda + myrow;
#pragma unroll
    for (int c = 0; c < NB; ++c) x[c] = (valid && c < nb) ? Ar[static_cast<size_t>(c) * lda] : 0.0;
  }
  __syncthreads();
  // CTA 0 overwrites the diagonal block in place; it must not do so before every panel CTA has read the original
  if (blockIdx.x > 0 && tid == 0) atomicAdd(loaded, 1);
  const int failed = factor_block64<FAST>(S, LT, rd, colbuf, &sfail);
  if (failed) {
    if (blockIdx.x == 0 && tid == 0) *flag = k0 + failed;
    return;
  }
  if (blockIdx.x == 0) {
    if (tid == 0) {
      const int expect = static_cast<int>(gridDim.x) - 1;
      while (atomicAdd(loaded, 0) < expect) __nanosleep(100);
    }
    __syncthreads();
    const int r = tid & (NB - 1);
#pragma unroll 4
    for (int c = tid >> 6; c < NB; c += PT / NB)
      if (r < nb && c < nb && r >= c) Ab[static_cast<size_t>(c) * lda + r] = LT[c * LTS + r];
    return;
  }
  double* Aw = A + static_cast<size_t>(k0) * lda + myrow;
  auto emit = [&](int k, double v) {
    if (valid && k < nb) Aw[static_cast<size_t>(k) * lda] = v;
  };
  // first half with the full window, second half with a window of the 32 columns that are left
  solve_steps_rot<NB, NB / 2, 4, FAST>(x, LT, rd, 0, emit);
  double xh[NB / 2];
#pragma unroll
  for (int i = 0; i < NB / 2; ++i) xh[i] = x[i];
  solve_steps_rot<NB / 2, NB / 2, 4, FAST>(xh, LT, rd, NB / 2, emit);
}

// --------------------------------------------------------------------------------------------------------------
// DMMA tile update:  C(64x64) -= A(64xK) * B(64xK)^T  with A, B, C blocks of one matrix, lower-triangular tile grid
// (row tiles x col_tiles; tiles above the diagonal exit).  The operand panel is the `kdepth` columns starting at k0
// (in chunks of NB); the trailing matrix starts right after it.  Two uses:
//   * inner update of a 64-column step (kdepth = nb <= 64), restricted to the columns still inside the outer panel;
//   * look-ahead update of the next outer panel's columns (kdepth = 256): many small tiles (one wave, 3 CTAs/SM)
//     finish sooner than a few 128x128 ones, and this update sits on the critical path of the chain.
// 4 warps, each owning a 32x32 sub-tile = 4x4 m8n8k4 fragments.
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) dmma_tile_kernel(double* __restrict__ A, int lda, int n, int k0, int nb,
                                                        int col_tiles, const int* __restrict__ flag, int kdepth) {
  extern __shared__ double smem[];
  if (*flag != 0) return;
  double* As = smem;
  double* Bs = smem + NB * LDT;
  const int t0 = k0 + max(nb, kdepth);  // first row/col of the trailing matrix
  const int ti = blockIdx.x / col_tiles, tj = blockIdx.x % col_tiles;
  if (tj > ti) return;
  const int row0 = t0 + ti * NB, col0 = t0 + tj * NB;
  const int rows = min(NB, n - row0), cols = min(NB, n - col0);
  const double* Asrc = A + static_cast<size_t>(k0) * lda + row0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  // accumulate +A B^T on top of -C: the epilogue is then a plain store of -acc, and the C tile is fetched while the
  // operand tiles land (the launch is latency-bound: the global round trips must overlap)
  double acc[4][4][2];
  double* Cg = A + static_cast<size_t>(col0) * lda + row0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h;
        acc[i][j][h] = (r < rows && c < cols) ? -Cg[static_cast<size_t>(c) * lda + r] : 0.0;
      }
  }
  const int nchunks = max(1, kdepth / NB);
  const int kw = (kdepth > nb) ? NB : nb;  // columns per chunk
  for (int ch = 0; ch < nchunks; ++ch) {
    if (ch > 0) __syncthreads();  // everybody is done with the previous chunk's tiles
    const double* Ac = Asrc + static_cast<size_t>(ch) * NB * lda;
    const double* Bc = A + static_cast<size_t>(k0 + ch * NB) * lda + col0;
    for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
      const int r = e % NB, c = e / NB;
      const bool oka = r < rows && c < kw, okb = r < cols && c < kw;
      cp_async8(As + c * LDT + r, oka ? Ac + static_cast<size_t>(c) * lda + r : Ac, oka);
      cp_async8(Bs + c * LDT + r, okb ? Bc + static_cast<size_t>(c) * lda + r : Bc, okb);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
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
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = wm + i * 8 + lr;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = wn + j * 8 + lc * 2 + h;
        if (r < rows && c < cols) Cg[static_cast<size_t>(c) * lda + r] = -acc[i][j][h];
      }
  }
}

// --------------------------------------------------------------------------------------------------------------
// Outer trailing update of the two-level blocked Cholesky:
//     C(128x128 tile of the trailing matrix, lower tiles only) -= A_rows(128 x W) * A_cols(128 x W)^T
// 8 warps (4 x 2), each a 32x64 sub-tile = 4x8 m8n8k4 DMMA fragments (64 FP64 accumulators per thread); operands are
// streamed in K-chunks of 16 through a 3-stage cp.async pipeline; the accumulator tile is staged through shared memory
// so that the read-modify-write of C is fully coalesced.
// --------------------------------------------------------------------------------------------------------------
constexpr int GT = 128;       // tile edge
constexpr int GK = 16;        // K chunk
constexpr int GST = 3;        // pipeline stages
constexpr int GLD = GT + 4;   // 132 = 4 (mod 16): conflict-free fragment loads

constexpr int GTHREADS = 512;  // 16 warps = 4 x 4 warp tiles of 32 x 32 (4 warps per scheduler keep the DMMA pipe fed)

// Trailing update A[t0:, t0:] -= P P^T, P = A[t0:, p0:p0+W], restricted to the column tiles [tj_lo, tj_hi) of the
// lower-triangular 128x128 tile grid.  Persistent: CTA b works on tiles b, b + gridDim.x, ... (column-major tile
// order), so a launch can be confined to a subset of the SMs while the next panel's factorisation uses the others.
__global__ void __launch_bounds__(GTHREADS, 1) dmma_gemm_kernel(double* __restrict__ A, int lda, int n, int p0, int W,
                                                                int tj_lo, int tj_hi, const int* __restrict__ flag) {
  extern __shared__ double gsm[];
  if (*flag != 0) return;
  const int t0 = p0 + W;
  const int tiles = (n - t0 + GT - 1) / GT;
  tj_hi = min(tj_hi, tiles);
  // tiles in column tj: row tiles tj .. tiles-1
  int total = 0;
  for (int tj = tj_lo; tj < tj_hi; ++tj) total += tiles - tj;
  const int tid = threadIdx.x;
  const int nchunks = W / GK;
  const int warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 32;
  const int lr = lane >> 2, lc = lane & 3;
  double* As = gsm;                    // [GST][GK][GLD]
  double* Bs = gsm + GST * GK * GLD;   // [GST][GK][GLD]
  for (int b = blockIdx.x; b < total; b += gridDim.x) {
    int tj = tj_lo, rem = b;
    while (rem >= tiles - tj) {
      rem -= tiles - tj;
      ++tj;
    }
    const int ti = tj + rem;
    const int row0 = t0 + ti * GT, col0 = t0 + tj * GT;
    const int rows = min(GT, n - row0), cols = min(GT, n - col0);
    const double* Ag = A + static_cast<size_t>(p0) * lda + row0;
    const double* Bg = A + static_cast<size_t>(p0) * lda + col0;

    auto load_chunk = [&](int kc, int stage) {
      double* as = As + stage * GK * GLD;
      double* bs = Bs + stage * GK * GLD;
#pragma unroll
      for (int e = tid; e < GT * GK; e += GTHREADS) {
        const int m = e % GT, k = e / GT;
        cp_async8(as + k * GLD + m, m < rows ? Ag + static_cast<size_t>(kc * GK + k) * lda + m : Ag, m < rows);
        cp_async8(bs + k * GLD + m, m < cols ? Bg + static_cast<size_t>(kc * GK + k) * lda + m : Bg, m < cols);
      }
    };

    double acc[4][4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

#pragma unroll
    for (int st = 0; st < GST - 1; ++st) {
      if (st < nchunks) load_chunk(st, st);
      cp_async_commit();
    }
    for (int kc = 0; kc < nchunks; ++kc) {
      cp_async_wait<GST - 2>();
      __syncthreads();
      const int nxt = kc + GST - 1;
      if (nxt < nchunks) load_chunk(nxt, nxt % GST);
      cp_async_commit();
      const double* as = As + (kc % GST) * GK * GLD;
      const double* bs = Bs + (kc % GST) * GK * GLD;
#pragma unroll
      for (int kk = 0; kk < GK; kk += 4) {
        double a[4], bb[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = as[(kk + lc) * GLD + wm + i * 8 + lr];
#pragma unroll
        for (int j = 0; j < 4; ++j) bb[j] = bs[(kk + lc) * GLD + wn + j * 8 + lr];
#pragma unroll
        for (int i = 0; i < 4; i += 2)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            dmma_m16n8k4(acc[i][j][0], acc[i][j][1], acc[i + 1][j][0], acc[i + 1][j][1], a[i], a[i + 1], bb[j]);
      }
    }
    cp_async_wait<0>();
    __syncthreads();
    // stage the accumulator tile: Cs[c][r] (column-major, ld GLD), then coalesced C -= Cs
    double* Cs = gsm;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) Cs[(wn + j * 8 + lc * 2 + h) * GLD + wm + i * 8 + lr] = acc[i][j][h];
    __syncthreads();
    double* Cg = A + static_cast<size_t>(col0) * lda + row0;
    for (int e = tid; e < GT * GT; e += GTHREADS) {
      const int r = e % GT, c = e / GT;
      if (r < rows && c < cols) {
        double* dst = Cg + static_cast<size_t>(c) * lda + r;
        *dst = *dst - Cs[c * GLD + r];
      }
    }
    __syncthreads();  // Cs aliases the pipeline buffers of the next tile
  }
}

// --------------------------------------------------------------------------------------------------------------
// Blocked triangular solve, one CTA per slab of 32 right-hand sides.
//   TRANS = false: X <- L^-1 X (block rows top-down);  TRANS = true: X <- L^-T X (bottom-up).
// Per block row: acc = sum_j Ltile(k,j) * X_j via 32x32x32 shared-memory products, then the 32x32 diagonal block is
// solved by column-oriented substitution (the operation order of the reference's TriangularMatrixVectorSolve, so
// small integer systems come out exact), one barrier per eliminated unknown.
// --------------------------------------------------------------------------------------------------------------
template <bool TRANS>
__global__ void __launch_bounds__(256) trsm_kernel(const double* __restrict__ L, int n, double* __restrict__ X,
                                                   int ldx, int nrhs) {
  constexpr int T = kTrsmNB;
  __shared__ double Ls[T][T + 1];
  __shared__ double Xs[T][T + 1];
  __shared__ double Ys[2][T];
  const int col0 = blockIdx.x * T;
  const int tid = threadIdx.x;
  const int c = tid & 31, rg = tid >> 5;  // output column, row group (rows rg + 8*i)
  const int lm = tid & 31, lq = tid >> 5; // load mapping: fast index, slow index (+8*i)
  const int nbk = (n + T - 1) / T;
  const bool col_ok = (col0 + c) < nrhs;

  for (int step = 0; step < nbk; ++step) {
    const int k = TRANS ? (nbk - 1 - step) : step;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    const int jbeg = TRANS ? (k + 1) : 0, jend = TRANS ? nbk : k;
    for (int j = jbeg; j < jend; ++j) {
      // Ls[r][m] = (op(L))(k*T + r, j*T + m)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int slow = lq + 8 * i;
        if (!TRANS) {
          const int r = k * T + lm, m = j * T + slow;  // L(r, m), contiguous in r
          Ls[lm][slow] = (r < n && m < n) ? L[static_cast<size_t>(m) * n + r] : 0.0;
        } else {
          const int m = j * T + lm, r = k * T + slow;  // L(m, r), contiguous in m
          Ls[slow][lm] = (r < n && m < n) ? L[static_cast<size_t>(r) * n + m] : 0.0;
        }
        const int xr = j * T + lm, xc = col0 + slow;
        Xs[lm][slow] = (xr < n && xc < nrhs) ? X[static_cast<size_t>(xc) * ldx + xr] : 0.0;
      }
      __syncthreads();
#pragma unroll 8
      for (int m = 0; m < T; ++m) {
        const double xv = Xs[m][c];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] += Ls[rg + 8 * i][m] * xv;
      }
      __syncthreads();
    }
    // diagonal block L_kk -> Ls (lower part; identity on the padding), right-hand side minus products -> registers
    double val[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = rg + 8 * i;
      const int xr = k * T + r;
      const double bval = (xr < n && col_ok) ? X[static_cast<size_t>(col0 + c) * ldx + xr] : 0.0;
      val[i] = bval - acc[i];
      const int slow = lq + 8 * i;  // column of the block
      const int gr = k * T + lm, gc = k * T + slow;
      double lv = 0.0;
      if (gr < n && gc < n) {
        if (lm >= slow) lv = L[static_cast<size_t>(gc) * n + gr];
      } else if (lm == slow) {
        lv = 1.0;
      }
      Ls[lm][slow] = lv;
    }
    __syncthreads();
    for (int rr = 0; rr < T; ++rr) {
      const int r = TRANS ? (T - 1 - rr) : rr;
      if (rg == (r & 7)) {
        const int i = r >> 3;
        double y = 0.0;
#pragma unroll
        for (int ii = 0; ii < 4; ++ii)
          if (ii == i) {
            y = val[ii] / Ls[r][r];
            val[ii] = y;
          }
        Ys[rr & 1][c] = y;
      }
      __syncthreads();
      const double y = Ys[rr & 1][c];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = rg + 8 * i;
        if (!TRANS) {
          if (row > r) val[i] = val[i] - y * Ls[row][r];
        } else {
          if (row < r) val[i] = val[i] - Ls[r][row] * y;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int xr = k * T + rg + 8 * i;
      if (xr < n && col_ok) X[static_cast<size_t>(col0 + c) * ldx + xr] = val[i];
    }
    __syncthreads();  // make this block row visible to the next iterations of this CTA
  }
}

int g_launches = 0;

// --------------------------------------------------------------------------------------------------------------
// Few right-hand sides, large n (the K^-1 y solve of a big fit): the slab kernel above would run on one SM.
// Instead march over 128-wide diagonal blocks: a single CTA solves the block (column-oriented substitution out of
// shared memory), then a grid-wide GEMV removes its contribution from the remaining rows — L is streamed exactly once.
// --------------------------------------------------------------------------------------------------------------
constexpr int VB = 128;

// Solves the VB x VB diagonal block for one right-hand side.  Four 32-unknown sub-blocks in sequence: the owning warp
// solves its sub-block out of registers (lane i holds unknown i and its row of the 32x32 triangle; each solved unknown
// is broadcast by shuffle — no block barrier inside the recurrence), then the warps that are still waiting fold the 32
// new unknowns into their right-hand sides.  Four barriers per block instead of one per unknown.
template <bool TRANS>
__global__ void __launch_bounds__(VB) trsv_diag_kernel(const double* __restrict__ L, int n, int b0,
                                                       double* __restrict__ x) {
  extern __shared__ double S[];  // [VB][VB+1] lower block of L (row r, col c at S[r*(VB+1)+c])
  __shared__ double xs[VB];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int nb = min(VB, n - b0);
#pragma unroll 8
  for (int c = 0; c < VB; ++c) {
    double v = 0.0;
    if (t < nb && c <= t) v = L[static_cast<size_t>(b0 + c) * n + b0 + t];
    S[t * (VB + 1) + c] = v;
  }
  double v = (t < nb) ? x[b0 + t] : 0.0;
  const double rd = (t < nb) ? 1.0 / L[static_cast<size_t>(b0 + t) * n + b0 + t] : 0.0;  // off the critical chain
  __syncthreads();
#pragma unroll 1
  for (int sb = 0; sb < VB / 32; ++sb) {
    const int q = TRANS ? (VB / 32 - 1 - sb) : sb;
    if (warp == q) {
      double lr[32];  // forward: L[32q+lane][32q+j] (j < lane);  backward: L[32q+j][32q+lane] (j > lane)
#pragma unroll
      for (int j = 0; j < 32; ++j)
        lr[j] = TRANS ? S[(32 * q + j) * (VB + 1) + 32 * q + lane] : S[(32 * q + lane) * (VB + 1) + 32 * q + j];
#pragma unroll
      for (int st = 0; st < 32; ++st) {
        const int c = TRANS ? (31 - st) : st;
        const double xc = __shfl_sync(0xffffffffu, v * rd, c);
        if (lane == c) v = xc;
        if (TRANS ? (lane < c) : (lane > c)) v = v - xc * lr[c];
      }
      xs[32 * q + lane] = v;
    }
    __syncthreads();
    if (TRANS ? (warp < q) : (warp > q)) {
#pragma unroll 8
      for (int c = 0; c < 32; ++c) {
        const double l = TRANS ? S[(32 * q + c) * (VB + 1) + t] : S[t * (VB + 1) + 32 * q + c];
        v = v - xs[32 * q + c] * l;
      }
    }
  }
  if (t < nb) x[b0 + t] = v;
}

// forward: x[i] -= sum_c L[i, b0+c] x[b0+c] for i >= b0+nb.  CTA = 64 rows x 4 column quarters (coalesced down the
// columns, 4-way unrolled for memory-level parallelism), quarters combined through shared memory in a fixed order.
__global__ void __launch_bounds__(256) trsv_update_fwd_kernel(const double* __restrict__ L, int n, int b0, int nb,
                                                              double* __restrict__ x) {
  __shared__ double xs[VB];
  __shared__ double part[4][64];
  if (threadIdx.x < nb) xs[threadIdx.x] = x[b0 + threadIdx.x];
  __syncthreads();
  const int rl = threadIdx.x & 63, qd = threadIdx.x >> 6;
  const int i = b0 + nb + blockIdx.x * 64 + rl;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  if (i < n) {
    const int cbeg = qd * (VB / 4), cend = min(nb, cbeg + VB / 4);
    const double* col = L + static_cast<size_t>(b0) * n + i;
    int c = cbeg;
    for (; c + 3 < cend; c += 4) {
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[u] = fma(col[static_cast<size_t>(c + u) * n], xs[c + u], acc[u]);
    }
    for (; c < cend; ++c) acc[0] = fma(col[static_cast<size_t>(c) * n], xs[c], acc[0]);
  }
  part[qd][rl] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
  __syncthreads();
  if (qd == 0 && i < n) x[i] = x[i] - ((part[0][rl] + part[1][rl]) + (part[2][rl] + part[3][rl]));
}

// backward: x[i] -= sum_r L[b0+r, i] x[b0+r] for i < b0 ; one warp per column i (contiguous read), shuffle reduce
__global__ void __launch_bounds__(256) trsv_update_bwd_kernel(const double* __restrict__ L, int n, int b0, int nb,
                                                              double* __restrict__ x) {
  __shared__ double xs[VB];
  if (threadIdx.x < nb) xs[threadIdx.x] = x[b0 + threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= b0) return;
  const double* col = L + static_cast<size_t>(i) * n + b0;
  double acc = 0.0;
  for (int r = lane; r < nb; r += 32) acc = fma(col[r], xs[r], acc);
  acc = warp_sum(acc);
  if (lane == 0) x[i] = x[i] - acc;
}

// --------------------------------------------------------------------------------------------------------------
// Single-launch triangular solve for one right-hand side ("chained" trsv): one CTA per block of VB unknowns, all
// co-resident.  CTA b accumulates  sum_j L_bj x_j  over the blocks it depends on as soon as each x_j is published
// (ready[j], release/acquire through L2), then solves its diagonal block with the warp-level recurrence and publishes
// x_b.  The critical path per block is one 128x128 matrix-vector product + one diagonal solve instead of two dependent
// kernel launches, and the off-critical products run ahead while the CTA waits.  Deadlock-free: CTA b only waits on
// blocks that wait on strictly fewer blocks, and every CTA is resident (grid <= #SMs, checked by the host).  A bounded
// spin turns a lost dependency into an error code instead of a hang.
// --------------------------------------------------------------------------------------------------------------
constexpr int CT = 512;  // threads of the chained solver

__device__ __forceinline__ void wait_ready(const int* flag, int* abort_flag) {
  for (unsigned spins = 0; ld_acquire(flag) == 0; ++spins) {
    if (spins > (1u << 22)) {  // ~1 s: far beyond any legitimate wait
      atomicExch(abort_flag, 1);
      break;
    }
    __nanosleep(20);
  }
}

template <bool TRANS>
__global__ void __launch_bounds__(CT) trsv_chain_kernel(const double* __restrict__ L, int n, const double* __restrict__ rhs,
                                                        double* __restrict__ xout, int* __restrict__ ready,
                                                        int* __restrict__ abort_flag, int nblk) {
  extern __shared__ double S[];  // [VB][VB+1] lower diagonal block (row r, col c at S[r*(VB+1)+c])
  __shared__ double xs[VB];
  __shared__ double part[CT / VB][VB];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int b = TRANS ? (nblk - 1 - static_cast<int>(blockIdx.x)) : static_cast<int>(blockIdx.x);
  const int b0 = b * VB, nb = min(VB, n - b0);
  // diagonal block: thread (r, quarter) loads 32 columns of its row
  {
    const int r = t & (VB - 1), q = t >> 7;
#pragma unroll 8
    for (int c = q * 32; c < q * 32 + 32; ++c) {
      double v = 0.0;
      if (r < nb && c <= r) v = L[static_cast<size_t>(b0 + c) * n + b0 + r];
      S[r * (VB + 1) + c] = v;
    }
  }
  double v = 0.0;
  if (!TRANS) {
    // row r = t & 127, column quarter q of every dependency block: coalesced down the columns
    const int r = t & (VB - 1), q = t >> 7;
    double acc = 0.0;
    for (int j = 0; j < b; ++j) {
      wait_ready(ready + j, abort_flag);
      const double* col = L + static_cast<size_t>(j * VB + q * 32) * n + b0 + r;
      const double* xj = xout + j * VB + q * 32;
      if (r < nb) {
#pragma unroll 8
        for (int c = 0; c < 32; ++c) acc = fma(col[static_cast<size_t>(c) * n], __ldcg(xj + c), acc);
      }
    }
    part[q][r] = acc;
    __syncthreads();
    if (t < VB) v = (t < nb) ? rhs[b0 + t] - ((part[0][t] + part[1][t]) + (part[2][t] + part[3][t])) : 0.0;
  } else {
    // warp w owns columns 8w..8w+7 of this block; lanes run down the rows of every dependency block (contiguous)
    double acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.0;
    for (int j = nblk - 1; j > b; --j) {
      wait_ready(ready + j, abort_flag);
      const int j0 = j * VB, jn = min(VB, n - j0);
      double xr[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) xr[k] = (lane + 32 * k < jn) ? __ldcg(xout + j0 + lane + 32 * k) : 0.0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = warp * 8 + i;
        if (c < nb) {
          const double* col = L + static_cast<size_t>(b0 + c) * n + j0;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (lane + 32 * k < jn) acc[i] = fma(col[lane + 32 * k], xr[k], acc[i]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const double sum = warp_sum(acc[i]);
      if (lane == 0) part[0][warp * 8 + i] = sum;
    }
    __syncthreads();
    if (t < VB) v = (t < nb) ? rhs[b0 + t] - part[0][t] : 0.0;
  }
  const double rd = (t < nb) ? 1.0 / L[static_cast<size_t>(b0 + t) * n + b0 + t] : 0.0;
  __syncthreads();  // S complete
  // warp-level solve of the diagonal block by the first VB threads (see trsv_diag_kernel); all threads hit the barriers
#pragma unroll 1
  for (int sb = 0; sb < VB / 32; ++sb) {
    const int q = TRANS ? (VB / 32 - 1 - sb) : sb;
    if (t < VB && warp == q) {
      double lr[32];
#pragma unroll
      for (int j = 0; j < 32; ++j)
        lr[j] = TRANS ? S[(32 * q + j) * (VB + 1) + 32 * q + lane] : S[(32 * q + lane) * (VB + 1) + 32 * q + j];
#pragma unroll
      for (int st = 0; st < 32; ++st) {
        const int c = TRANS ? (31 - st) : st;
        const double xc = __shfl_sync(0xffffffffu, v * rd, c);
        if (lane == c) v = xc;
        if (TRANS ? (lane < c) : (lane > c)) v = v - xc * lr[c];
      }
      xs[32 * q + lane] = v;
    }
    __syncthreads();
    if (t < VB && (TRANS ? (warp < q) : (warp > q))) {
#pragma unroll 8
      for (int c = 0; c < 32; ++c) {
        const double l = TRANS ? S[(32 * q + c) * (VB + 1) + t] : S[t * (VB + 1) + 32 * q + c];
        v = v - xs[32 * q + c] * l;
      }
    }
  }
  if (t < nb) xout[b0 + t] = v;
  __threadfence();
  __syncthreads();
  if (t == 0) st_release(ready + b, 1);
}

// returns false if the chained kernel cannot be used (more blocks than SMs) or gave up waiting (its CTAs could not
// all become resident, e.g. other streams occupy the device): x is untouched in that case and the caller falls back
bool trsv_chained(const double* L, int n, double* x, bool trans, cudaStream_t s) {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int nblk = (n + VB - 1) / VB;
  if (nblk > sms) return false;
  const size_t smem = static_cast<size_t>(VB) * (VB + 1) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(trsv_chain_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  CMOE_CUDA(cudaFuncSetAttribute(trsv_chain_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  DevBuf<int> flags(nblk + 1);
  DevBuf<double> out(n);
  CMOE_CUDA(cudaMemsetAsync(flags.p, 0, (nblk + 1) * sizeof(int), s));
  if (trans) {
    trsv_chain_kernel<true><<<nblk, CT, smem, s>>>(L, n, x, out.p, flags.p, flags.p + nblk, nblk);
  } else {
    trsv_chain_kernel<false><<<nblk, CT, smem, s>>>(L, n, x, out.p, flags.p, flags.p + nblk, nblk);
  }
  count_launch();
  CMOE_CUDA(cudaGetLastError());
  int aborted = 0;
  CMOE_CUDA(cudaMemcpyAsync(&aborted, flags.p + nblk, sizeof(int), cudaMemcpyDeviceToHost, s));
  CMOE_CUDA(cudaStreamSynchronize(s));
  if (aborted) return false;
  CMOE_CUDA(cudaMemcpyAsync(x, out.p, static_cast<size_t>(n) * sizeof(double), cudaMemcpyDeviceToDevice, s));
  CMOE_CUDA(cudaStreamSynchronize(s));  // scratch is freed on return
  return true;
}

void trsv_blocked(const double* L, int n, double* x, bool trans, cudaStream_t s) {
  const size_t smem = static_cast<size_t>(VB) * (VB + 1) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(trsv_diag_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  CMOE_CUDA(cudaFuncSetAttribute(trsv_diag_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  const int nblk = (n + VB - 1) / VB;
  for (int step = 0; step < nblk; ++step) {
    const int b = trans ? (nblk - 1 - step) : step;
    const int b0 = b * VB, nb = min(VB, n - b0);
    if (!trans) {
      trsv_diag_kernel<false><<<1, VB, smem, s>>>(L, n, b0, x);
      const int rest = n - b0 - nb;
      if (rest > 0) trsv_update_fwd_kernel<<<(rest + 63) / 64, 256, 0, s>>>(L, n, b0, nb, x);
    } else {
      trsv_diag_kernel<true><<<1, VB, smem, s>>>(L, n, b0, x);
      if (b0 > 0) trsv_update_bwd_kernel<<<(b0 + 7) / 8, 256, 0, s>>>(L, n, b0, nb, x);
    }
    g_launches += 2;
  }
  CMOE_CUDA(cudaGetLastError());
}



}  // namespace

int launches_issued() { return g_launches; }
// run-time switches (initialised from the environment, changeable through cmoe_set_option — the tests flip them to
// cover both paths in one process)
namespace {
int& opt_legacy() {
  static int v = [] {
    const char* e = std::getenv("CMOE_LEGACY_LINALG");
    return (e && e[0] == '1') ? 1 : 0;
  }();
  return v;
}
int& opt_cov_tma() {
  static int v = [] {
    const char* e = std::getenv("CMOE_COV_TMA");
    return (e && e[0] == '1') ? 1 : 0;
  }();
  return v;
}
int& opt_members_in_flight() {
  static int v = 0;
  return v;
}
}  // namespace
bool legacy_linalg() { return opt_legacy() != 0; }
int ensemble_members_in_flight() { return opt_members_in_flight(); }
bool cov_tma_enabled() { return opt_cov_tma() != 0; }
int set_option(const char* name, int value) {
  const std::string n(name ? name : "");
  if (n == "legacy_linalg") {
    opt_legacy() = value ? 1 : 0;
  } else if (n == "cov_tma") {
    opt_cov_tma() = value ? 1 : 0;
  } else if (n == "ensemble_members_in_flight") {
    if (value < 0) return -1;
    opt_members_in_flight() = value;
  } else {
    return -1;
  }
  return 0;
}
void count_launch(int n) { g_launches += n; }

// Side stream + events for the look-ahead schedule, created once per host thread and device.
struct LookaheadCtx {
  int device = -1;
  cudaStream_t side = nullptr;
  std::vector<cudaEvent_t> chain_done, rest_done;
  void ensure(int dev, size_t panels) {
    if (device != dev) {
      // contexts of other devices are left to process teardown; a handle is bound to one device for its lifetime
      device = dev;
      side = nullptr;
      chain_done.clear();
      rest_done.clear();
    }
    if (!side) CMOE_CUDA(cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking));
    while (chain_done.size() < panels) {
      cudaEvent_t a, b;
      CMOE_CUDA(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
      CMOE_CUDA(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
      chain_done.push_back(a);
      rest_done.push_back(b);
    }
  }
};

// Right-looking blocked Cholesky with two-level blocking and one-panel look-ahead:
//   for every 256-column outer panel: four 64-column steps (fused diagonal factorisation + panel solve, then the
//   DMMA update of the columns still inside the outer panel), then the 128x128-tiled DMMA trailing update, split into
//   (a) the next outer panel's columns — on the main stream, the factorisation chain continues as soon as it is done —
//   and (b) everything to the right of it, on a side stream confined to a subset of the SMs so that it overlaps the
//   next panel's latency-bound chain.  (a) of panel p waits for (b) of panel p-1 (both touch the same columns).
void potrf_lower(double* A, int n, int* flag, cudaStream_t s) {
  if (potrf_lower_coop(A, n, flag, s)) return;
  constexpr int W = 256;  // outer panel width (4 inner blocks of NB)
  const size_t smem = 2 * NB * LDT * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(dmma_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem)));
  const size_t smem_panel = (static_cast<size_t>(NB) * LTS + NB + 128 + NB + NB * (NB + 1)) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(potrf_panel_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_panel)));
  CMOE_CUDA(cudaFuncSetAttribute(potrf_panel_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_panel)));
  const size_t smem_gemm = static_cast<size_t>(GT) * GLD * sizeof(double);  // >= 2*GST*GK*GLD doubles as well
  static_assert(GT * GLD >= 2 * GST * GK * GLD, "accumulator staging must cover the pipeline buffers");
  CMOE_CUDA(cudaFuncSetAttribute(dmma_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem_gemm)));
  CMOE_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), s));
  const int nsteps = (n + NB - 1) / NB;
  DevBuf<int> loaded_buf(nsteps);  // one arrival counter per block step
  int* loaded = loaded_buf.p;
  CMOE_CUDA(cudaMemsetAsync(loaded, 0, nsteps * sizeof(int), s));
  const int fast_chain = n > 4 * NB ? 1 : 0;  // small systems keep IEEE sqrt / divide (exact known-answer cases)
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int npanels = (n + W - 1) / W;
  const bool lookahead = npanels >= 4;  // below ~1000 rows the trailing updates are too small to be worth overlapping
  static thread_local LookaheadCtx ctx;
  if (lookahead) ctx.ensure(dev, npanels);
  const int rest_ctas = std::max(32, sms - 40);  // SMs left to the chain kernels while (b) runs
  int last_rest = -1;
  for (int p0 = 0, pi = 0; p0 < n; p0 += W, ++pi) {
    const int pw = min(W, n - p0);         // this panel's width
    const int pend = p0 + pw;
    for (int k0 = p0; k0 < pend; k0 += NB) {
      const int nb = min(NB, n - k0);
      const int rem = n - k0 - nb;
      const int row_tiles = (rem + NB - 1) / NB;
      const int panel_ctas = 1 + (rem + PT - 1) / PT;
      if (fast_chain) {
        potrf_panel_kernel<true><<<panel_ctas, PT, smem_panel, s>>>(A, n, n, k0, nb, flag, loaded + k0 / NB);
      } else {
        potrf_panel_kernel<false><<<panel_ctas, PT, smem_panel, s>>>(A, n, n, k0, nb, flag, loaded + k0 / NB);
      }
      count_launch();
      // inner trailing update: only the columns that still belong to this outer panel
      const int col_tiles = (pend - (k0 + nb) + NB - 1) / NB;
      if (rem > 0 && col_tiles > 0) {
        dmma_tile_kernel<<<row_tiles * col_tiles, 128, smem, s>>>(A, n, n, k0, nb, col_tiles, flag, nb);
        count_launch();
      }
    }
    const int rem = n - pend;
    if (rem > 0 && pw == W) {
      const int tiles = (rem + GT - 1) / GT;
      constexpr int kNextTiles = W / GT;  // column tiles of the next outer panel
      if (!lookahead || tiles <= kNextTiles) {
        if (last_rest >= 0) {
          CMOE_CUDA(cudaStreamWaitEvent(s, ctx.rest_done[last_rest], 0));
          last_rest = -1;
        }
        dmma_gemm_kernel<<<tiles * (tiles + 1) / 2, GTHREADS, smem_gemm, s>>>(A, n, n, p0, W, 0, tiles, flag);
        count_launch();
      } else {
        CMOE_CUDA(cudaEventRecord(ctx.chain_done[pi], s));
        if (last_rest >= 0) CMOE_CUDA(cudaStreamWaitEvent(s, ctx.rest_done[last_rest], 0));
        // (a): one wave of 64x64 tiles, K = 256 in four chunks — finishes in a fraction of the time a few 128x128
        // CTAs need, and this update sits on the critical path of the chain
        const int nrt = (rem + NB - 1) / NB, nct = std::min(W / NB, nrt);
        dmma_tile_kernel<<<nrt * nct, 128, smem, s>>>(A, n, n, p0, NB, nct, flag, W);
        count_launch();
        CMOE_CUDA(cudaStreamWaitEvent(ctx.side, ctx.chain_done[pi], 0));
        const int rt = tiles - kNextTiles;
        const int rest_total = rt * (rt + 1) / 2;
        dmma_gemm_kernel<<<std::min(rest_total, rest_ctas), GTHREADS, smem_gemm, ctx.side>>>(A, n, n, p0, W, kNextTiles,
                                                                                            tiles, flag);
        count_launch();
        CMOE_CUDA(cudaEventRecord(ctx.rest_done[pi], ctx.side));
        last_rest = pi;
      }
    }
  }
  if (last_rest >= 0) CMOE_CUDA(cudaStreamWaitEvent(s, ctx.rest_done[last_rest], 0));
  CMOE_CUDA(cudaGetLastError());
  CMOE_CUDA(cudaStreamSynchronize(s));  // the counter scratch is freed on return
}

void trsm_lower(const double* L, int n, double* X, int ldx, int nrhs, bool trans, cudaStream_t s) {
  if (n == 0 || nrhs == 0) return;
  if (nrhs <= 4 && n >= 1024) {
    for (int r = 0; r < nrhs; ++r) {
      double* xr = X + static_cast<size_t>(r) * ldx;
      if (!legacy_linalg() && trsv_coop(L, n, xr, trans, s)) continue;
      if (!trsv_chained(L, n, xr, trans, s)) trsv_blocked(L, n, xr, trans, s);
    }
    return;
  }
  trsm_lower_blocked(L, n, X, ldx, nrhs, trans, s);
}

void trsm_lower_blocked(const double* L, int n, double* X, int ldx, int nrhs, bool trans, cudaStream_t s) {
  if (n == 0 || nrhs == 0) return;
  const int grid = (nrhs + kTrsmNB - 1) / kTrsmNB;
  if (trans) {
    trsm_kernel<true><<<grid, 256, 0, s>>>(L, n, X, ldx, nrhs);
  } else {
    trsm_kernel<false><<<grid, 256, 0, s>>>(L, n, X, ldx, nrhs);
  }
  count_launch();
  CMOE_CUDA(cudaGetLastError());
}

void potrs_lower(const double* L, int n, double* X, int ldx, int nrhs, cudaStream_t s) {
  if (nrhs <= 4 && n >= 1024 && !legacy_linalg()) {
    // few right-hand sides on a large factor: both triangular solves of a column back to back (one synchronisation);
    // a column the cooperative kernel declines (it leaves the right-hand side untouched) takes the two-step path
    for (int r = 0; r < nrhs; ++r) {
      double* col = X + static_cast<size_t>(r) * ldx;
      if (trsv_coop_pair(L, n, col, s)) continue;
      trsm_lower(L, n, col, ldx, 1, false, s);
      trsm_lower(L, n, col, ldx, 1, true, s);
    }
    return;
  }
  trsm_lower(L, n, X, ldx, nrhs, false, s);
  trsm_lower(L, n, X, ldx, nrhs, true, s);
}

}  // namespace cmoe

// Lower-confidence-bound batch selection in one device call (DESIGN.md K13).
//
// Replaces (reference): lower_confidence_bound_optimization, moe/optimal_learning/python/cpp_wrappers/
// lower_confidence_bound.py:52-80, with what its calls do underneath: ComputeMeanOfPoints (gpp_math.cpp:662), the
// [0,0] entry of GetCholVarWrapper (gpp_python_gaussian_process.cpp:156-175) per candidate, and one AddPointsToGP refit
// (gpp_math.cpp:1699-1718) per further point.
//
//   screen      per chunk of candidates in the handle's sampling workspace: V = L^-1 K(X, x) (build_mix_covariance +
//               one blocked forward solve), sigma0^2(x) = k(x,x) - |V(x)|^2 (lcb_screen_kernel), mu = posterior_mean_points
//   selection   first point = argmin(mu - sigma), satisfied set = {mu - sigma <= min(mu + sigma)} in candidate order
//   rounds      no refit: with c0(s, x) the covariance given the data, M = Sigma0(S, S) + D and its bordered factor L_M,
//               each round appends one block row [R_j, L_jj] of L_M (lcb_border_kernel) and, per surviving candidate,
//               w_j(x) = L_jj^-1 (c0(s_j rows, x) - R_j w_<j(x)),  sigma_{j+1}^2 = sigma_j^2 - |w_j(x)|^2
//               (lcb_round_kernel); the next point is argmax sigma over the satisfied set.
// Failures are flagged on the device (LcbStatus) and stop the later kernels; the host reads the flag after the screen
// (it needs the size of the satisfied set) and once after the last round.  The GP handle is not modified.
#include <algorithm>
#include <climits>
#include <cmath>

#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {

namespace {

constexpr double kPivotTol = 1.0e-16;
constexpr int kWarps = 4;  // candidates per CTA of the screen and round kernels, one warp each
constexpr int kSelThreads = 1024;
constexpr int kMaxB = CMOE_MAX_DIM + 1;  // rows per point, 1 + g

struct LcbStatus {
  int failed;  // 0, or 1 once a pivot or a candidate's variance failed `> 1e-16`
  int info;    // leading minor in the enlarged matrix (bordered step) or 1 (a candidate's variance)
  int cand;    // lowest failing candidate index (INT_MAX: none)
  int nsat;    // size of the satisfied set
};

__device__ __forceinline__ int lcb_row_type(const KernelSpec& spec, int local) {
  return local ? spec.derivs[local - 1] : -1;
}

__device__ __forceinline__ void flag_candidate(LcbStatus* st, int cand) {
  atomicMin(&st->cand, cand);
  st->info = 1;
  atomicExch(&st->failed, 1);
}

// sigma0^2(x) = k(x,x) - |L^-1 k(X,x)|^2 for the nc candidates of one chunk; one warp per candidate, each lane sums the
// rows r = lane mod 32 in ascending order and the lanes are combined by a fixed butterfly, so the result does not depend
// on the chunk.  A variance that is not > 1e-16 (the value pivot of the reference's Cholesky) fails the candidate.
__global__ void __launch_bounds__(kWarps * 32) lcb_screen_kernel(const __grid_constant__ KernelSpec spec,
                                                                 const double* __restrict__ V, int n,
                                                                 const double* __restrict__ P, int nc, int c0,
                                                                 double* __restrict__ sd, double* __restrict__ s2,
                                                                 LcbStatus* st) {
  const int lane = threadIdx.x & 31, c = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (c >= nc) return;
  const double* v = V + static_cast<size_t>(c) * n;
  double acc = 0.0;
  for (int r = lane; r < n; r += 32) acc = fma(v[r], v[r], acc);
  acc = warp_sum(acc);
  if (lane != 0) return;
  const double* x = P + static_cast<size_t>(c) * spec.dim;
  const double var = cov_entry(spec, kernel_parts(spec, weighted_sqdist(spec, x, x)), x, x, -1, -1) - acc;
  const int idx = c0 + c;
  s2[idx] = var;
  if (var > kPivotTol) {
    sd[idx] = sqrt(var);
  } else {
    sd[idx] = 0.0;
    flag_candidate(st, idx);
  }
}

// One CTA: sel[0] = argmin(mu - sd) (first occurrence), then the satisfied set {mu - sd <= min(mu + sd)} compacted in
// candidate order into sat[], its size into st->nsat.
__global__ void __launch_bounds__(kSelThreads) lcb_select_kernel(const double* __restrict__ mu,
                                                                 const double* __restrict__ sd, int C, LcbStatus* st,
                                                                 int* __restrict__ sel, int* __restrict__ sat) {
  __shared__ double sv[kSelThreads / 32], su[kSelThreads / 32];
  __shared__ int si[kSelThreads / 32];
  __shared__ int wcount[kSelThreads / 32];
  __shared__ int base;
  if (st->failed) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double best = INFINITY, ub = INFINITY;
  int bidx = INT_MAX;
  for (int i = tid; i < C; i += kSelThreads) {
    const double t = mu[i] - sd[i], u = mu[i] + sd[i];
    if (t < best) {
      best = t;
      bidx = i;
    }
    ub = fmin(ub, u);
  }
  block_best<false>(best, bidx, sv, si);
  for (int o = 16; o > 0; o >>= 1) ub = fmin(ub, __shfl_xor_sync(0xffffffffu, ub, o));
  if (lane == 0) su[warp] = ub;
  __syncthreads();
  double upper = INFINITY;
  for (int w = 0; w < kSelThreads / 32; ++w) upper = fmin(upper, su[w]);
  if (tid == 0) {
    sel[0] = (bidx == INT_MAX) ? 0 : bidx;
    base = 0;
  }
  __syncthreads();
  for (int i0 = 0; i0 < C; i0 += kSelThreads) {
    const int i = i0 + tid;
    const bool ok = i < C && (mu[i] - sd[i]) <= upper;
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) wcount[warp] = __popc(m);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += wcount[w];
    if (ok) sat[off + __popc(m & ((1u << lane) - 1u))] = i;
    __syncthreads();
    if (tid == 0) {
      int t = base;
      for (int w = 0; w < kSelThreads / 32; ++w) t += wcount[w];
      base = t;
    }
    __syncthreads();
  }
  if (tid == 0) st->nsat = base;
}

// out[dim] = candidate sel[0]
__global__ void lcb_gather_kernel(const double* __restrict__ cand, int dim, const int* __restrict__ sel,
                                  double* __restrict__ out) {
  if (static_cast<int>(threadIdx.x) < dim) out[threadIdx.x] = cand[static_cast<size_t>(*sel) * dim + threadIdx.x];
}

// G[r][c] = T_k[:, r] . T[:, c] for the b rows of the newest point (block k) and the (k+1) b columns of blocks 0..k
// (T_l = L^-1 K(X, s_l rows), b columns per block); one CTA per entry, fixed-order block sum.
__global__ void __launch_bounds__(256) lcb_cross_kernel(const double* __restrict__ T, int n, int b, int k,
                                                        double* __restrict__ G, const LcbStatus* st) {
  __shared__ double scratch[8];
  if (st->failed) return;
  const int e = blockIdx.x, r = e % b, c = e / b, lb = c / b, t = c % b;
  const double* tr = T + (static_cast<size_t>(k) * b + r) * n;
  const double* tc = T + (static_cast<size_t>(lb) * b + t) * n;
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc = fma(tr[i], tc[i], acc);
  acc = block_sum(acc, scratch);
  if (threadIdx.x == 0) G[static_cast<size_t>(r) * (k + 1) * b + c] = acc;
}

// Block row k of L_M (row-major, leading dimension ld), M = Sigma0(S, S) + D, one CTA:
//   M_k = Kp(rows of point k) - G,  R_k = M_{k,<k} L_<k^-T (one warp per row, ascending columns),
//   L_kk = chol(M_kk - R_k R_k^T).  Kp = K(S, S) + D (build_covariance, (k+1) b square, column-major lower).
// A pivot that is not > 1e-16 sets info = its leading minor in the enlarged matrix, n0 + k b + j + 1.
__global__ void __launch_bounds__(256) lcb_border_kernel(const double* __restrict__ Kp, const double* __restrict__ G,
                                                         int b, int k, double* __restrict__ LM, int ld, int n0,
                                                         LcbStatus* st) {
  __shared__ double S[kMaxB * kMaxB];
  if (st->failed) return;
  const int kb = k * b, m = kb + b;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int r = warp; r < b; r += nw) {
    double* Rr = LM + static_cast<size_t>(kb + r) * ld;
    const double* Gr = G + static_cast<size_t>(r) * m;
    for (int c = 0; c < kb; ++c) {
      const double* Lc = LM + static_cast<size_t>(c) * ld;
      double acc = 0.0;
      for (int cc = lane; cc < c; cc += 32) acc = fma(Rr[cc], Lc[cc], acc);
      acc = warp_sum(acc);
      if (lane == 0) Rr[c] = (Kp[static_cast<size_t>(c) * m + kb + r] - Gr[c] - acc) / Lc[c];
      __syncwarp();
    }
  }
  __syncthreads();
  for (int e = warp; e < b * b; e += nw) {
    const int r = e / b, t = e % b;
    if (t > r) continue;
    const double* Rr = LM + static_cast<size_t>(kb + r) * ld;
    const double* Rt = LM + static_cast<size_t>(kb + t) * ld;
    double acc = 0.0;
    for (int c = lane; c < kb; c += 32) acc = fma(Rr[c], Rt[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) S[r * kMaxB + t] = Kp[static_cast<size_t>(kb + t) * m + kb + r] - G[static_cast<size_t>(r) * m + kb + t] - acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int j = 0; j < b; ++j) {
      double d = S[j * kMaxB + j];
      for (int c = 0; c < j; ++c) d -= S[j * kMaxB + c] * S[j * kMaxB + c];
      if (!(d > kPivotTol)) {
        st->info = n0 + kb + j + 1;
        st->failed = 1;
        break;
      }
      d = sqrt(d);
      S[j * kMaxB + j] = d;
      for (int i = j + 1; i < b; ++i) {
        double v = S[i * kMaxB + j];
        for (int c = 0; c < j; ++c) v -= S[i * kMaxB + c] * S[j * kMaxB + c];
        S[i * kMaxB + j] = v / d;
      }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < b * b; e += blockDim.x) {
    const int r = e / b, t = e % b;
    if (t <= r) LM[static_cast<size_t>(kb + r) * ld + kb + t] = S[r * kMaxB + t];
  }
}

// One round for the satisfied candidates, one warp each (position p, candidate sat[p]):
//   c0(s_k row t, x) = k(s_k row t, x) - sum_rows k(x, X_row) B[row][t]     (B = K^-1 K(X, s_k rows), n x b)
//   w = L_kk^-1 (c0 - R_k w_<k(x)),  sigma^2 -= |w|^2
// Lanes stride over the training points (ascending) and are combined by a fixed butterfly; the triangular steps run on
// lane 0 in ascending order.  Each CTA leaves max sigma (ties: lowest position) in part_v / part_i.
__global__ void __launch_bounds__(kWarps * 32) lcb_round_kernel(
    const __grid_constant__ KernelSpec spec, const double* __restrict__ X, int N, const double* __restrict__ cand,
    const int* __restrict__ sat, int nsat, const double* __restrict__ B, int n, const double* __restrict__ sp,
    const double* __restrict__ LM, int ld, int k, const double* __restrict__ s2_screen, double* __restrict__ W,
    double* __restrict__ s2, double* __restrict__ part_v, int* __restrict__ part_i, LcbStatus* st) {
  extern __shared__ double lsm[];  // [kWarps][b][32] lane accumulators, then [kWarps][b] right-hand sides
  __shared__ double xs[kWarps][CMOE_MAX_DIM];
  __shared__ double ss[CMOE_MAX_DIM];
  __shared__ double bv[kWarps];
  __shared__ int bi[kWarps];
  __shared__ int stop;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, dim = spec.dim, b = 1 + spec.g, kb = k * b;
  if (tid == 0) stop = st->failed;
  __syncthreads();
  if (stop) return;
  const int p = blockIdx.x * kWarps + warp;
  const bool live = p < nsat;
  for (int e = tid; e < dim; e += blockDim.x) ss[e] = sp[e];
  if (live)
    for (int e = lane; e < dim; e += 32) xs[warp][e] = cand[static_cast<size_t>(sat[p]) * dim + e];
  __syncthreads();
  double best = -INFINITY;
  int bidx = INT_MAX;
  if (live) {
    const double* x = xs[warp];
    double* acc = lsm + static_cast<size_t>(warp) * b * 32;
    double* u = lsm + static_cast<size_t>(kWarps) * b * 32 + warp * b;
    double a0 = 0.0;
    for (int t = 0; t < b; ++t) acc[t * 32 + lane] = 0.0;
    for (int j = lane; j < N; j += 32) {
      const double* xj = X + static_cast<size_t>(j) * dim;
      const KParts kp = kernel_parts(spec, weighted_sqdist(spec, x, xj));
      for (int cc = 0; cc < b; ++cc) {
        const double v = cov_entry(spec, kp, x, xj, -1, lcb_row_type(spec, cc));
        const double* Bj = B + static_cast<size_t>(j) * b + cc;
        if (b == 1) {
          a0 = fma(v, Bj[0], a0);
        } else {
          for (int t = 0; t < b; ++t) acc[t * 32 + lane] = fma(v, Bj[static_cast<size_t>(t) * n], acc[t * 32 + lane]);
        }
      }
    }
    const KParts ks = kernel_parts(spec, weighted_sqdist(spec, ss, x));
    const double* Wp = W + static_cast<size_t>(p) * ld;
    for (int t = 0; t < b; ++t) {
      const double kx = warp_sum(b == 1 ? a0 : acc[t * 32 + lane]);
      const double* Rt = LM + static_cast<size_t>(kb + t) * ld;
      double r = 0.0;
      for (int c = lane; c < kb; c += 32) r = fma(Rt[c], Wp[c], r);
      r = warp_sum(r);
      if (lane == 0) u[t] = (cov_entry(spec, ks, ss, x, lcb_row_type(spec, t), -1) - kx) - r;
    }
    __syncwarp();
    if (lane == 0) {
      double v2 = (k == 0) ? s2_screen[sat[p]] : s2[p];
      double* Wo = W + static_cast<size_t>(p) * ld + kb;
      for (int t = 0; t < b; ++t) {
        const double* Lt = LM + static_cast<size_t>(kb + t) * ld + kb;
        double w = u[t];
        for (int c = 0; c < t; ++c) w -= Lt[c] * u[c];
        w /= Lt[t];
        u[t] = w;
        Wo[t] = w;
        v2 -= w * w;
      }
      s2[p] = v2;
      if (v2 > kPivotTol) {
        best = sqrt(v2);
        bidx = p;
      } else {
        flag_candidate(st, sat[p]);
      }
    }
  }
  block_best<true>(best, bidx, bv, bi);
  if (tid == 0) {
    part_v[blockIdx.x] = best;
    part_i[blockIdx.x] = bidx;
  }
}

// *sel_out = sat[argmax over the CTA partials] (ties: lowest position); one warp
__global__ void lcb_argmax_kernel(const double* __restrict__ part_v, const int* __restrict__ part_i, int nparts,
                                  const int* __restrict__ sat, int* __restrict__ sel_out, const LcbStatus* st) {
  if (st->failed) return;
  const int lane = threadIdx.x;
  double best = -INFINITY;
  int bidx = INT_MAX;
  for (int q = lane; q < nparts; q += 32)
    if (beats<true>(part_v[q], part_i[q], best, bidx)) {
      best = part_v[q];
      bidx = part_i[q];
    }
  warp_best<true>(best, bidx);
  if (lane == 0) *sel_out = sat[bidx == INT_MAX ? 0 : bidx];
}

}  // namespace

}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_lcb_select(const cmoe_gp* gp, const double* candidates, int num_candidates, int num_to_sample,
                               int* selected, double* mean, double* sd, int* num_satisfied, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_candidates >= 1 && num_to_sample >= 1, CMOE_ERR_BOUNDS,
                 "num_candidates and num_to_sample must be >= 1");
    CMOE_REQUIRE(gp != nullptr && candidates != nullptr && selected != nullptr, CMOE_ERR_INVALID_VALUE,
                 "gp, candidates and selected must not be NULL");
    const KernelSpec& spec = gp->spec;
    const int dim = spec.dim, b = 1 + spec.g, C = num_candidates, q = num_to_sample;
    const long long rows_ll = static_cast<long long>(q - 1) * b;
    CMOE_REQUIRE(rows_ll <= kMaxLcbSelectedRows, CMOE_ERR_BOUNDS,
                 "(num_to_sample - 1) * (1 + num_derivatives) must be <= 1024");
    const size_t cdim = static_cast<size_t>(C) * dim;
    for (size_t e = 0; e < cdim; ++e)
      CMOE_REQUIRE(std::isfinite(candidates[e]), CMOE_ERR_INVALID_VALUE, "candidates must be finite");
    require_device(gp->device);
    cudaStream_t s = gp->stream;
    const int n = gp->n, N = gp->N, rows = static_cast<int>(rows_ll);

    DevBuf<double> dCand(cdim), dMu(C), dSd(C), dS2(C);
    DevBuf<int> dSel(q), dSat(C), dDer(spec.g > 0 ? spec.g : 1);
    DevBuf<LcbStatus> dSt(1);
    const LcbStatus st0{0, 0, INT_MAX, 0};
    dSt.upload(&st0, 1, s);
    dCand.upload(candidates, cdim, s);
    if (spec.g > 0) dDer.upload(spec.derivs, spec.g, s);
    CMOE_CUDA(cudaMemsetAsync(dSel.p, 0, q * sizeof(int), s));

    // screen, in chunks of the sampling workspace (one column of V per candidate)
    SampleWork& w = sample_work(*gp);
    const int chunk = static_cast<int>(chunk_items(C, kSampleWorkspaceBytes, sizeof(double) * n));
    w.V.ensure(static_cast<size_t>(chunk) * n);
    for (int c0 = 0; c0 < C; c0 += chunk) {
      const int nc = std::min(chunk, C - c0);
      const double* Pc = dCand.p + static_cast<size_t>(c0) * dim;
      build_mix_covariance(spec, gp->dX.p, N, Pc, nc, dDer.p, 0, w.V.p, s);
      // the blocked kernel whatever the column count: a candidate's solve does not depend on the chunk it lands in
      trsm_lower_blocked(gp->dK.p, n, w.V.p, n, nc, false, s);
      posterior_mean_points(*gp, Pc, nc, dDer.p, 0, dMu.p + c0, nullptr, s);
      lcb_screen_kernel<<<(nc + kWarps - 1) / kWarps, kWarps * 32, 0, s>>>(spec, w.V.p, n, Pc, nc, c0, dSd.p, dS2.p,
                                                                          dSt.p);
      count_launch();
    }
    lcb_select_kernel<<<1, kSelThreads, 0, s>>>(dMu.p, dSd.p, C, dSt.p, dSel.p, dSat.p);
    count_launch();
    CMOE_CUDA(cudaGetLastError());
    LcbStatus st{};
    dSt.download(&st, 1, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    auto raise_candidate = [](const LcbStatus& f) {
      throw Error(CMOE_ERR_SINGULAR,
                  "GP-Variance matrix singular at candidate " + std::to_string(f.cand) +
                      ". Check for candidates duplicating points_sampled (or earlier selections) with 0 noise.",
                  1);
    };
    if (st.failed) raise_candidate(st);
    const int nsat = st.nsat;
    CMOE_REQUIRE(static_cast<size_t>(nsat) * rows <= kMaxLcbRoundDoubles, CMOE_ERR_BOUNDS,
                 "num_satisfied * (num_to_sample - 1) * (1 + num_derivatives) must be <= 2^28");

    if (q > 1) {
      // The rounds' solves take the blocked kernel: trsm_lower sends few columns of a large factor to the cooperative
      // single-vector solver, which synchronises the host, and the rounds run without a synchronise.  The blocked
      // kernel is one CTA per 32 columns, so at large n it sets a round's time (DESIGN.md K13).
      const int nparts = (nsat + kWarps - 1) / kWarps;
      DevBuf<double> Psel(static_cast<size_t>(q) * dim), Pss, T(static_cast<size_t>(q - 1) * b * n),
          B(static_cast<size_t>(b) * n), Kp(static_cast<size_t>(rows) * rows), G(static_cast<size_t>(b) * rows),
          LM(static_cast<size_t>(rows) * rows), W(static_cast<size_t>(nsat) * rows), s2(nsat), part_v(nparts);
      DevBuf<int> part_i(nparts);
      Pss.alloc(static_cast<size_t>((q + 127) / 128) * 128 * dim);  // sized once: no reallocation between rounds
      const size_t smem_round = (static_cast<size_t>(kWarps) * b * 32 + static_cast<size_t>(kWarps) * b) * sizeof(double);
      for (int k = 0; k + 1 < q; ++k) {
        const int m = (k + 1) * b;
        double* Tk = T.p + static_cast<size_t>(k) * b * n;
        lcb_gather_kernel<<<1, 32, 0, s>>>(dCand.p, dim, dSel.p + k, Psel.p + static_cast<size_t>(k) * dim);
        count_launch();
        build_mix_covariance(spec, gp->dX.p, N, Psel.p + static_cast<size_t>(k) * dim, 1, dDer.p, spec.g, Tk, s);
        trsm_lower_blocked(gp->dK.p, n, Tk, n, b, false, s);  // T_k = L^-1 K(X, s_k rows)
        CMOE_CUDA(cudaMemcpyAsync(B.p, Tk, static_cast<size_t>(b) * n * sizeof(double), cudaMemcpyDeviceToDevice, s));
        trsm_lower_blocked(gp->dK.p, n, B.p, n, b, true, s);  // B = K^-1 K(X, s_k rows)
        scale_points(*gp, Psel.p, k + 1, Pss, s);
        CMOE_CUDA(cudaMemsetAsync(Kp.p, 0, static_cast<size_t>(m) * m * sizeof(double), s));
        build_covariance(spec, Psel.p, Pss.p, k + 1, gp->dnoise.p, Kp.p, s);  // K(S, S) + D, as append_points
        lcb_cross_kernel<<<m * b, 256, 0, s>>>(T.p, n, b, k, G.p, dSt.p);
        lcb_border_kernel<<<1, 256, 0, s>>>(Kp.p, G.p, b, k, LM.p, rows, n, dSt.p);
        lcb_round_kernel<<<nparts, kWarps * 32, smem_round, s>>>(spec, gp->dX.p, N, dCand.p, dSat.p, nsat, B.p, n,
                                                                 Psel.p + static_cast<size_t>(k) * dim, LM.p, rows, k,
                                                                 dS2.p, W.p, s2.p, part_v.p, part_i.p, dSt.p);
        lcb_argmax_kernel<<<1, 32, 0, s>>>(part_v.p, part_i.p, nparts, dSat.p, dSel.p + k + 1, dSt.p);
        count_launch(4);
      }
      CMOE_CUDA(cudaGetLastError());
      dSt.download(&st, 1, s);
      CMOE_CUDA(cudaStreamSynchronize(s));
      if (st.failed && st.cand != INT_MAX) raise_candidate(st);
      if (st.failed)
        throw Error(CMOE_ERR_SINGULAR,
                    "Covariance matrix (K) singular. Check for duplicate points_sampled (with 0 noise) and/or extreme "
                    "hyperparameter values.",
                    st.info);
    }
    dSel.download(selected, q, s);
    if (mean) dMu.download(mean, C, s);
    if (sd) dSd.download(sd, C, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    if (num_satisfied) *num_satisfied = nsat;
  });
}

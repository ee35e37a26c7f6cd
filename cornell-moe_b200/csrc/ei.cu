// q-EI Monte-Carlo estimator and its pathwise gradient, batched over candidates.
//
// Replaces ExpectedImprovementEvaluator::ComputeExpectedImprovement / ComputeGradExpectedImprovement
// (reference gpp_math.cpp:1991-2033, 2050-2126) and EvaluateEIAtPointList (gpp_math.cpp:2305-2356).
//
// Kernel 1 (one thread per MC sample): Philox normals (or table replay) -> y = L z -> improvement and winner.
// Kernel 2 (one CTA per candidate): fixed-order reduction of sum(improvement), count[winner] and
//   Zsum[winner][i] = sum z_i, then  grad[k] = -(1/mc) ( count[k] dmu_k + sum_{w,i} dL_k[w,i] Zsum[w][i] ),
//   which is the reference's per-sample accumulation (gpp_math.cpp:2105-2119) with the sums exchanged.
#include <algorithm>

#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {

namespace {

__global__ void __launch_bounds__(256) ei_sample_kernel(int U, int num_mc, double best_so_far, uint64_t seed,
                                                        const double* __restrict__ table,
                                                        const double* __restrict__ mu,
                                                        const double* __restrict__ chol, const int* __restrict__ fail,
                                                        double* __restrict__ zbuf, double* __restrict__ imp,
                                                        int* __restrict__ winner) {
  extern __shared__ double sm[];
  const int c = blockIdx.y;
  if (fail[c] != 0) return;
  double* Ls = sm;           // [U][U] column-major
  double* ms = sm + U * U;   // [U]
  for (int e = threadIdx.x; e < U * U; e += blockDim.x) Ls[e] = chol[static_cast<size_t>(c) * U * U + e];
  for (int e = threadIdx.x; e < U; e += blockDim.x) ms[e] = mu[static_cast<size_t>(c) * U + e];
  __syncthreads();
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= num_mc) return;
  double z[kMaxQ];
  if (table != nullptr) {
    for (int i = 0; i < U; ++i) z[i] = table[static_cast<size_t>(s) * U + i];
  } else {
    for (int k = 0; 2 * k < U; ++k) {
      double a, b;
      philox_normal_pair(seed, static_cast<uint64_t>(s), k, a, b);
      z[2 * k] = a;
      if (2 * k + 1 < U) z[2 * k + 1] = b;
    }
  }
  double* zo = zbuf + (static_cast<size_t>(c) * num_mc + s) * U;
  for (int i = 0; i < U; ++i) zo[i] = z[i];
  double best = 0.0;
  int win = -1;
  for (int j = 0; j < U; ++j) {
    double y = Ls[j + j * U] * z[j];
    for (int i = j - 1; i >= 0; --i) y += Ls[j + i * U] * z[i];
    const double e = best_so_far - (ms[j] + y);
    if (e > best) {  // strict >: the first maximiser wins (gpp_math.cpp:2092)
      best = e;
      win = j;
    }
  }
  imp[static_cast<size_t>(c) * num_mc + s] = best;
  winner[static_cast<size_t>(c) * num_mc + s] = win;
}

__global__ void __launch_bounds__(256) ei_reduce_kernel(int U, int q, int dim, int nd, int num_mc,
                                                        const double* __restrict__ zbuf,
                                                        const double* __restrict__ imp,
                                                        const int* __restrict__ winner,
                                                        const double* __restrict__ gmu,
                                                        const double* __restrict__ gchol,
                                                        const int* __restrict__ fail, double* __restrict__ ei,
                                                        double* __restrict__ grad) {
  extern __shared__ double sm[];
  __shared__ double red[8];
  const int c = blockIdx.x, tid = threadIdx.x;
  if (fail[c] != 0) {
    if (tid == 0) ei[c] = nan("");
    return;
  }
  const double* ic = imp + static_cast<size_t>(c) * num_mc;
  const int* wc = winner + static_cast<size_t>(c) * num_mc;
  double part = 0.0;
  for (int s = tid; s < num_mc; s += blockDim.x) part += ic[s];
  const double total = block_sum(part, red);
  if (tid == 0) ei[c] = total / static_cast<double>(num_mc);
  if (grad == nullptr) return;
  double* Zsum = sm;            // [U][U]  (winner, i)
  double* cnt = sm + U * U;     // [U]
  const double* zc = zbuf + static_cast<size_t>(c) * num_mc * U;
  for (int o = tid; o < U * U + U; o += blockDim.x) {
    double acc = 0.0;
    if (o < U * U) {
      const int w = o / U, i = o % U;
      for (int s = 0; s < num_mc; ++s)
        if (wc[s] == w) acc += zc[static_cast<size_t>(s) * U + i];
      Zsum[o] = acc;
    } else {
      const int w = o - U * U;
      for (int s = 0; s < num_mc; ++s)
        if (wc[s] == w) acc += 1.0;
      cnt[w] = acc;
    }
  }
  __syncthreads();
  for (int o = tid; o < q * dim; o += blockDim.x) {
    const int k = o / dim, d = o % dim;
    const double* G = gchol + (static_cast<size_t>(c) * nd + k) * U * U * dim;
    double g = cnt[k] * gmu[(static_cast<size_t>(c) * nd + k) * dim + d];
    for (int w = 0; w < U; ++w)
      for (int i = 0; i <= w; ++i) g += G[(static_cast<size_t>(w) * U + i) * dim + d] * Zsum[w * U + i];
    grad[(static_cast<size_t>(c) * q + k) * dim + d] = -g / static_cast<double>(num_mc);
  }
}

}  // namespace

// candidates (host) -> union sets on the device: set c = [candidate c (q points); points_being_sampled (p points)]
void upload_union_sets(PosteriorBatch& pb, const double* candidates, int nc, int q, const double* Xp, int p, int dim,
                       cudaStream_t s) {
  std::vector<double> h(static_cast<size_t>(nc) * (q + p) * dim);
  for (int c = 0; c < nc; ++c) {
    double* dst = h.data() + static_cast<size_t>(c) * (q + p) * dim;
    std::copy(candidates + static_cast<size_t>(c) * q * dim, candidates + static_cast<size_t>(c + 1) * q * dim, dst);
    if (p) std::copy(Xp, Xp + static_cast<size_t>(p) * dim, dst + static_cast<size_t>(q) * dim);
  }
  pb.P.upload(h.data(), h.size(), s);
  CMOE_CUDA(cudaStreamSynchronize(s));  // h goes out of scope
}

namespace {
void ei_eval_chunk(const cmoe_gp& gp, const double* candidates, int nc, int q, const double* Xp, int p, int num_mc,
                   double best_so_far, uint64_t seed, const double* dtable, double* ei_host, double* grad_host) {
  cudaStream_t s = gp.stream;
  const int U = q + p, dim = gp.spec.dim;
  const bool want_grad = grad_host != nullptr;
  PosteriorBatch pb;
  pb.configure(gp, nc, U, nullptr, 0, want_grad ? q : 0, s);
  upload_union_sets(pb, candidates, nc, q, Xp, p, dim, s);
  pb.run(gp, /*diag_mode=*/1, /*want_chol=*/true, want_grad, s);
  int which = 0;
  const int f = pb.first_failure(s, &which);
  if (f != 0) throw_singular_union(f);
  DevBuf<double> zbuf(static_cast<size_t>(nc) * num_mc * U), imp(static_cast<size_t>(nc) * num_mc);
  DevBuf<int> win(static_cast<size_t>(nc) * num_mc);
  DevBuf<double> dei(nc), dgrad(want_grad ? static_cast<size_t>(nc) * q * dim : 1);
  // (U^2 + U) doubles: past the default 48 KiB from U = 78 on, 74.5 KB at U = kMaxQ = 96
  const size_t smem1 = (static_cast<size_t>(U) * U + U) * sizeof(double);
  constexpr int kMaxSmem = (kMaxQ * kMaxQ + kMaxQ) * sizeof(double);
  CMOE_CUDA(cudaFuncSetAttribute(ei_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  CMOE_CUDA(cudaFuncSetAttribute(ei_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  ei_sample_kernel<<<dim3((num_mc + 255) / 256, nc), 256, smem1, s>>>(U, num_mc, best_so_far, seed, dtable, pb.mu.p,
                                                                      pb.chol.p, pb.fail.p, zbuf.p, imp.p, win.p);
  ei_reduce_kernel<<<nc, 256, smem1, s>>>(U, q, dim, want_grad ? q : 0, num_mc, zbuf.p, imp.p, win.p, pb.gmu.p,
                                          pb.gchol.p, pb.fail.p, dei.p, want_grad ? dgrad.p : nullptr);
  count_launch(2);
  CMOE_CUDA(cudaGetLastError());
  dei.download(ei_host, nc, s);
  if (want_grad) dgrad.download(grad_host, static_cast<size_t>(nc) * q * dim, s);
  CMOE_CUDA(cudaStreamSynchronize(s));
}
}  // namespace

// any number of candidates: the per-sample scratch (z, improvement, winner) is bounded to ~2 GiB per chunk, and a chunk
// holds at most 65535 candidates (grid.y of ei_sample_kernel) — for the C entry point and the multistart drivers alike
void ei_eval_batch(const cmoe_gp& gp, const double* candidates, int nc, int q, const double* Xp, int p, int num_mc,
                   double best_so_far, uint64_t seed, const double* dtable, double* ei_host, double* grad_host) {
  const int U = q + p, dim = gp.spec.dim;
  const size_t per_cand = static_cast<size_t>(num_mc) * (U + 2) * sizeof(double);
  const int batch = static_cast<int>(chunk_items(nc, size_t(2) << 30, per_cand, kMaxGridY));
  for (int c0 = 0; c0 < nc; c0 += batch) {
    const int nb = std::min(batch, nc - c0);
    ei_eval_chunk(gp, candidates + static_cast<size_t>(c0) * q * dim, nb, q, Xp, p, num_mc, best_so_far, seed, dtable,
                  ei_host + c0, grad_host ? grad_host + static_cast<size_t>(c0) * q * dim : nullptr);
  }
}

}  // namespace cmoe

using namespace cmoe;  // NOLINT

extern "C" int cmoe_ei_eval(const cmoe_gp* gp, const double* candidates, int num_candidates, int q,
                            const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                            const double* normals_table, double* ei, double* grad_ei, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_candidates >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    CMOE_REQUIRE(q >= 1 && p >= 0 && num_mc >= 1, CMOE_ERR_BOUNDS, "q >= 1, p >= 0, num_mc >= 1 required");
    require_device(gp->device);
    const int U = q + p;
    DevBuf<double> dtable;
    if (normals_table) dtable.upload(normals_table, static_cast<size_t>(num_mc) * U, gp->stream);
    ei_eval_batch(*gp, candidates, num_candidates, q, points_being_sampled, p, num_mc, best_so_far, seed,
                  normals_table ? dtable.p : nullptr, ei, grad_ei);
  });
}

// GaussianProcess handle: covariance build -> blocked Cholesky -> K^-1 (y - mean), all on the device.
// Replaces GaussianProcess::GaussianProcess / RecomputeDerivedVariables / AddPointsToGP
// (reference gpp_math.cpp:553-573, 481-511, 1699-1718).
#include <algorithm>
#include <cmath>

#include "device_math.cuh"
#include "internal.cuh"

namespace cmoe {

namespace {
thread_local std::string g_last_error;

__global__ void center_values_kernel(const double* __restrict__ y, int N, int b, double mean,
                                     double* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= N * b) return;
  out[r] = y[r] - ((r % b == 0) ? mean : 0.0);  // only function-value rows carry the constant prior mean
}

// Length-scaled coordinates of the fast covariance build, centred first: that kernel forms -r^2/2 as
// x.y - |x|^2/2 - |y|^2/2, whose absolute error grows with |x|^2 + |y|^2 in length-scale units — a domain far from the
// origin ([1000, 1010] with l = 1) would otherwise lose ~1e-10 relative on every entry.  The kernels are translation
// invariant, so any common shift is exact in exact arithmetic; coincident points still map to identical coordinates.
// The centre is kept on the handle (cmoe_gp::centre): the q-KG operands (kg.cu) use the same expanded form and are put
// in the same frame, so a fit and a q-KG plan always share one origin.
__global__ void scale_points_kernel(const __grid_constant__ KernelSpec spec, const __grid_constant__ Centre centre,
                                    const double* __restrict__ X, int N, double* __restrict__ Xs) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * spec.dim) return;
  const int d = e % spec.dim;
  Xs[e] = (X[e] - centre.c[d]) * spec.inv_len[d];
}

Centre centre_of(const std::vector<double>& hX, int N, int dim) {
  Centre c{};
  for (int d = 0; d < dim; ++d) {
    double m = 0.0;
    for (int i = 0; i < N; ++i) m += hX[static_cast<size_t>(i) * dim + d];
    c.c[d] = N > 0 ? m / N : 0.0;
  }
  return c;
}

// the handle's centre from its training points (every (re)fit and append)
Centre update_centre(cmoe_gp* gp) {
  const Centre c = centre_of(gp->hX, gp->N, gp->spec.dim);
  std::copy(c.c, c.c + CMOE_MAX_DIM, gp->centre);
  return c;
}

// ---- incremental append (cmoe_gp_add_sampled_points) --------------------------------------------------------------
// S22[i][j] -= sum_r T[r][i] T[r][j] for i >= j (T = L^-1 K12, n0 x mm column-major); one CTA per entry.
__global__ void __launch_bounds__(256) append_schur_kernel(const double* __restrict__ T, int n0, int mm,
                                                           double* __restrict__ S22) {
  __shared__ double scratch[8];
  int e = blockIdx.x, j = 0;  // lower-triangular entry index -> (i, j), column-major enumeration
  while (e >= mm - j) {
    e -= mm - j;
    ++j;
  }
  const int i = j + e;
  const double* ti = T + static_cast<size_t>(i) * n0;
  const double* tj = T + static_cast<size_t>(j) * n0;
  double acc = 0.0;
  for (int r = threadIdx.x; r < n0; r += blockDim.x) acc = fma(ti[r], tj[r], acc);
  acc = block_sum(acc, scratch);
  if (threadIdx.x == 0) S22[static_cast<size_t>(j) * mm + i] -= acc;
}

// K1[(n0 + i), r] = T[r, i]  (the new rows of the factor), K1 column-major with leading dimension n1
__global__ void append_rows_kernel(const double* __restrict__ T, int n0, int mm, double* __restrict__ K1, int n1) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<size_t>(n0) * mm) return;
  const int i = static_cast<int>(e % mm), r = static_cast<int>(e / mm);
  K1[static_cast<size_t>(r) * n1 + n0 + i] = T[static_cast<size_t>(i) * n0 + r];
}

// The TMA covariance build copies whole 128-row slabs of the scaled points: keep the allocation padded (and defined)
// up to the next multiple of 128 rows.
void ensure_scaled_points(DevBuf<double>& buf, int N, int dim, cudaStream_t s) {
  const size_t rows = (static_cast<size_t>(N) + 127) / 128 * 128;
  if (buf.count < rows * dim) buf.alloc(rows * dim);
  CMOE_CUDA(cudaMemsetAsync(buf.p + static_cast<size_t>(N) * dim, 0, (rows - N) * dim * sizeof(double), s));
}
}  // namespace

void set_last_error(const std::string& msg) { g_last_error = msg; }

void require_device(int device) {
  int count = 0;
  cudaError_t err = cudaGetDeviceCount(&count);
  if (err != cudaSuccess || count == 0) {
    cudaGetLastError();
    throw Error(CMOE_ERR_NO_DEVICE,
                "cornell-moe_b200: no CUDA device visible; this library has no CPU compute path");
  }
  if (device < 0 || device >= count) throw Error(CMOE_ERR_BOUNDS, "device ordinal out of range");
  CMOE_CUDA(cudaSetDevice(device));
}

void fill_kernel_spec(KernelSpec& s, int kernel, int dim, int g, const int* derivs, double alpha,
                      const double* lengths) {
  s = KernelSpec{};
  s.kernel = kernel;
  s.dim = dim;
  s.g = g;
  s.alpha = alpha;
  for (int k = 0; k < CMOE_MAX_DIM; ++k) {
    s.lsq[k] = 1.0;
    s.inv_len[k] = 0.0;
  }
  for (int k = 0; k < dim; ++k) {
    s.lsq[k] = lengths[k] * lengths[k];
    s.inv_len[k] = 1.0 / lengths[k];
  }
  for (int k = 0; k < g; ++k) s.derivs[k] = derivs[k];
}

void fit_gp(cmoe_gp* gp, bool mean_change) {
  drop_cached_plan(gp);  // the cached workspace refers to the previous training set
  ++gp->generation;
  const KernelSpec& spec = gp->spec;
  const int N = gp->N, b = 1 + spec.g, n = N * b;
  gp->n = n;
  cudaStream_t s = gp->stream;
  gp->dX.upload(gp->hX.data(), gp->hX.size(), s);
  gp->dy.upload(gp->hy.data(), gp->hy.size(), s);
  gp->dnoise.upload(gp->hnoise.data(), gp->hnoise.size(), s);
  gp->dK.ensure(static_cast<size_t>(n) * n);
  gp->dKinvY.ensure(n);
  ensure_scaled_points(gp->dXs, N, spec.dim, s);
  if (gp->dFlag.count == 0) gp->dFlag.alloc(1);

  scale_points_kernel<<<(N * spec.dim + 255) / 256, 256, 0, s>>>(spec, update_centre(gp), gp->dX.p, N, gp->dXs.p);
  count_launch();
  EventTimer t0, t1, t2;
  t0.start(s);
  if (spec.g > 0) CMOE_CUDA(cudaMemsetAsync(gp->dK.p, 0, static_cast<size_t>(n) * n * sizeof(double), s));
  build_covariance(spec, gp->dX.p, gp->dXs.p, N, gp->dnoise.p, gp->dK.p, s);
  t0.stop(s);
  t1.start(s);
  potrf_lower(gp->dK.p, n, gp->dFlag.p, s);
  t1.stop(s);
  int flag = 0;
  CMOE_CUDA(cudaMemcpyAsync(&flag, gp->dFlag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CMOE_CUDA(cudaStreamSynchronize(s));
  if (flag != 0) {
    throw Error(CMOE_ERR_SINGULAR,
                "Covariance matrix (K) singular. Check for duplicate points_sampled (with 0 noise) and/or extreme "
                "hyperparameter values.",
                flag);
  }
  if (mean_change) {
    // mean_ = average of the function values (gpp_math.cpp:498-504); same summation order as the reference
    double m = 0.0;
    for (int i = 0; i < N; ++i) m += gp->hy[static_cast<size_t>(i) * b];
    gp->mean = m / N;
  }
  t2.start(s);
  center_values_kernel<<<(n + 255) / 256, 256, 0, s>>>(gp->dy.p, N, b, gp->mean, gp->dKinvY.p);
  count_launch();
  potrs_lower(gp->dK.p, n, gp->dKinvY.p, n, 1, s);
  t2.stop(s);
  CMOE_CUDA(cudaGetLastError());
  CMOE_CUDA(cudaStreamSynchronize(s));
  gp->fit_usec[0] = t0.ms() * 1e3;
  gp->fit_usec[1] = t1.ms() * 1e3;
  gp->fit_usec[2] = t2.ms() * 1e3;
}


// O(N^2) append of m points to a fitted GP (the reference refits from scratch and leaves this as a TODO,
// gpp_math.cpp:1699-1718):  K1 = [K K12; K12^T K22]  =>  L1 = [L 0; (L^-1 K12)^T  chol(K22 - K12^T K^-1 K12)].
// Everything is built beside the live state and swapped in at the end, so a singular update leaves the handle intact.
// The new rows' diagonal carries new_noise [1+g] (host), or the GP's own noise when it is NULL.
void append_points(cmoe_gp* gp, const double* new_points, const double* new_values, int m, const double* new_noise) {
  const KernelSpec& spec = gp->spec;
  const int dim = spec.dim, b = 1 + spec.g, N0 = gp->N, n0 = gp->n, mm = m * b, n1 = n0 + mm;
  cudaStream_t s = gp->stream;
  DevBuf<double> dXn(static_cast<size_t>(m) * dim), dXsn;
  ensure_scaled_points(dXsn, m, dim, s);
  DevBuf<double> K1(static_cast<size_t>(n1) * n1), T(static_cast<size_t>(n0) * mm), S22(static_cast<size_t>(mm) * mm);
  DevBuf<int> dDer(spec.g > 0 ? spec.g : 1), flag(1);
  DevBuf<double> dNoise;
  if (new_noise) dNoise.upload(new_noise, b, s);
  dXn.upload(new_points, static_cast<size_t>(m) * dim, s);
  if (spec.g > 0) dDer.upload(spec.derivs, spec.g, s);
  scale_points_kernel<<<(m * dim + 255) / 256, 256, 0, s>>>(spec, centre_of(gp->hX, N0, dim), dXn.p, m, dXsn.p);
  // old factor -> top-left block under the new leading dimension
  CMOE_CUDA(cudaMemcpy2DAsync(K1.p, static_cast<size_t>(n1) * sizeof(double), gp->dK.p,
                              static_cast<size_t>(n0) * sizeof(double), static_cast<size_t>(n0) * sizeof(double), n0,
                              cudaMemcpyDeviceToDevice, s));
  build_mix_covariance(spec, gp->dX.p, N0, dXn.p, m, dDer.p, spec.g, T.p, s);
  trsm_lower(gp->dK.p, n0, T.p, n0, mm, false, s);  // T = L^-1 K12
  CMOE_CUDA(cudaMemsetAsync(S22.p, 0, S22.count * sizeof(double), s));
  build_covariance(spec, dXn.p, dXsn.p, m, new_noise ? dNoise.p : gp->dnoise.p, S22.p, s);
  append_schur_kernel<<<mm * (mm + 1) / 2, 256, 0, s>>>(T.p, n0, mm, S22.p);
  append_rows_kernel<<<static_cast<unsigned>((static_cast<size_t>(n0) * mm + 255) / 256), 256, 0, s>>>(T.p, n0, mm, K1.p,
                                                                                                   n1);
  count_launch(3);
  potrf_lower(S22.p, mm, flag.p, s);
  int f = 0;
  CMOE_CUDA(cudaMemcpyAsync(&f, flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CMOE_CUDA(cudaStreamSynchronize(s));
  if (f != 0) {
    throw Error(CMOE_ERR_SINGULAR,
                "Covariance matrix (K) singular. Check for duplicate points_sampled (with 0 noise) and/or extreme "
                "hyperparameter values.",
                n0 + f);
  }
  CMOE_CUDA(cudaMemcpy2DAsync(K1.p + static_cast<size_t>(n0) * n1 + n0, static_cast<size_t>(n1) * sizeof(double), S22.p,
                              static_cast<size_t>(mm) * sizeof(double), static_cast<size_t>(mm) * sizeof(double), mm,
                              cudaMemcpyDeviceToDevice, s));
  // commit: host copies, device arrays, mean, K^-1 (y - mean)
  drop_cached_plan(gp);
  ++gp->generation;
  gp->hX.insert(gp->hX.end(), new_points, new_points + static_cast<size_t>(m) * dim);
  gp->hy.insert(gp->hy.end(), new_values, new_values + static_cast<size_t>(mm));
  gp->N = N0 + m;
  gp->n = n1;
  gp->dK = std::move(K1);
  gp->dX.upload(gp->hX.data(), gp->hX.size(), s);
  gp->dy.upload(gp->hy.data(), gp->hy.size(), s);
  ensure_scaled_points(gp->dXs, gp->N, dim, s);
  gp->dKinvY.ensure(n1);
  scale_points_kernel<<<(gp->N * dim + 255) / 256, 256, 0, s>>>(spec, update_centre(gp), gp->dX.p, gp->N, gp->dXs.p);
  double mu = 0.0;  // mean_ = average of the function values (gpp_math.cpp:498-504), same summation order
  for (int i = 0; i < gp->N; ++i) mu += gp->hy[static_cast<size_t>(i) * b];
  gp->mean = mu / gp->N;
  center_values_kernel<<<(n1 + 255) / 256, 256, 0, s>>>(gp->dy.p, gp->N, b, gp->mean, gp->dKinvY.p);
  count_launch(2);
  potrs_lower(gp->dK.p, n1, gp->dKinvY.p, n1, 1, s);
  CMOE_CUDA(cudaGetLastError());
  CMOE_CUDA(cudaStreamSynchronize(s));
}


void scale_points(const cmoe_gp& gp, const double* P, int m, DevBuf<double>& Ps, cudaStream_t s) {
  const int dim = gp.spec.dim;
  ensure_scaled_points(Ps, m, dim, s);
  scale_points_kernel<<<(m * dim + 255) / 256, 256, 0, s>>>(gp.spec, centre_of(gp), P, m, Ps.p);
  count_launch();
}

cmoe_gp* clone_gp_to_device(const cmoe_gp* src, int device) {
  require_device(device);
  std::unique_ptr<cmoe_gp> gp(new cmoe_gp());
  gp->device = device;
  gp->spec = src->spec;
  gp->N = src->N;
  gp->n = src->n;
  gp->mean = src->mean;
  gp->hX = src->hX;
  gp->hy = src->hy;
  gp->hnoise = src->hnoise;
  gp->hlengths = src->hlengths;
  std::copy(src->centre, src->centre + CMOE_MAX_DIM, gp->centre);
  gp->generation = src->generation;
  CMOE_CUDA(cudaStreamCreateWithFlags(&gp->stream, cudaStreamNonBlocking));
  cudaStream_t s = gp->stream;
  auto peer = [&](DevBuf<double>& dst, const DevBuf<double>& from, size_t count) {
    dst.ensure(std::max(count, from.count));
    if (count)
      CMOE_CUDA(cudaMemcpyPeerAsync(dst.p, device, from.p, src->device, std::min(count, from.count) * sizeof(double), s));
  };
  const size_t n = static_cast<size_t>(src->n);
  peer(gp->dX, src->dX, src->hX.size());
  peer(gp->dXs, src->dXs, src->dXs.count);
  peer(gp->dy, src->dy, src->hy.size());
  peer(gp->dnoise, src->dnoise, src->hnoise.size());
  peer(gp->dK, src->dK, n * n);
  peer(gp->dKinvY, src->dKinvY, n);
  gp->dFlag.alloc(1);
  CMOE_CUDA(cudaStreamSynchronize(s));
  return gp.release();
}

}  // namespace cmoe

cmoe_gp::~cmoe_gp() {
  for (cmoe_gp* r : replicas) cmoe_gp_destroy(r);
  replicas.clear();
  cmoe::drop_cached_plan(this);
  if (stream) {
    cudaSetDevice(device);
    cudaStreamDestroy(stream);
  }
}

using namespace cmoe;  // NOLINT

extern "C" {

const char* cmoe_last_error(void) { return g_last_error.c_str(); }
const char* cmoe_version(void) { return "cornell-moe_b200 0.1 (sm_90a)"; }

int cmoe_device_count(void) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return count;
}

int cmoe_gp_create(int kernel, double alpha, const double* lengths, const double* points_sampled,
                   const double* points_sampled_value, const double* noise_variance, const int* derivatives,
                   int num_derivatives, int dim, int num_sampled, int device, cmoe_gp** gp_out, int* info) {
  if (gp_out) *gp_out = nullptr;
  return guarded(info, [&] {
    CMOE_REQUIRE(gp_out != nullptr, CMOE_ERR_INVALID_VALUE, "gp_out is NULL");
    CMOE_REQUIRE(kernel == CMOE_KERNEL_SQUARE_EXPONENTIAL || kernel == CMOE_KERNEL_MATERN_NU_2P5,
                 CMOE_ERR_INVALID_VALUE, "unknown covariance kernel id");
    CMOE_REQUIRE(dim >= 1 && dim <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, CMOE_MAX_DIM]");
    CMOE_REQUIRE(num_sampled >= 1, CMOE_ERR_BOUNDS, "num_sampled must be >= 1");
    CMOE_REQUIRE(num_derivatives >= 0 && num_derivatives <= dim, CMOE_ERR_BOUNDS, "num_derivatives out of range");
    // hyperparameter validation as InitializeCovariance, gpp_covariance.cpp:74-98
    CMOE_REQUIRE(alpha > 0.0, CMOE_ERR_BOUNDS, "Invalid hyperparameter (alpha).");
    for (int k = 0; k < dim; ++k) CMOE_REQUIRE(lengths[k] > 0.0, CMOE_ERR_BOUNDS, "Invalid hyperparameter (length).");
    for (int k = 0; k < num_derivatives; ++k)
      CMOE_REQUIRE(derivatives[k] >= 0 && derivatives[k] < dim, CMOE_ERR_BOUNDS, "derivative index out of range");
    require_device(device);
    std::unique_ptr<cmoe_gp> gp(new cmoe_gp());
    gp->device = device;
    fill_kernel_spec(gp->spec, kernel, dim, num_derivatives, derivatives, alpha, lengths);
    gp->N = num_sampled;
    gp->hX.assign(points_sampled, points_sampled + static_cast<size_t>(num_sampled) * dim);
    gp->hy.assign(points_sampled_value,
                  points_sampled_value + static_cast<size_t>(num_sampled) * (1 + num_derivatives));
    gp->hnoise.assign(noise_variance, noise_variance + 1 + num_derivatives);
    gp->hlengths.assign(lengths, lengths + dim);
    CMOE_CUDA(cudaStreamCreateWithFlags(&gp->stream, cudaStreamNonBlocking));
    fit_gp(gp.get(), true);
    *gp_out = gp.release();
  });
}

// log p(y | X, theta): one GP fit with 1e-6 added to every noise entry, then two host reductions over n numbers.
int cmoe_log_marginal_likelihood(int kernel, double alpha, const double* lengths, const double* points_sampled,
                                 const double* points_sampled_value, const double* noise_variance,
                                 const int* derivatives, int num_derivatives, int dim, int num_sampled, int device,
                                 double* log_likelihood, int* info) {
  if (log_likelihood) *log_likelihood = 0.0;
  if (num_derivatives < 0 || noise_variance == nullptr || log_likelihood == nullptr) {
    return guarded(info, [&] { CMOE_REQUIRE(false, CMOE_ERR_INVALID_VALUE, "invalid argument"); });
  }
  std::vector<double> nz(noise_variance, noise_variance + 1 + num_derivatives);
  for (double& v : nz) v += 1.0e-6;  // gpp_model_selection.cpp:546-549
  cmoe_gp* gp = nullptr;
  int linfo = 0;
  const int rc = cmoe_gp_create(kernel, alpha, lengths, points_sampled, points_sampled_value, nz.data(), derivatives,
                                num_derivatives, dim, num_sampled, device, &gp, &linfo);
  if (rc == CMOE_ERR_SINGULAR) {
    // the reference ignores the failed factorisation and returns whatever the garbage factor gives (:551-553)
    *log_likelihood = -std::numeric_limits<double>::infinity();
    if (info) *info = linfo;
    return CMOE_OK;
  }
  if (rc != CMOE_OK) {
    if (info) *info = linfo;
    return rc;
  }
  const int out = guarded(info, [&] {
    require_device(gp->device);
    const int n = gp->n, bs = 1 + gp->spec.g;
    std::vector<double> diag(n), b(n);
    // diagonal of the column-major factor: n elements, (n+1) doubles apart
    CMOE_CUDA(cudaMemcpy2DAsync(diag.data(), sizeof(double), gp->dK.p, static_cast<size_t>(n + 1) * sizeof(double),
                                sizeof(double), n, cudaMemcpyDeviceToHost, gp->stream));
    gp->dKinvY.download(b.data(), n, gp->stream);
    CMOE_CUDA(cudaStreamSynchronize(gp->stream));
    double term1 = 0.0, term2 = 0.0;
    for (int i = 0; i < n; ++i) {
      const double yc = gp->hy[i] - ((i % bs == 0) ? gp->mean : 0.0);
      term1 += yc * b[i];
      term2 -= std::log(diag[i]);
    }
    const double kLog2Pi = 1.8378770664093453;
    *log_likelihood = -0.5 * term1 + term2 - 0.5 * static_cast<double>(n) * kLog2Pi;
  });
  cmoe_gp_destroy(gp);
  return out;
}

void cmoe_gp_destroy(cmoe_gp* gp) {
  if (!gp) return;
  cudaSetDevice(gp->device);
  delete gp;
}

int cmoe_set_option(const char* name, int value) {
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(set_option(name, value) == 0, CMOE_ERR_INVALID_VALUE, "unknown option name");
  });
}

int cmoe_gp_dim(const cmoe_gp* gp) { return gp->spec.dim; }
int cmoe_gp_device(const cmoe_gp* gp) { return gp->device; }
int cmoe_gp_num_sampled(const cmoe_gp* gp) { return gp->N; }
int cmoe_gp_num_derivatives(const cmoe_gp* gp) { return gp->spec.g; }

int cmoe_gp_get_state(const cmoe_gp* gp, double* K_chol, double* K_inv_y, double* mean) {
  return guarded(nullptr, [&] {
    require_device(gp->device);
    const int n = gp->n;
    if (K_chol) {
      gp->dK.download(K_chol, static_cast<size_t>(n) * n, gp->stream);
      CMOE_CUDA(cudaStreamSynchronize(gp->stream));
      for (int j = 1; j < n; ++j)  // strictly-upper part is undefined on the device (never written): report zeros
        std::fill(K_chol + static_cast<size_t>(j) * n, K_chol + static_cast<size_t>(j) * n + j, 0.0);
    }
    if (K_inv_y) {
      gp->dKinvY.download(K_inv_y, n, gp->stream);
      CMOE_CUDA(cudaStreamSynchronize(gp->stream));
    }
    if (mean) *mean = gp->mean;
  });
}

int cmoe_gp_add_sampled_points(cmoe_gp* gp, const double* new_points, const double* new_points_value,
                               int num_new_points, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_new_points >= 0, CMOE_ERR_BOUNDS, "num_new_points must be >= 0");
    require_device(gp->device);
    if (num_new_points == 0) return;
    append_points(gp, new_points, new_points_value, num_new_points);
  });
}

int cmoe_gp_fit_timings(const cmoe_gp* gp, double* usec3) {
  for (int i = 0; i < 3; ++i) usec3[i] = gp->fit_usec[i];
  return CMOE_OK;
}

int cmoe_bench_cov_build(const cmoe_gp* gp, int repeats, double* usec_per_build) {
  return guarded(nullptr, [&] {
    require_device(gp->device);
    DevBuf<double> scratch(static_cast<size_t>(gp->n) * gp->n);
    cudaStream_t s = gp->stream;
    build_covariance(gp->spec, gp->dX.p, gp->dXs.p, gp->N, gp->dnoise.p, scratch.p, s);  // warm-up
    EventTimer t;
    t.start(s);
    for (int r = 0; r < repeats; ++r) build_covariance(gp->spec, gp->dX.p, gp->dXs.p, gp->N, gp->dnoise.p, scratch.p, s);
    t.stop(s);
    *usec_per_build = t.ms() * 1e3 / repeats;
  });
}

int cmoe_bench_cholesky(const cmoe_gp* gp, int repeats, double* usec_per_factor) {
  return guarded(nullptr, [&] {
    require_device(gp->device);
    const size_t nn = static_cast<size_t>(gp->n) * gp->n;
    DevBuf<double> K0(nn), work(nn);
    DevBuf<int> flag(1);
    cudaStream_t s = gp->stream;
    if (gp->spec.g > 0) K0.zero(s);
    build_covariance(gp->spec, gp->dX.p, gp->dXs.p, gp->N, gp->dnoise.p, K0.p, s);
    double total = 0.0;
    for (int r = 0; r < repeats + 1; ++r) {
      CMOE_CUDA(cudaMemcpyAsync(work.p, K0.p, nn * sizeof(double), cudaMemcpyDeviceToDevice, s));
      EventTimer t;
      t.start(s);
      potrf_lower(work.p, gp->n, flag.p, s);
      t.stop(s);
      if (r > 0) total += t.ms();
    }
    *usec_per_factor = total * 1e3 / repeats;
  });
}

int cmoe_cholesky(int n, double* a, int device, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(n >= 1, CMOE_ERR_BOUNDS, "n must be >= 1");
    require_device(device);
    cudaStream_t s;
    CMOE_CUDA(cudaStreamCreate(&s));
    const size_t nn = static_cast<size_t>(n) * n;
    DevBuf<double> A(nn);
    DevBuf<int> flag(1);
    A.upload(a, nn, s);
    potrf_lower(A.p, n, flag.p, s);
    int f = 0;
    CMOE_CUDA(cudaMemcpyAsync(&f, flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    // copy back only the lower triangle; like the reference the strictly-upper part keeps the caller's input
    std::vector<double> tmp(nn);
    A.download(tmp.data(), nn, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    cudaStreamDestroy(s);
    if (f != 0) throw Error(CMOE_ERR_SINGULAR, "cholesky matrix singular", f);
    for (int j = 0; j < n; ++j)
      for (int i = j; i < n; ++i) a[static_cast<size_t>(j) * n + i] = tmp[static_cast<size_t>(j) * n + i];
  });
}

int cmoe_potrs(int n, int nrhs, const double* chol, double* x, int device) {
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(n >= 1 && nrhs >= 0, CMOE_ERR_BOUNDS, "bad sizes");
    require_device(device);
    cudaStream_t s;
    CMOE_CUDA(cudaStreamCreate(&s));
    DevBuf<double> L(static_cast<size_t>(n) * n), X(static_cast<size_t>(n) * nrhs);
    L.upload(chol, static_cast<size_t>(n) * n, s);
    X.upload(x, static_cast<size_t>(n) * nrhs, s);
    potrs_lower(L.p, n, X.p, n, nrhs, s);
    X.download(x, static_cast<size_t>(n) * nrhs, s);
    CMOE_CUDA(cudaStreamSynchronize(s));
    cudaStreamDestroy(s);
  });
}

int cmoe_philox_normals(uint64_t seed, uint64_t first_draw, int num_draws, int per_draw, double* out, int device) {
  return guarded(nullptr, [&] {
    require_device(device);
    DevBuf<double> d(static_cast<size_t>(num_draws) * per_draw);
    philox_normals_device(seed, first_draw, num_draws, per_draw, d.p, 0);
    CMOE_CUDA(cudaMemcpy(out, d.p, d.count * sizeof(double), cudaMemcpyDeviceToHost));
  });
}

}  // extern "C"

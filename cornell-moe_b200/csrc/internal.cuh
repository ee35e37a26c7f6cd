// Internal declarations shared by the CUDA translation units of libcornell_moe_b200.so.
// Everything here is host-side C++ plumbing around hand-written sm_90a kernels; there is no CPU compute path.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/cmoe_b200.h"

namespace cmoe {

// ---------------------------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------------------------
struct Error : public std::runtime_error {
  int code;
  int info;
  Error(int code_in, const std::string& msg, int info_in = 0) : std::runtime_error(msg), code(code_in), info(info_in) {}
};

void set_last_error(const std::string& msg);

#define CMOE_CUDA(call)                                                                                  \
  do {                                                                                                   \
    cudaError_t err__ = (call);                                                                          \
    if (err__ != cudaSuccess) {                                                                          \
      char buf__[512];                                                                                   \
      snprintf(buf__, sizeof(buf__), "%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(err__)); \
      throw ::cmoe::Error(CMOE_ERR_RUNTIME, buf__);                                                      \
    }                                                                                                    \
  } while (0)

// a macro's value as a string literal
#define CMOE_STR_(x) #x
#define CMOE_STR(x) CMOE_STR_(x)

#define CMOE_REQUIRE(cond, code, msg)                 \
  do {                                                \
    if (!(cond)) throw ::cmoe::Error((code), (msg)); \
  } while (0)

// Runs f(), translating exceptions into the C-ABI status codes.
template <class F>
int guarded(int* info, F&& f) {
  try {
    if (info) *info = 0;
    cudaGetLastError();  // a non-sticky error left behind by an earlier, unrelated call must not fail this one
    f();
    return CMOE_OK;
  } catch (const Error& e) {
    set_last_error(e.what());
    if (info) *info = e.info;
    return e.code;
  } catch (const std::exception& e) {
    set_last_error(e.what());
    return CMOE_ERR_RUNTIME;
  }
}

void require_device(int device);  // throws CMOE_ERR_NO_DEVICE / CMOE_ERR_BOUNDS

// ---------------------------------------------------------------------------------------------------------------
// device memory
// ---------------------------------------------------------------------------------------------------------------
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t count = 0;
  DevBuf() = default;
  explicit DevBuf(size_t n) { alloc(n); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), count(o.count) { o.p = nullptr; o.count = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; count = o.count; o.p = nullptr; o.count = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void alloc(size_t n) {
    release();
    count = n;
    if (n) CMOE_CUDA(cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T)));
  }
  void ensure(size_t n) { if (n > count) alloc(n); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    count = 0;
  }
  void upload(const T* host, size_t n, cudaStream_t s) {
    ensure(n);
    if (n) CMOE_CUDA(cudaMemcpyAsync(p, host, n * sizeof(T), cudaMemcpyHostToDevice, s));
  }
  void download(T* host, size_t n, cudaStream_t s) const {
    if (n) CMOE_CUDA(cudaMemcpyAsync(host, p, n * sizeof(T), cudaMemcpyDeviceToHost, s));
  }
  void zero(cudaStream_t s) { if (count) CMOE_CUDA(cudaMemsetAsync(p, 0, count * sizeof(T), s)); }
};

struct EventTimer {
  cudaEvent_t a = nullptr, b = nullptr;
  EventTimer() { cudaEventCreate(&a); cudaEventCreate(&b); }
  ~EventTimer() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
  void start(cudaStream_t s) { cudaEventRecord(a, s); }
  void stop(cudaStream_t s) { cudaEventRecord(b, s); }
  float ms() { float t = 0.f; cudaEventSynchronize(b); cudaEventElapsedTime(&t, a, b); return t; }
};

// ---------------------------------------------------------------------------------------------------------------
// covariance kernel description, passed by value to every kernel
// ---------------------------------------------------------------------------------------------------------------
struct KernelSpec {
  int kernel;  // CMOE_KERNEL_*
  int dim;
  int g;       // number of derivative observations per sampled point
  double alpha;
  double lsq[CMOE_MAX_DIM];      // l_k^2
  double inv_len[CMOE_MAX_DIM];  // 1 / l_k
  int derivs[CMOE_MAX_DIM];      // observed partial-derivative indices of the training data
};

// ---------------------------------------------------------------------------------------------------------------
// the GP handle
// ---------------------------------------------------------------------------------------------------------------
}  // namespace cmoe

struct cmoe_gp {
  int device = 0;
  cmoe::KernelSpec spec{};
  int N = 0;  // points
  int n = 0;  // rows = N * (1 + g)
  double mean = 0.0;
  std::vector<double> hX, hy, hnoise, hlengths;
  // mean of the training points: the origin of dXs and of every q-KG operand (scaled coordinates are (x - centre) / l)
  double centre[CMOE_MAX_DIM] = {};
  cudaStream_t stream = nullptr;
  cmoe::DevBuf<double> dX;        // [N][dim]
  cmoe::DevBuf<double> dXs;       // [N][dim] (x - centre) / l (the fast covariance build)
  cmoe::DevBuf<double> dy;        // [n]
  cmoe::DevBuf<double> dnoise;    // [1+g]
  cmoe::DevBuf<double> dK;        // [n*n] column-major Cholesky factor (lower)
  cmoe::DevBuf<double> dKinvY;    // [n]
  cmoe::DevBuf<int> dFlag;        // [1] Cholesky failure index
  double fit_usec[3] = {0, 0, 0};
  uint64_t generation = 0;  // bumped by every (re)fit / append: explicit q-KG plans are bound to one generation
  // one cached q-KG plan (device workspace) so that repeated cmoe_kg_eval calls with the same configuration — every
  // step of an outer optimiser — do not re-allocate gigabytes of scratch; owned by kg.cu
  mutable struct cmoe_kg_plan* cached_plan = nullptr;
  // replicas of this GP on other devices (multi-GPU multistart inside one call); rebuilt when the generation changes
  mutable std::vector<cmoe_gp*> replicas;
  // device workspace of the joint-sampling calls (sample.cu), grown on demand and kept until the handle is destroyed
  mutable std::shared_ptr<void> sample_ws;
  // device workspace of the large-union evaluations (kg_large.cu, ei_large.cu) whose first member is this handle
  // (cmoe::LargeUnionWork), grown on demand up to one evaluation's need and kept until the handle is destroyed
  mutable std::shared_ptr<void> large_union_ws;
  mutable uint64_t replicas_generation = 0;
  ~cmoe_gp();
};

namespace cmoe {

constexpr int kTrsmNB = 32;
// largest grid.y (and grid.z) of a launch; the batched drivers that put one candidate per blockIdx.y split at this size
constexpr size_t kMaxGridY = 65535;

// ---- gp.cu ----
// the origin of the covariance-build frame (cmoe_gp::centre) as a kernel argument
struct Centre {
  double c[CMOE_MAX_DIM];
};
inline Centre centre_of(const cmoe_gp& gp) {
  Centre c{};
  for (int d = 0; d < CMOE_MAX_DIM; ++d) c.c[d] = gp.centre[d];
  return c;
}
void fit_gp(cmoe_gp* gp, bool mean_change);
// s <- the KernelSpec of (alpha, lengths[dim]) with derivative indices derivs[g]; entries past dim and g are l = 1,
// 1/l = 0 and index 0.  In place: the list calls fill one per set.
void fill_kernel_spec(KernelSpec& s, int kernel, int dim, int g, const int* derivs, double alpha,
                      const double* lengths);
// O(N^2) append of m points and their values [m][1+g]; the new rows' diagonal carries new_noise [1+g] (host), or the
// GP's own noise when it is NULL.  A singular update throws CMOE_ERR_SINGULAR and leaves the handle intact.
void append_points(cmoe_gp* gp, const double* new_points, const double* new_values, int m,
                   const double* new_noise = nullptr);
// bit-identical copy of a fitted GP on another device (peer copies of the factor; no refit)
cmoe_gp* clone_gp_to_device(const cmoe_gp* gp, int device);
// Ps <- the m points P (device) in the length-scaled, centred coordinates of gp's covariance build (the Xs argument of
// build_covariance), exactly as append_points scales the points it adds; Ps is padded as build_covariance needs.
void scale_points(const cmoe_gp& gp, const double* P, int m, DevBuf<double>& Ps, cudaStream_t s);
// ---- kg.cu ----
void drop_cached_plan(const cmoe_gp* gp);

// ---- linalg.cu -----------------------------------------------------------------------------------------------
// In-place blocked lower Cholesky of the n*n column-major matrix A (lda = n).  *flag (device) receives 0 or the
// failing leading-minor index (k+1), with the reference's pivot test (> 1e-16).  Enqueued on `s` (large systems also
// use an internal side stream for the look-ahead update); returns after the factorisation has completed.
void potrf_lower(double* A, int n, int* flag, cudaStream_t s);
// potrf_coop.cu: one cooperative launch per 256-column panel (n >= 1024, even); false = not applicable, A untouched
bool potrf_lower_coop(double* A, int n, int* flag, cudaStream_t s);
// X <- (L L^T)^-1 X for nrhs right-hand sides; X is n*nrhs column-major with leading dimension ldx.
void potrs_lower(const double* L, int n, double* X, int ldx, int nrhs, cudaStream_t s);
// X <- L^-1 X (trans = false) or L^-T X (trans = true).  nrhs <= 4 with n >= 1024 takes the single-launch chained
// solver (which synchronises `s`); everything else is trsm_lower_blocked.
void trsm_lower(const double* L, int n, double* X, int ldx, int nrhs, bool trans, cudaStream_t s);
// The blocked multi-RHS kernel for any nrhs, asynchronous on `s`: one CTA per 32 columns, and each column's result
// depends only on that column, so a column comes out the same however many columns share the call.
void trsm_lower_blocked(const double* L, int n, double* X, int ldx, int nrhs, bool trans, cudaStream_t s);
// trsv_coop.cu: one cooperative launch, owner + helper CTAs per 128-unknown block row; false = not applicable / gave up
bool trsv_coop(const double* L, int n, double* x, bool trans, cudaStream_t s);
bool trsv_coop_pair(const double* L, int n, double* x, cudaStream_t s);

// ---- sample.cu: batched blocked Cholesky (DESIGN.md K8) -------------------------------------------------------
constexpr int kMaxSampleQ = 8192;                          // rows of one set's matrix
constexpr size_t kSampleWorkspaceBytes = size_t(2) << 30;  // device workspace of one chunk (or of one set, if larger)
// sets per chunk: one CTA row per set on grid.y / grid.z of the per-set launches (cov_tile, batched Cholesky,
// sample_rows, lhs, the likelihood list), well inside their 65535.  It does not bound the chunk's points:
// build_mix_covariance puts those on grid.x.
constexpr int kMaxChunkSets = 4096;
// In-place lower Cholesky of nsets Q x Q column-major matrices (only the lower triangle is read); fail[nsets] must be
// zero on entry and receives 0 or the 1-based leading minor of the first pivot that fails `> 1e-16`.  `stage` holds the
// diagonal factors until the end (nsets * ceil(Q/64) * 64 * 64 doubles).  Asynchronous on `s`.
void potrf_batched(double* A, int Q, int nsets, int* fail, DevBuf<double>& stage, cudaStream_t s);
// the same with the caller's stage buffer (at least nsets * ceil(Q/64) * 64 * 64 doubles)
void potrf_batched(double* A, int Q, int nsets, int* fail, double* stage, cudaStream_t s);
// Device workspace of the sampling calls and of the LCB screen (lcb.cu), kept on the GP handle (cmoe_gp::sample_ws) and
// grown on demand, so repeated calls do not allocate and free up to kSampleWorkspaceBytes each time.  Released with the
// handle.
struct SampleWork {
  DevBuf<double> P, V, A, mu, y, part_v, opt, stage, table;
  DevBuf<int> dPs, fail, part_i, amin;
};
// the handle's SampleWork, created on first use
inline SampleWork& sample_work(const cmoe_gp& gp) {
  if (!gp.sample_ws) gp.sample_ws = std::make_shared<SampleWork>();
  return *static_cast<SampleWork*>(gp.sample_ws.get());
}
// The K8 posterior stages for the nc sets whose points are in w.P (num points, gs derivative rows dPs = w.dPs each,
// Q = num (1 + gs) <= 8192): V = L^-1 K(X, P) in w.V (n x nc Q, ld n), the mean in w.mu and the lower triangle of
// Var = K(P, P) - V^T V + jitter I in w.A ([nc][Q][Q] column-major; the upper triangle is not written).  Asynchronous.
void posterior_cov_large(const cmoe_gp& gp, SampleWork& w, int nc, int num, int gs, double jitter, cudaStream_t s);
// the same on the caller's buffers (P, dPs read; V, mu, A written)
void posterior_cov_large(const cmoe_gp& gp, const double* P, const int* dPs, double* V, double* mu, double* A, int nc,
                         int num, int gs, double jitter, cudaStream_t s);
// upper triangle of nsets Q x Q column-major matrices <- 0 (zero_upper) or <- the lower triangle (mirror_lower)
void zero_upper(int nsets, int Q, double* A, cudaStream_t s);
void mirror_lower(int nsets, int Q, double* A, cudaStream_t s);

// Items per chunk of a batched call: as many as fit in `budget` bytes at `bytes_per_item` each, at most `total` and
// `cap` (a grid-dimension or set-count limit), and at least one.
inline size_t chunk_items(size_t total, size_t budget, size_t bytes_per_item, size_t cap = SIZE_MAX) {
  return std::max<size_t>(1, std::min<size_t>({total, budget / bytes_per_item, cap}));
}

// streaming multiprocessors of the current device
inline int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// Step size of gradient-descent iteration i (from 0): pre_mult (i + 1)^-gamma, gpp_optimization.hpp:736
inline double gd_step_size(double pre_mult, double gamma, int i) {
  return pre_mult * std::pow(static_cast<double>(i + 1), -gamma);
}

// ---- lcb.cu: LCB batch selection (DESIGN.md K13) ----------------------------------------------------------------
// rows of the selected-set block, (q - 1)(1 + g): its bordered factor is built by one CTA, round by round
constexpr int kMaxLcbSelectedRows = 1024;
// the rounds' per-candidate vectors w(x), C' (q - 1)(1 + g) doubles, are held in one workspace-sized buffer
constexpr size_t kMaxLcbRoundDoubles = kSampleWorkspaceBytes / sizeof(double);

// ---- posterior.cu -------------------------------------------------------------------------------------------
constexpr int kMaxQ = CMOE_MAX_SET_ROWS;  // largest (q+p)*(1+num_derivatives) handled by the per-set kernels

// Device-resident posterior quantities for a batch of nc point sets (num points each, gs derivative rows per point).
struct PosteriorBatch {
  int nc = 0, num = 0, gs = 0, Q = 0, nd = 0, n = 0, dim = 0;
  DevBuf<double> P;      // [nc][num][dim]   (filled by the caller before run())
  DevBuf<int> dPs;       // [gs]
  DevBuf<double> Ks, B;  // [n][nc*Q] column-major: K* and K^-1 K*
  DevBuf<double> mu;     // [nc][Q]
  DevBuf<double> var;    // [nc][Q*Q]
  DevBuf<double> chol;   // [nc][Q*Q] Cholesky of (var + diagonal term), upper triangle zeroed
  DevBuf<double> gmu;    // [nc][nd*(1+gs)][dim]
  DevBuf<double> E;      // [nc][nd*(1+gs)][Q][dim]
  DevBuf<double> gvar;   // [nc][nd][Q][Q][dim]
  DevBuf<double> gchol;  // [nc][nd][Q][Q][dim]
  DevBuf<int> fail;      // [nc]
  void configure(const cmoe_gp& gp, int nc, int num, const int* dPs_host, int gs, int nd, cudaStream_t s);
  // diag_mode: 0 none, 1 +1e-6 (EI), 2 +noise_variance[type] (KG)
  void run(const cmoe_gp& gp, int diag_mode, bool want_chol, bool want_grad_chol, cudaStream_t s);
  int first_failure(cudaStream_t s, int* which_set);
};

// Mean (and, if gmu != NULL, its gradient) at npts independent points of P [npts][dim] with the derivative rows
// dPs[gs] (device): mu [npts][1+gs], gmu [npts][1+gs][dim].  No K^-1 K*, no bound on the number of points.
void posterior_mean_points(const cmoe_gp& gp, const double* P, size_t npts, const int* dPs, int gs, double* mu,
                           double* gmu, cudaStream_t s);

// ---- multistart.cu -------------------------------------------------------------------------------------------
constexpr int kTopK = 20;  // hard-coded in the reference (gpp_knowledge_gradient_optimization.hpp:901, gpp_math.hpp:1765)
// indices of the (up to) kTopK largest values, in the order the reference feeds them to the optimiser
std::vector<int> top_k_indices(const double* values, int n);
// closed-form one-point EI (gpp_math.cpp:2196-2253) at nc points [nc][dim] and, if grads is not NULL, its gradient
// [nc][dim], from cmoe_gp_posterior's mean and variance
void analytic_ei(const cmoe_gp* gp, const double* pts, int nc, double best_so_far, double* values, double* grads);
// throws CMOE_ERR_BOUNDS for a tensor-product box [dim][2] with min > max in some dimension
void validate_bounds(const double* b, int dim);
// An ensemble (one GP per hyper-parameter sample) is non-empty and its members share dim, g and device.
void check_ensemble(const cmoe_gp* const* gps, int num_gp);
// Member m's values v[nc] and gradients g[nc][ps] (g, grads NULL: none) into the ensemble's sums, called in member
// order: member 0's start the sums (its own bits, so a one-member sum is the member's result), later members are added.
void add_member(int m, int nc, size_t ps, const double* v, const double* g, double* values, double* grads);

// The evaluation path of a union of q candidate and p pending points.  q-KG past CMOE_MAX_KG_ROWS rows,
// (q + p)(1 + g), runs the large-union stages of kg_large.cu instead of the plans of kg.cu; q-EI past kMaxQ rows runs
// the tiles of ei_large.cu instead of the per-set kernels of ei.cu.
inline bool kg_union_is_large(int q, int p, int g) {
  return static_cast<long long>(q + p) * (1 + g) > CMOE_MAX_KG_ROWS;
}
inline bool ei_union_is_large(int q, int p) { return q + p > kMaxQ; }

// ---- kg.cu ---------------------------------------------------------------------------------------------------
// P [nc][q + p][dim] <- each candidate's q points, then the p pending points.  Asynchronous on `s`.
void build_union_sets(const double* cand, const double* Xp, int nc, int q, int p, int dim, double* P, cudaStream_t s);

// ---- ei.cu ---------------------------------------------------------------------------------------------------
void upload_union_sets(PosteriorBatch& pb, const double* candidates, int nc, int q, const double* Xp, int p, int dim,
                       cudaStream_t s);
void ei_eval_batch(const cmoe_gp& gp, const double* candidates, int nc, int q, const double* Xp, int p, int num_mc,
                   double best_so_far, uint64_t seed, const double* dtable, double* ei_host, double* grad_host);
// ---- the large-union stages: one evaluation of an ensemble of num_gp >= 1 GPs (a single GP is the one-member ensemble)
// values[nc] and grads[nc][q][dim] (or NULL) receive the members' results summed in member order; with one member they
// are that member's own.  The draws are made once per evaluation and shared by every member.  The evaluation's device
// workspace is at most 2 GiB, on gps[0]'s handle (large_union_work).  A singular union throws CMOE_ERR_SINGULAR with
// the leading minor of the first failing candidate of the first failing member.
// kg_large.cu: cmoe_kg_eval for 1 <= (q + p)(1 + g) <= CMOE_MAX_KG_LARGE_ROWS (DESIGN.md K17, K18).  normals_table:
// host ((num_mc + 1) / 2) (q + p)(1 + g) values or NULL (Philox); stale_union (q points or NULL): the discretisation
// set's union part keeps these q points (the reference drivers' quirk, cmoe_kg_plan_set_stale_union); stats (or NULL)
// receives the members' counters summed.
void kg_large_eval(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* inner,
                   const double* inner_bounds, const double* discrete_pts, int num_pts, const double* candidates,
                   int num_candidates, int q, const double* points_being_sampled, int p, int num_mc,
                   const double* best_so_far, uint64_t seed, const double* normals_table, const double* stale_union,
                   double* values, double* grads, cmoe_kg_stats* stats);
// ei_large.cu: the q-EI of ei.cu for 1 <= q + p <= kMaxSampleQ (DESIGN.md K16, K18).  dtable: device [num_mc][q + p]
// or NULL (Philox).
void ei_large_eval(const cmoe_gp* const* gps, int num_gp, const double* candidates, int num_candidates, int q,
                   const double* points_being_sampled, int p, int num_mc, const double* best_so_far, uint64_t seed,
                   const double* dtable, double* values, double* grads);
// Consecutive 256-byte aligned pieces of one device region (the large-union stages' workspaces); with base == NULL it
// only counts the bytes.
struct Carve {
  char* base = nullptr;
  size_t off = 0;
  template <typename T>
  T* take(size_t count) {
    off = (off + 255) & ~size_t(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};
// Bound on the alignment padding of one carved chunk workspace (at most 64 pieces of up to 255 bytes each): a chunk of
// c candidates takes at most c times the one-candidate layout plus kCarveSlack.
constexpr size_t kCarveSlack = 64 * 256;
// CMOE_ERR_SINGULAR for a singular union covariance, *info = minor (the 1-based leading minor that failed)
[[noreturn]] void throw_singular_union(int minor);
// The region the large-union evaluations above carve their buffers from, on the first member's handle, and one event
// per member.  Every evaluation ends with its members' streams synchronised, so the next one may reuse the region.
struct LargeUnionWork {
  DevBuf<double> arena;
  std::vector<cudaEvent_t> done;
  LargeUnionWork() = default;
  LargeUnionWork(const LargeUnionWork&) = delete;
  LargeUnionWork& operator=(const LargeUnionWork&) = delete;
  ~LargeUnionWork();
};
// gp's LargeUnionWork with an arena of at least `bytes` (grown by replacement, never kept larger than one evaluation's
// need)
LargeUnionWork& large_union_work(const cmoe_gp& gp, size_t bytes);
// gp's LargeUnionWork with the arena laid out by layout(Carve&): called once to measure, once more to carve the arena
template <class Layout>
LargeUnionWork& carve_large_union_work(const cmoe_gp& gp, Layout&& layout) {
  Carve cv;
  layout(cv);
  LargeUnionWork& w = large_union_work(gp, cv.off);
  cv = Carve{reinterpret_cast<char*>(w.arena.p)};
  layout(cv);
  return w;
}
// How many members run at once and how many candidates each runs per chunk.  `avail` bytes hold the members' slots; a
// slot is a chunk at `per` bytes per candidate, kCarveSlack for alignment and, after the chunk, whatever the caller
// splits evenly between the slots.  width_cap bounds the members in flight further, as does
// cmoe_set_option("ensemble_members_in_flight").
struct MemberSchedule {
  int width, chunk;
};
MemberSchedule schedule_members(int num_gp, int num_candidates, size_t avail, size_t per, size_t width_cap = SIZE_MAX);
// bytes of one member's slot: the largest member's chunk workspace, rounded up so that every slot starts aligned
inline size_t slot_stride(size_t bytes) { return (bytes + 255) & ~size_t(255); }
// Enqueues run(m, m % width) for m = 0 .. num_gp - 1 on member m's stream; member m waits for member m - width, whose
// slot it reuses.  Returns once every member's stream has finished, also when run throws.
void run_members(const cmoe_gp* const* gps, int num_gp, int width, LargeUnionWork& w,
                 const std::function<void(int, int)>& run);
// Reads back the members' device results dval [num_gp][nc], dgrad [num_gp][nc][ps] (or NULL) and dfail [num_gp][nc] on
// `s`; throws CMOE_ERR_SINGULAR for the first failing member in member order, else sums the members in member order
// (add_member).
void drain_members(cudaStream_t s, int num_gp, int nc, size_t ps, const double* dval, const double* dgrad,
                   const int* dfail, double* values, double* grads);
// Out = A B for `batch` column-major problems (A m x kd, B kd x nn; batch z at A + z sa, B + z sb, Out + z so), 64 x 64
// DMMA tiles.  Asynchronous on `s`.
void gemm_nn(int m, int nn, int kd, const double* A, int lda, size_t sa, const double* B, int ldb, size_t sb,
             double* Out, int ldo, size_t so, int batch, cudaStream_t s);
// out = in^T for `batch` column-major rows x cols matrices, stored back to back (out: cols x rows).  Asynchronous on `s`.
void transpose_batched(int rows, int cols, const double* in, double* out, int batch, cudaStream_t s);
// Reverse mode through nc Cholesky factors C (U x U, column-major, upper triangle zero): T1 holds Cbar on entry (the
// adjoint of C, lower triangle) and 2 Sigmabar on exit, Sigmabar the adjoint of Sigma = C C^T (symmetric).  T2 is
// scratch of the same size.  Asynchronous on `s`.
void cholesky_adjoint(const double* C, int U, int nc, double* T1, double* T2, cudaStream_t s);

// ---- cov.cu --------------------------------------------------------------------------------------------------
// Lower triangle of K(X,X) + diag(noise by observation type), n*n column-major.
// Xs = X scaled by 1/l (used by the g == 0 fast path).
void build_covariance(const KernelSpec& spec, const double* X, const double* Xs, int N, const double* noise, double* K,
                      cudaStream_t s);
// K(X, P): rows = sampled rows (N*(1+g)), cols = P rows (num*(1+gs)); column-major, ld = n.
void build_mix_covariance(const KernelSpec& spec, const double* X, int N, const double* P, int num, const int* dPs,
                          int gs, double* out, cudaStream_t s);

// device-side Philox table for tests
void philox_normals_device(uint64_t seed, uint64_t first_draw, int num_draws, int per_draw, double* out,
                           cudaStream_t s);

// CMOE_LEGACY_LINALG=1 routes the large-N fit through the round-1 kernels (launch-per-step Cholesky, chained trsv,
// LDGSTS covariance build): an A/B switch for profiling, and a fall-back should a device mis-handle cooperative launches
bool legacy_linalg();
// CMOE_COV_TMA=1 builds K(X,X) with the TMA / DMMA kernel (tile stores through a tensor map); off by default: at d = 10
// it measures 62 us against 52 us for the LDGSTS kernel (see DESIGN.md K1)
bool cov_tma_enabled();
int set_option(const char* name, int value);
// cmoe_set_option("ensemble_members_in_flight", k): at most k ensemble members in flight on the large-union stages
// (0, the default: as many as the 2 GiB workspace holds)
int ensemble_members_in_flight();

int launches_issued();        // global counter of kernel launches made by this library (host side)
void count_launch(int n = 1);

}  // namespace cmoe

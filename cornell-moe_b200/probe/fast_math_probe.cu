// Device probe of the hand-written math routines that replace the CUDA math library in the kernels, for
// tests/test_gpu_fast_math.py.  Each thread evaluates one argument by calling the product's own header function, after
// staging its table exactly as the product kernels do.  Not part of the product library or its C header.
//
//   int cmoe_probe_eval(int routine, const double* in, long long n, double* out, int device)
//
// in and out are host arrays: in holds n arguments (n (p, a) pairs for the pivot step, n (t, H) pairs for
// exp2k_shifted), out receives n results of
// kProbeOut[routine] doubles each (see ProbeRoutine).  Returns 0, or -1 for an unknown routine / bad size, or the
// cudaError_t of the first CUDA call that failed.
#include <cuda_runtime.h>

#include "device_math.cuh"
#include "kg_mc.cuh"
#include "linalg_dev.cuh"

namespace {

enum ProbeRoutine {
  kExpFast = 0,     // exp_fast(t)                                 -> 1 double
  kExpTab = 1,      // exp_tab(t), g_exp_tab staged                -> 1
  kExpTab2k = 2,    // exp_tab2k(t), g_exp_tab2k staged            -> 1
  kExpTabCov = 3,   // exp_tab_cov(t, tab), kCovExp2Table staged   -> 1
  kSincos = 4,      // rff_sincos(a)                               -> (sin, cos)
  kSqrtRsqrt = 5,   // sqrt_rsqrt(p)                               -> (l, y)
  kPivotFast = 6,   // chol_pivot_fast(p, a), chol_pivot_recip     -> (l, q, 1/l)
  kExp2kShifted = 7,  // exp2k_shifted(t, 1.5 2^52 + H), table staged -> (value, n, k) of its shifted double
  kExpTab2kNk = 8,    // exp_tab2k's shifted double of t               -> (n, k)
  kNumRoutines = 9,
};
constexpr int kProbeIn[kNumRoutines] = {1, 1, 1, 1, 1, 1, 2, 2, 1};
constexpr int kProbeOut[kNumRoutines] = {1, 1, 1, 1, 2, 2, 3, 3, 2};
constexpr int kProbeThreads = 256;
// cov.cu's kCovExp2Table (it lives in that translation unit only), from the same file
__device__ const double kCovExp2Table[64] = {
#include "exp2_table64.inc"
};

__global__ void __launch_bounds__(kProbeThreads) probe_kernel(int routine, const double* __restrict__ in, long long n,
                                                              double* __restrict__ out) {
  __shared__ double cov_tab[64];
  // staging: block-uniform, every thread reaches the barriers
  if (routine == kExpTab) cmoe::exp_table_stage();
  if (routine == kExpTab2k || routine == kExp2kShifted) cmoe::exp_table2k_stage();
  if (routine == kExpTabCov) {
    if (threadIdx.x < 64) cov_tab[threadIdx.x] = kCovExp2Table[threadIdx.x];
    __syncthreads();
  }
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  switch (routine) {
    case kExpFast: out[i] = cmoe::exp_fast(in[i]); break;
    case kExpTab: out[i] = cmoe::exp_tab(in[i]); break;
    case kExpTab2k: out[i] = cmoe::exp_tab2k(in[i]); break;
    case kExpTabCov: out[i] = cmoe::exp_tab_cov(in[i], cov_tab); break;
    case kSincos: cmoe::rff_sincos(in[i], out[2 * i], out[2 * i + 1]); break;
    case kSqrtRsqrt: cmoe::sqrt_rsqrt(in[i], out[2 * i], out[2 * i + 1]); break;
    case kPivotFast:
      cmoe::chol_pivot_fast(in[2 * i], in[2 * i + 1], out[3 * i], out[3 * i + 1]);
      out[3 * i + 2] = cmoe::chol_pivot_recip(in[2 * i], out[3 * i]);
      break;
    case kExp2kShifted: {
      // n = round(t + H) (its low word) and k = n >> 11, clamped, as exp2k_shifted forms them
      const double t = in[2 * i], C = cmoe::kExp2kShift + in[2 * i + 1], nfs = t + C;
      out[3 * i] = cmoe::exp2k_shifted(t, C);
      out[3 * i + 1] = __double2loint(nfs);
      out[3 * i + 2] = cmoe::exp2k_exponent(nfs);
      break;
    }
    case kExpTab2kNk: {
      const double nfs = cmoe::exp_tab2k_round(in[i]);
      out[2 * i] = __double2loint(nfs);
      out[2 * i + 1] = cmoe::exp2k_exponent(nfs);
      break;
    }
    default: break;
  }
}

}  // namespace

extern "C" int cmoe_probe_eval(int routine, const double* in, long long n, double* out, int device) {
  if (routine < 0 || routine >= kNumRoutines || n < 0 || n > (1LL << 30)) return -1;
  if (n == 0) return 0;
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return static_cast<int>(e);
  const size_t in_bytes = sizeof(double) * kProbeIn[routine] * n, out_bytes = sizeof(double) * kProbeOut[routine] * n;
  double *din = nullptr, *dout = nullptr;
  if ((e = cudaMalloc(&din, in_bytes)) == cudaSuccess && (e = cudaMalloc(&dout, out_bytes)) == cudaSuccess &&
      (e = cudaMemcpy(din, in, in_bytes, cudaMemcpyHostToDevice)) == cudaSuccess) {
    const unsigned blocks = static_cast<unsigned>((n + kProbeThreads - 1) / kProbeThreads);
    probe_kernel<<<blocks, kProbeThreads>>>(routine, din, n, dout);
    if ((e = cudaGetLastError()) == cudaSuccess) e = cudaMemcpy(out, dout, out_bytes, cudaMemcpyDeviceToHost);
  }
  cudaFree(din);
  cudaFree(dout);
  return static_cast<int>(e);
}

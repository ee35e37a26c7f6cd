// Throughput of the FP64 instruction mix of the q-KG tile row loops (DESIGN.md K6), without their dependencies: each
// warp issues NM independent DMMA m16n8k4 (K8: m16n8k8) and NV independent DFMA per iteration, the counts of one 8-row
// block of a LINE round (6 DMMA, 132 FP64 vector instructions) or of a POINT round (12 DMMA, 88); with K = 8 products
// as one DMMA.16x8x8, 3 and 6 DMMA, and with the kKappa-unit exps (exp2k_shifted) 120 and 72 FP64 vector instructions;
// at the tile kernel's residency of 2 CTAs of 128 threads per SM (8 warps, 2 per scheduler) and at 1 CTA.  Prints one
// JSON line per mix: SM cycles per block and scheduler, from CUDA event time at the card's maximum SM clock, next to
// the work model's 2 cycles per DFMA-equivalent with a DMMA counted as 8 DFMAs per k4 step.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/fp64_mix_probe profiles/fp64_mix_probe.cu && /tmp/fp64_mix_probe
#include <cstdio>
#include <cuda_runtime.h>

template <int NM, int NV, bool K8>
__global__ void __launch_bounds__(128) mix_kernel(double* out, int iters) {
  constexpr int CH = 12;  // independent DFMA chains per thread (enough to cover the DFMA latency with one warp/scheduler)
  double c[NM][4], v[CH];
#pragma unroll
  for (int i = 0; i < NM; ++i) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0.0;
#pragma unroll
  for (int i = 0; i < CH; ++i) v[i] = threadIdx.x * 1e-9 + i * 1e-9;
  const double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9, m = 0.999999, k = 1e-12;
#pragma unroll 1
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NM; ++i) {
      if (K8) {
        asm volatile(
            "mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%4,%5}, {%6,%6}, {%0,%1,%2,%3};\n"
            : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
            : "d"(a), "d"(b), "d"(b));
      } else {
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                     : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
                     : "d"(a), "d"(b), "d"(b));
      }
#pragma unroll
      for (int jj = 0; jj < NV / NM; ++jj) {
        const int j = i * (NV / NM) + jj;
        v[j % CH] = fma(v[j % CH], m, k);
      }
    }
#pragma unroll
    for (int j = 0; j < NV % NM; ++j) v[j] = fma(v[j], m, k);
  }
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < NM; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
#pragma unroll
  for (int i = 0; i < CH; ++i) s += v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int NM, int NV, bool K8 = false>
static void run(const char* name, int sms, int ctas_per_sm) {
  const int grid = sms * ctas_per_sm, iters = 1 << 14;
  // shared memory sized so that at most ctas_per_sm CTAs fit on an SM: the grid runs as one wave of that residency
  int smem_per_sm = 0, clock_khz = 0, resident = 0;
  cudaDeviceGetAttribute(&smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, 0);
  cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, 0);
  const int smem = smem_per_sm / ctas_per_sm - 2048;
  cudaFuncSetAttribute(mix_kernel<NM, NV, K8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(mix_kernel<NM, NV, K8>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, mix_kernel<NM, NV, K8>, 128, smem);
  double* out;
  cudaMalloc(&out, sizeof(double) * grid * 128);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  mix_kernel<NM, NV, K8><<<grid, 128, smem>>>(out, iters);  // warm-up
  cudaEventRecord(e0);
  mix_kernel<NM, NV, K8><<<grid, 128, smem>>>(out, iters);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  // every warp-iteration (one block of the mix), spread over the 4 schedulers of each SM
  const double cycles = ms * 1e-3 * clock_khz * 1e3 * sms * 4 / (static_cast<double>(grid) * 4 * iters);
  printf("{\"mix\": \"%s\", \"dmma\": %d, \"dmma_k\": %d, \"fp64_vector\": %d, \"ctas_per_sm\": %d, \"resident\": %d, "
         "\"cycles_per_block_per_scheduler\": %.2f, \"clock_mhz\": %d, \"model_cycles_8dfma_per_dmma\": %.1f, "
         "\"error\": \"%s\"}\n",
         name, NM, K8 ? 8 : 4, NV, ctas_per_sm, resident, cycles, clock_khz / 1000, 2.0 * (NV + (K8 ? 16 : 8) * NM),
         cudaGetErrorString(cudaGetLastError()));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(out);
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int r = 2; r >= 1; --r) {
    run<6, 132>("LINE block", sms, r);
    run<12, 88>("POINT block", sms, r);
    run<6, 0>("6 DMMA alone", sms, r);
    run<1, 132>("1 DMMA + 132 FP64 vector", sms, r);
    run<3, 132, true>("LINE block k8, exp_tab2k", sms, r);
    run<3, 120, true>("LINE block k8, exp2k_shifted", sms, r);
    run<6, 88, true>("POINT block k8, exp_tab2k", sms, r);
    run<6, 72, true>("POINT block k8, exp2k_shifted", sms, r);
  }
  return 0;
}

// Microbenchmark: register-resident fp64 peaks on sm_90a.
//   (1) DMMA  : mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 chains
//   (2) DFMA  : fma.rn.f64 chains
// Prints JSON lines (a measured DMMA ceiling for the block-GEMM kernel's roofline).
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { \
  printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

template <int NACC>
__global__ void __launch_bounds__(256) dmma_kernel(double* out, int iters, double a0, double b0) {
  double acc[NACC][2];
#pragma unroll
  for (int i = 0; i < NACC; ++i) { acc[i][0] = 0.0; acc[i][1] = 0.0; }
  double a = a0 + threadIdx.x * 1e-9, b = b0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) {
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                   : "+d"(acc[i][0]), "+d"(acc[i][1]) : "d"(a), "d"(b));
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NACC; ++i) s += acc[i][0] + acc[i][1];
  if (s == 123.456) out[0] = s;
}

template <int NACC>
__global__ void __launch_bounds__(256) dfma_kernel(double* out, int iters, double a0, double b0) {
  double acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = i;
  double a = a0 + threadIdx.x * 1e-9, b = b0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = fma(a, acc[i], b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NACC; ++i) s += acc[i];
  if (s == 123.456) out[0] = s;
}

template <typename F>
static float time_ms(F f, int reps) {
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  f(); f(); CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    CK(cudaEventRecord(e0)); f(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
  }
  return best;
}

int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  int sms = p.multiProcessorCount;
  double* out; CK(cudaMalloc(&out, 8));
  printf("{\"device\": \"%s\", \"sms\": %d, \"clock_khz\": %d}\n", p.name, sms, p.clockRate);
  const int iters = 4096;
  for (int bps = 1; bps <= 4; bps *= 2) {
    {
      constexpr int NACC = 16;
      int grid = sms * bps;
      float ms = time_ms([&] { dmma_kernel<NACC><<<grid, 256>>>(out, iters, 1.0, 1e-9); }, 5);
      double flops = 2.0 * 256 /*fma per warp mma*/ * NACC * (double)iters * (256 / 32) * grid;
      printf("{\"bench\": \"dmma_m8n8k4\", \"blocks_per_sm\": %d, \"warps_per_sm\": %d, \"ms\": %.4f, \"tflops\": %.3f}\n",
             bps, bps * 8, ms, flops / ms * 1e-9);
    }
    {
      constexpr int NACC = 16;
      int grid = sms * bps;
      float ms = time_ms([&] { dfma_kernel<NACC><<<grid, 256>>>(out, iters, 1.0, 1e-9); }, 5);
      double flops = 2.0 * NACC * (double)iters * 256 * grid;
      printf("{\"bench\": \"dfma\", \"blocks_per_sm\": %d, \"warps_per_sm\": %d, \"ms\": %.4f, \"tflops\": %.3f}\n",
             bps, bps * 8, ms, flops / ms * 1e-9);
    }
  }
  // sustained: ~2 s of DMMA back to back
  {
    constexpr int NACC = 16; int grid = sms * 2;
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    int n = 0;
    for (; n < 400; ++n) dmma_kernel<NACC><<<grid, 256>>>(out, iters, 1.0, 1e-9);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    double flops = 2.0 * 256 * NACC * (double)iters * 8 * grid * n;
    printf("{\"bench\": \"dmma_sustained\", \"ms\": %.2f, \"tflops\": %.3f}\n", ms, flops / ms * 1e-9);
    CK(cudaEventRecord(e0));
    for (n = 0; n < 400; ++n) dfma_kernel<NACC><<<grid, 256>>>(out, iters, 1.0, 1e-9);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms, e0, e1));
    flops = 2.0 * NACC * (double)iters * 256 * grid * n;
    printf("{\"bench\": \"dfma_sustained\", \"ms\": %.2f, \"tflops\": %.3f}\n", ms, flops / ms * 1e-9);
  }
  return 0;
}

// Microbenchmark: the s8 tensor-core ceiling on sm_90a that the Ozaki-II int8 GEMM (ozaki2_gemm_2sm_kernel) is measured against.
//   One persistent CTA per SM, two warpgroups, each issuing wgmma.mma_async m64n256k32.s32.s8.s8 on operands resident in shared
//   memory (SWIZZLE_128B K-major tiles, the GEMM's layout and issue pattern: 4 wgmmas per 128-byte K stage, one stage in flight),
//   no global-memory traffic.  Prints JSON lines: TOPS for a short run and for ~2 s back to back, with the card's name, power
//   limit, SM clock and power draw read by nvidia-smi while the sustained run is on the device.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 tools/igmma_peak.cu -o tools/igmma_peak
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { \
  printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

constexpr int A_BYTES = 2 * 64 * 128, B_BYTES = 256 * 128, SMEM = 1024 + A_BYTES + B_BYTES;

__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  return static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
#define OPS16(a, o) "+r"(a[o]), "+r"(a[o + 1]), "+r"(a[o + 2]), "+r"(a[o + 3]), "+r"(a[o + 4]), "+r"(a[o + 5]), "+r"(a[o + 6]), \
  "+r"(a[o + 7]), "+r"(a[o + 8]), "+r"(a[o + 9]), "+r"(a[o + 10]), "+r"(a[o + 11]), "+r"(a[o + 12]), "+r"(a[o + 13]),          \
  "+r"(a[o + 14]), "+r"(a[o + 15])
__device__ __forceinline__ void wgmma_s8(int32_t (&d)[128], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 "
               "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, "
               "%25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
               "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, "
               "%71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, "
               "%94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, "
               "%114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n\t}"
               : OPS16(d, 0), OPS16(d, 16), OPS16(d, 32), OPS16(d, 48), OPS16(d, 64), OPS16(d, 80), OPS16(d, 96), OPS16(d, 112)
               : "l"(da), "l"(db), "r"(acc));
}

// stages = K stages of 128 bytes per warpgroup; the accumulator restarts every 128 stages (a work item of the K = 16384 GEMM)
__global__ void __launch_bounds__(256, 1) igmma_kernel(int stages, int* out) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* smem = smem_dyn + ((1024u - (static_cast<uint32_t>(__cvta_generic_to_shared(smem_dyn)) & 1023u)) & 1023u);
  for (int i = threadIdx.x; i < (A_BYTES + B_BYTES) / 4; i += blockDim.x)
    reinterpret_cast<uint32_t*>(smem)[i] = 0x01ff02feu * (i + 1);
  __syncthreads();
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the generic-proxy fill, visible to wgmma
  const int wg = threadIdx.x >> 7;
  const uint32_t a0 = static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + wg * (64 * 128);
  const uint32_t b0 = static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + A_BYTES;
  int32_t acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0;
  int32_t sum = 0;
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
  for (int j = 0; j < stages; ++j) {
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_s8(acc, desc_sw128(a0 + 32 * k), desc_sw128(b0 + 32 * k), ((j & 127) | k) != 0);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    if (j > 0) asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
  for (int i = 0; i < 128; ++i) sum += acc[i];
  if (sum == 0x7fffffff) out[0] = sum;
}

static void smi(char* buf, size_t n) {
  buf[0] = 0;
  FILE* f = popen("nvidia-smi -i 0 --query-gpu=name,power.limit,clocks.sm,clocks.max.sm,power.draw --format=csv,noheader 2>/dev/null", "r");
  if (!f) return;
  if (!fgets(buf, static_cast<int>(n), f)) buf[0] = 0;
  pclose(f);
  buf[strcspn(buf, "\n")] = 0;
}

int main() {
  cudaDeviceProp p;
  CK(cudaGetDeviceProperties(&p, 0));
  const int sms = p.multiProcessorCount;
  int* out;
  CK(cudaMalloc(&out, 4));
  CK(cudaFuncSetAttribute(igmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  const int stages = 128 * 64;
  const double ops_per_launch = 2.0 * 64 * 256 * 128 * 2 /*warpgroups*/ * static_cast<double>(stages) * sms;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  auto launch = [&] { igmma_kernel<<<sms, 256, SMEM>>>(stages, out); };
  launch();
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < 5; ++r) {
    CK(cudaEventRecord(e0));
    launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms < best) best = ms;
  }
  printf("{\"bench\": \"igmma_m64n256k32_s8\", \"device\": \"%s\", \"sms\": %d, \"ms\": %.4f, \"tops\": %.1f}\n", p.name, sms, best,
         ops_per_launch / best * 1e-9);
  // sustained: back-to-back launches for ~2 s; the card is sampled half-way through
  int n = static_cast<int>(2000.0f / best) + 1;
  CK(cudaEventRecord(e0));
  for (int i = 0; i < n; ++i) launch();
  CK(cudaEventRecord(e1));
  char info[256];
  for (int i = 0; i < 10 && cudaEventQuery(e1) == cudaErrorNotReady; ++i) {  // ~1 s in
    struct timespec ts = {0, 100000000};
    nanosleep(&ts, nullptr);
  }
  smi(info, sizeof info);
  CK(cudaEventSynchronize(e1));
  float ms;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  printf("{\"bench\": \"igmma_m64n256k32_s8_sustained\", \"launches\": %d, \"ms\": %.1f, \"tops\": %.1f, "
         "\"nvidia_smi_during_run\": \"%s\", \"fields\": \"name, power.limit, clocks.sm, clocks.max.sm, power.draw\"}\n",
         n, ms, ops_per_launch * n / ms * 1e-9, info);
  return 0;
}

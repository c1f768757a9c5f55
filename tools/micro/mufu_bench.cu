// Micro-benchmark: MUFU.EX2 throughput per SM (and with interleaved FFMA), to size the softmax loop of attention_tc.cu.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/micro/mufu_bench tools/micro/mufu_bench.cu
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int MODE>
__global__ void k(float* out, int iters) {
  float a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = -0.001f * (threadIdx.x + i);
  float f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = 1.0f + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (MODE != 1) a[i] = ex2(a[i]) - 1.0f;          // MUFU (+1 FADD)
      if (MODE >= 1) {
#pragma unroll
        for (int r = 0; r < (MODE == 2 ? 4 : 8); ++r) f[i] = fmaf(f[i], 0.999f, 0.001f);
      }
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += a[i] + f[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int MODE>
void run(const char* name, int warps_per_sm) {
  int dev = 0, sms = 0, khz = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, dev);
  const int threads = warps_per_sm * 32, iters = 20000;
  float* out;
  cudaMalloc(&out, sizeof(float) * sms * threads);
  k<MODE><<<sms, threads>>>(out, 100);
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a);
  k<MODE><<<sms, threads>>>(out, iters);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  const double mufu = (MODE != 1) ? (double)sms * threads * iters * 8 : 0;
  const double ffma = (MODE >= 1) ? (double)sms * threads * iters * 8 * (MODE == 2 ? 4 : 8) : 0;
  printf("%-28s warps/SM %2d  %8.3f ms  MUFU %.2f /ns/SM  FFMA %.2f /ns/SM  (nominal clock %.2f GHz)\n", name, warps_per_sm, ms,
         mufu / (ms * 1e6) / sms, ffma / (ms * 1e6) / sms, khz / 1e6);
  cudaFree(out);
}

int main() {
  for (int w : {4, 8, 16, 32}) run<0>("ex2 only", w);
  for (int w : {8, 32}) run<1>("ffma only", w);
  for (int w : {8, 32}) run<2>("ex2 + 4 ffma", w);
  return 0;
}

// Microbenchmark: throughput of legacy mma.sync.m16n8k8 (tf32) on sm_90a, per SM and whole chip.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 mma_sync_rate.cu -o mma_sync_rate
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(float* out, int iters) {
  float c[4][4] = {};
  unsigned a[4] = {0x3f800000u + threadIdx.x, 0x3f900000u, 0x3fa00000u, 0x3fb00000u};
  unsigned b[2] = {0x3f800000u, 0x3f810000u + threadIdx.x};
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                   : "+f"(c[j][0]), "+f"(c[j][1]), "+f"(c[j][2]), "+f"(c[j][3])
                   : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  }
  float s = 0;
  for (int j = 0; j < 4; ++j) for (int t = 0; t < 4; ++t) s += c[j][t];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  const int sms = prop.multiProcessorCount;
  int khz = 0;
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  const double hz = khz * 1e3;   // maximum SM clock: the per-clock figures assume the card holds it
  float* d; cudaMalloc(&d, (size_t)sms * 2 * 16 * 32 * 4);
  for (int warps = 4; warps <= 16; warps *= 2) {
    int iters = 20000;
    k<<<sms * 2, warps * 32>>>(d, 10); cudaDeviceSynchronize();
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0); k<<<sms * 2, warps * 32>>>(d, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double mmas = (double)sms * 2 * warps * iters * 4;
    double flops = mmas * 16 * 8 * 8 * 2;
    const double per_clk = mmas / (ms * 1e-3) / sms / hz;
    printf("warps/CTA=%2d (2 CTAs/SM): %.3f ms, %.1f TFLOP/s tf32, %.2f MMA/clk/SM @%.2f GHz, cycles per MMA per SMSP = %.1f\n",
           warps, ms, flops / ms / 1e9, per_clk, hz / 1e9, 4.0 / per_clk);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}

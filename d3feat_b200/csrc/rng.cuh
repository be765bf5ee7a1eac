// Counter-based random draws shared by RANSAC (registration.cu) and the training-pair sampler and augmentation
// (correspond.cu): every draw is splitmix64 of its own counter, so a result does not depend on how the work is spread
// over the GPU.
#pragma once
#include "common.cuh"

namespace d3f {

constexpr unsigned long long kGolden = 0x9E3779B97F4A7C15ull;

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// an index in [0, n) from a draw z: ((z >> 32) * n) >> 32
__device__ __forceinline__ int draw_index(unsigned long long z, int n) {
  return (int)(((z >> 32) * (unsigned long long)(unsigned)n) >> 32);
}

// RANSAC: index m of hypothesis h of pair p, counter ((p << 32) | h) * 8 + m
__device__ __forceinline__ int sample_index(int p, int h, int m, int n_c, unsigned long long seed) {
  const unsigned long long c = ((((unsigned long long)(unsigned)p) << 32) | (unsigned)h) * 8ull + (unsigned)m;
  const unsigned long long z = splitmix64(seed + c * kGolden);
  return draw_index(z, n_c);
}

}  // namespace d3f

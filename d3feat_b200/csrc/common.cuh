// Shared helpers for the d3feat_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/d3feat_b200.h"

namespace d3f {

// ---- error plumbing (thread-local, no global mutable state shared between host threads) -------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
void count_launch(int n = 1);

#define D3F_CUDA(call)                                         \
  do {                                                         \
    cudaError_t e__ = (call);                                  \
    if (e__ != cudaSuccess) return d3f::cuda_fail(e__, #call); \
  } while (0)

#define D3F_LAUNCH_CHECK(name)                                   \
  do {                                                           \
    d3f::count_launch();                                         \
    cudaError_t e__ = cudaGetLastError();                        \
    if (e__ != cudaSuccess) return d3f::cuda_fail(e__, name);    \
  } while (0)

#define D3F_REQUIRE(cond, code, ...) \
  do {                               \
    if (!(cond)) {                   \
      d3f::set_error(__VA_ARGS__);   \
      return (code);                 \
    }                                \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM
constexpr int kMaxBatch = 1024;

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
__host__ __device__ static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Bump allocator over a workspace: every buffer starts at a multiple of 256 bytes, and `off` ends at the bytes the
// takes need. Each workspace has one layout function that runs the same takes to size it (null base: every pointer
// is null) and to carve it.
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* p) : base((char*)p) {}
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 256);
    T* r = base != nullptr ? (T*)(base + off) : nullptr;
    off += n * sizeof(T);
    return r;
  }
};

// ---- device helpers -------------------------------------------------------------------------------
// order-preserving float <-> uint map (for atomicMin/atomicMax on floats)
__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// order-preserving key of a canonicalised value: numpy's order for argsort / argmax. Every NaN (either sign) is one
// positive quiet NaN above +inf; -0.0 equals +0.0, so the index decides. The key is never 0.
__device__ __forceinline__ unsigned score_ord(float s) {
  unsigned u = __float_as_uint(s);
  if ((u & 0x7fffffffu) > 0x7f800000u) u = 0x7fc00000u;   // any NaN, either sign -> +qNaN (above +inf)
  else if (u == 0x80000000u) u = 0u;                      // -0.0 -> +0.0 (numpy: equal, row order decides)
  return f2ord(__uint_as_float(u));
}

// Row count of a launch: kernels are launched on a capacity-sized grid and read the actual number of rows from device
// memory when the caller supplies it (the pyramid's level sizes are produced on the device; reading them back on the
// host would put a synchronisation into every step). n_dev == nullptr: the capacity IS the row count.
__device__ __forceinline__ int dyn_rows(int n_cap, const int* __restrict__ n_dev) {
  if (n_dev == nullptr) return n_cap;
  const int n = __ldg(n_dev);
  return n < n_cap ? (n < 0 ? 0 : n) : n_cap;
}

// Rows of a stacked batch that belong to a cloud: the row count cut at start[B]. Rows at or past start[B] (lengths
// summing to less than the row count) belong to no cloud; lengths summing to more cut the last cloud at the row count.
__device__ __forceinline__ int cloud_rows(int n_cap, const int* __restrict__ n_dev, const int* __restrict__ start,
                                          int B) {
  const int n = dyn_rows(n_cap, n_dev);
  const int e = start[B];
  return e < n ? (e < 0 ? 0 : e) : n;
}

// batch element of a stacked row index: largest b with start[b] <= i (start = exclusive scan of lengths)
__device__ __forceinline__ int batch_of(const int* __restrict__ start, int B, int i) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (start[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

}  // namespace d3f

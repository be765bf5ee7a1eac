// The kernel-point optimiser of kernels/kernel_points.py:102-174 (kernel_point_optimization_debug; contract:
// include/d3feat_b200.h, restated in oracle/kernel_points_np.py): T independent tries of K points repel each other
// and are drawn to the origin, under one stopping test over all tries.
//
// The stopping test couples every try at every iteration, so one CTA runs the whole loop: positions [T*K*3] and the
// previous norms [T*K] live in shared memory (T*K <= 6400: 200 KB), and an iteration is gradients, one block-wide max,
// the per-try maxima and the move, with barriers between them and no host synchronisation. Each thread owns points
// pt = tid, tid + blockDim, ...; the gradients of its points go to the output buffer, which holds the final points
// only after the loop. Every fp64 operation is one correctly rounded intrinsic (no contraction into FMA), in the
// oracle's order, so the result is bitwise the oracle's; there are no atomics.
#include <math.h>

#include "ops.cuh"

namespace d3f {

constexpr int kKpMaxIter = 10000;       // :104
constexpr int kKpMaxPoints = 6400;      // T * K: 100 tries of 64 points
constexpr int kKpThreads = 1024;
constexpr double kKpThresh = 1e-5;      // :67
constexpr double kKpClip = 0.05;        // :70
constexpr double kKpMovingFactor = 1e-2;
constexpr double kKpMovingDecay = 0.9995;

static size_t kp_smem_bytes(int n) { return (size_t)n * 4 * sizeof(double) + 32 * sizeof(unsigned long long); }

// NaN-propagating max (np.max): once m is NaN it stays NaN.
__device__ __forceinline__ double nan_max(double m, double v) { return (v != v || v > m) ? v : m; }

__global__ void __launch_bounds__(kKpThreads, 1)
kernel_point_optimize_kernel(const double* __restrict__ initial, int T, int K, int first_moving, int fixed,
                             double* __restrict__ points, double* __restrict__ saved, int* __restrict__ iterations) {
  extern __shared__ __align__(16) unsigned char kp_smem[];
  const int N = T * K;
  double* pos = (double*)kp_smem;                         // [N][3]
  double* old = pos + 3 * N;                              // [N] previous norms (:103, :140)
  unsigned long long* red = (unsigned long long*)(old + N);   // [32] per-warp maxima
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;

  for (int e = tid; e < 3 * N; e += blockDim.x) pos[e] = initial[e];
  for (int e = tid; e < N; e += blockDim.x) old[e] = 0.0;
  __syncthreads();

  int iters = 0;
  double mf = kKpMovingFactor;
  if (K > first_moving) {
    iters = kKpMaxIter;
    for (int it = 0; it < kKpMaxIter; ++it) {
      // gradients and norms (:109-129); the stop test's |old - new| over the moving points (:134-139)
      unsigned long long dmax = 0;                        // max of non-negative doubles as their bit patterns
      for (int pt = tid; pt < N; pt += blockDim.x) {
        const int j = pt % K;
        const double* P = pos + 3 * (pt - j);
        const double xj = pos[3 * pt], yj = pos[3 * pt + 1], zj = pos[3 * pt + 2];
        double sx = 0.0, sy = 0.0, sz = 0.0;
        for (int i = 0; i < K; ++i) {
          const double dx = __dsub_rn(P[3 * i], xj), dy = __dsub_rn(P[3 * i + 1], yj), dz = __dsub_rn(P[3 * i + 2], zj);
          const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
          const double den = __dadd_rn(__dmul_rn(d2, __dsqrt_rn(d2)), 1e-6);
          const double qx = __ddiv_rn(dx, den), qy = __ddiv_rn(dy, den), qz = __ddiv_rn(dz, den);
          if (i == 0) {
            sx = qx, sy = qy, sz = qz;
          } else {
            sx = __dadd_rn(sx, qx), sy = __dadd_rn(sy, qy), sz = __dadd_rn(sz, qz);
          }
        }
        double gx = __dadd_rn(sx, __dmul_rn(10.0, xj)), gy = __dadd_rn(sy, __dmul_rn(10.0, yj));
        const double gz = __dadd_rn(sz, __dmul_rn(10.0, zj));
        if (fixed == D3F_FIXED_VERTICALS && (j == 1 || j == 2)) gx = 0.0, gy = 0.0;   // :122-123
        const double nrm = __dsqrt_rn(
            __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)), __dmul_rn(gz, gz)), 1e-12));
        if (j >= first_moving) {
          const unsigned long long b = (unsigned long long)__double_as_longlong(fabs(__dsub_rn(old[pt], nrm)));
          dmax = b > dmax ? b : dmax;
        }
        old[pt] = nrm;                                    // only this thread reads or writes old[pt] until the barrier
        points[3 * pt] = gx, points[3 * pt + 1] = gy, points[3 * pt + 2] = gz;
      }
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long b = __shfl_xor_sync(0xffffffffu, dmax, o);
        dmax = b > dmax ? b : dmax;
      }
      if (lane == 0) red[warp] = dmax;
      __syncthreads();
      dmax = 0;
      for (int w = 0; w < nwarps; ++w) dmax = red[w] > dmax ? red[w] : dmax;
      // saved_gradient_norms[it] = max over each try's points (:130)
      for (int t = tid; t < T; t += blockDim.x) {         // T may exceed the CTA (up to 6400 tries of 1 point)
        double m = old[t * K];
        for (int k = 1; k < K; ++k) m = nan_max(m, old[t * K + k]);
        saved[(size_t)it * T + t] = m;
      }
      if (__longlong_as_double((long long)dmax) < kKpThresh) {   // every thread takes the same branch
        iters = it + 1;
        break;
      }
      // move (:146-155): moving = min(mf * norm, clip), 0 for the fixed point 0; p -= (moving * g) / (norm + 1e-6)
      for (int pt = tid; pt < N; pt += blockDim.x) {
        const double nrm = old[pt];
        double mv = __dmul_rn(mf, nrm);
        mv = mv > kKpClip ? kKpClip : mv;                 // np.minimum: a NaN stays NaN
        if (fixed != D3F_FIXED_NONE && pt % K == 0) mv = 0.0;
        const double den = __dadd_rn(nrm, 1e-6);
        for (int c = 0; c < 3; ++c)
          pos[3 * pt + c] = __dsub_rn(pos[3 * pt + c], __ddiv_rn(__dmul_rn(mv, points[3 * pt + c]), den));
      }
      mf = __dmul_rn(mf, kKpMovingDecay);                 // :174
      __syncthreads();                                    // positions, old and red are read again next iteration
    }
  }
  for (int e = tid; e < 3 * N; e += blockDim.x) points[e] = pos[e];
  if (tid == 0) *iterations = iters;
}

}  // namespace d3f

using namespace d3f;

extern "C" int d3f_kernel_point_optimize(const double* initial, int T, int K, int dimension, int fixed, double* points,
                                         double* saved_gradient_norms, int* iterations, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(dimension == 3, D3F_ERR_INVALID, "kernel_point_optimize: dimension=%d (only 3 is supported)", dimension);
  D3F_REQUIRE(fixed == D3F_FIXED_NONE || fixed == D3F_FIXED_CENTER || fixed == D3F_FIXED_VERTICALS, D3F_ERR_INVALID,
              "kernel_point_optimize: unknown fixed=%d", fixed);
  D3F_REQUIRE(T >= 1 && K >= 1 && (long long)T * K <= kKpMaxPoints, D3F_ERR_INVALID,
              "kernel_point_optimize: T=%d tries of K=%d points (need T, K >= 1 and T*K <= %d)", T, K, kKpMaxPoints);
  D3F_REQUIRE(initial && points && saved_gradient_norms && iterations, D3F_ERR_INVALID,
              "kernel_point_optimize: null pointer");
  const int first_moving = fixed == D3F_FIXED_CENTER ? 1 : fixed == D3F_FIXED_VERTICALS ? 3 : 0;
  const size_t smem = kp_smem_bytes(T * K);
  D3F_CUDA(cudaFuncSetAttribute(kernel_point_optimize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)kp_smem_bytes(kKpMaxPoints)));
  D3F_CUDA(cudaMemsetAsync(saved_gradient_norms, 0, (size_t)kKpMaxIter * T * sizeof(double), stream));
  kernel_point_optimize_kernel<<<1, kKpThreads, smem, stream>>>(initial, T, K, first_moving, fixed, points,
                                                                saved_gradient_norms, iterations);
  D3F_LAUNCH_CHECK("kernel_point_optimize_kernel");
  return D3F_OK;
}

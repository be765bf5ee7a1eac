// Training-mode pieces of the D3Feat graph (models/network_blocks.py, models/D3Feat.py with training = True):
//
//   batch norm, training mode   tf.layers.batch_normalization(training=True, epsilon=1e-6) on [N, C] (unfused TF):
//                               mean = sum x / N, var = sum (x - mean)^2 / N (tf.nn.moments), y = x*scale + shift
//                               (+ residual, LeakyReLU), moving -= (moving - batch) * (1 - momentum); backward
//                               dbeta = sum dz, dgamma = sum dz*xhat, dx = gamma*invstd*(dz - dbeta/N - xhat*dgamma/N)
//   ind_max_pool backward       reduce_max(gather(x || colmin(x), inds)): ties split evenly over the H entries, the
//                               shadow's shares routed through reduce_min to the rows equal to the column minimum
//   gather backward             closest_pool / tf.gather: dx[s] = sum of dout[q] over inds[q] == s, ascending q
//   l2_normalize backward       y = x * rsqrt(max(sum x^2, eps))
//   detection_scores backward   the adjoint of pool.cu's detection_scores
//
// Every gradient that scatters rows (several outputs reading one input row) is a gather over the reverse table of the
// indices (reverse_csr, kpconv_grad.cu): each input row sums its own list in a fixed order. Every sum across all rows
// of a level is made of partials over fixed 2048-row blocks, added in float64 in block order. No float atomics (only
// integer counts and the exact ordered-uint minimum / maximum), so every result is bitwise identical run to run and
// across streams. Shapes are exact (no device row counts).
#include "ops.cuh"
#include "sort.cuh"

namespace d3f {

constexpr int kRowBlock = 2048;   // rows per partial of a cross-row sum
constexpr float kFltMax = 3.402823466e38f;

static int grid_1d(long long n) {
  const long long b = (n + 255) / 256;
  return (int)max(1ll, min(b, (long long)kNumSMs * 16));
}

static int row_blocks(long long n) { return n > 0 ? (int)((n + kRowBlock - 1) / kRowBlock) : 1; }

// ---- reverse table, carved from a workspace --------------------------------------------------------------------
struct Csr {
  SortBuffers sb;
  int *counts, *offs, *scan;
};

static Csr take_csr(Carver& cv, int E, int Ns) {
  Csr c;
  c.sb.keys[0] = cv.take<uint64_t>(E);
  c.sb.keys[1] = cv.take<uint64_t>(E);
  c.sb.vals[0] = cv.take<uint32_t>(E);
  c.sb.vals[1] = cv.take<uint32_t>(E);
  c.sb.block_hist = cv.take<int>((size_t)256 * sort_num_blocks(E));
  c.counts = cv.take<int>((size_t)Ns + 1);
  c.offs = cv.take<int>((size_t)Ns + 1);
  c.scan = cv.take<int>((size_t)scan_num_blocks(Ns + 1) + 1);
  return c;
}

// ---- batch norm, training mode ----------------------------------------------------------------------------------
enum ColSumMode { kColSum = 0, kColSqDev = 1, kColBnGrad = 2 };

// dz = d(out)/d(pre-activation) * dout: LeakyReluGrad tests the pre-activation > 0, which has the output's sign
__device__ __forceinline__ float leaky_grad(float g, float out, float alpha) {
  return alpha >= 0.f && !(out > 0.f) ? g * alpha : g;
}

// p0[blk, c] (p1[blk, c]) = float64 sum over the rows of 2048-row block blk of
//   kColSum: x    kColSqDev: (x - mean)^2    kColBnGrad: dz, dz * (x - mean) * invstd
// 32 columns x 32 row lanes per CTA: each thread sums every 32nd row of the block, the 32 partials are added in a
// fixed order
template <int MODE>
__global__ void __launch_bounds__(1024) colsum_partial_kernel(const float* __restrict__ x, const float* __restrict__ out,
                                                             const float* __restrict__ dout, int N, int C,
                                                             const float* __restrict__ mean,
                                                             const float* __restrict__ invstd, float alpha,
                                                             double* __restrict__ p0, double* __restrict__ p1) {
  __shared__ double s0[32][33], s1[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int rb = blockIdx.y * kRowBlock, re = min(N, rb + kRowBlock);
  double a0 = 0.0, a1 = 0.0;
  if (c < C) {
    const double m = mean != nullptr ? (double)mean[c] : 0.0;
    const double is = invstd != nullptr ? (double)invstd[c] : 0.0;
    for (int r = rb + ty; r < re; r += 32) {
      const size_t i = (size_t)r * C + c;
      if (MODE == kColSum) {
        a0 += (double)x[i];
      } else if (MODE == kColSqDev) {
        const double d = (double)x[i] - m;
        a0 += d * d;
      } else {
        const double dz = (double)leaky_grad(dout[i], out[i], alpha);
        a0 += dz;
        a1 += dz * (((double)x[i] - m) * is);
      }
    }
  }
  s0[ty][tx] = a0;
  s1[ty][tx] = a1;
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int k = 1; k < 32; ++k) {
      a0 += s0[k][tx];
      a1 += s1[k][tx];
    }
    p0[(size_t)blockIdx.y * C + c] = a0;
    if (MODE == kColBnGrad) p1[(size_t)blockIdx.y * C + c] = a1;
  }
}

__device__ __forceinline__ double block_order_sum(const double* __restrict__ p, int nblk, int C, int c) {
  double s = 0.0;
  for (int b = 0; b < nblk; ++b) s += p[(size_t)b * C + c];
  return s;
}

__global__ void bn_mean_kernel(const double* __restrict__ p0, int nblk, int N, int C, float* __restrict__ mean) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) mean[c] = (float)(block_order_sum(p0, nblk, C, c) / (double)N);
}

// batch variance -> invstd, the affine of the apply pass, and the moving-average update (TF assign_moving_average)
__global__ void bn_stats_kernel(const double* __restrict__ p0, int nblk, int N, int C, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ mean, float decay, float eps,
                                float* __restrict__ moving_mean, float* __restrict__ moving_var,
                                float* __restrict__ invstd, float* __restrict__ scale, float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float var = (float)(block_order_sum(p0, nblk, C, c) / (double)N);
  const float is = (float)(1.0 / sqrt((double)var + (double)eps));
  const float sc = gamma[c] * is;
  invstd[c] = is;
  scale[c] = sc;
  shift[c] = beta[c] - mean[c] * sc;
  moving_mean[c] -= (moving_mean[c] - mean[c]) * decay;
  moving_var[c] -= (moving_var[c] - var) * decay;
}

// use_batch_norm = False: y = x + offset
__global__ void offset_affine_kernel(const float* __restrict__ beta, int C, float* __restrict__ scale,
                                     float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  scale[c] = 1.f;
  shift[c] = beta[c];
}

// dbeta = sum dz, dgamma = sum dz * xhat; a = dbeta / N, b = dgamma / N for the dx pass
__global__ void bn_grad_params_kernel(const double* __restrict__ p0, const double* __restrict__ p1, int nblk, int N,
                                      int C, float* __restrict__ dbeta, float* __restrict__ dgamma,
                                      float* __restrict__ a, float* __restrict__ b) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double sb = block_order_sum(p0, nblk, C, c), sg = block_order_sum(p1, nblk, C, c);
  if (dbeta) dbeta[c] = (float)sb;
  if (dgamma) dgamma[c] = (float)sg;
  a[c] = (float)(sb / (double)N);
  b[c] = (float)(sg / (double)N);
}

__global__ void __launch_bounds__(256) bn_dx_kernel(const float* __restrict__ x, const float* __restrict__ out,
                                                    const float* __restrict__ dout, int total, int C,
                                                    const float* __restrict__ gamma, const float* __restrict__ mean,
                                                    const float* __restrict__ invstd, float alpha,
                                                    const float* __restrict__ a, const float* __restrict__ b,
                                                    float* __restrict__ dx, float* __restrict__ dres) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % C;
    const float dz = leaky_grad(dout[i], out[i], alpha);
    if (dres) dres[i] = dz;
    if (dx) {
      if (gamma) {
        const float xh = (x[i] - mean[c]) * invstd[c];
        dx[i] = gamma[c] * invstd[c] * (dz - a[c] - xh * b[c]);
      } else {
        dx[i] = dz;
      }
    }
  }
}

// Both passes carve the same layout; the forward uses p0 and the two C-vectors (scale, shift), the backward all four.
struct BatchNormWs {
  double *p0, *p1;   // [row blocks, C] column partials
  float *a, *b;      // [C]
};

static size_t batch_norm_layout(int N, int C, void* base, BatchNormWs* w_out) {
  if (N < 0 || C < 1) return 0;
  const size_t nb = (size_t)row_blocks(N) * C;
  Carver cv(base);
  BatchNormWs w;
  w.p0 = cv.take<double>(nb);
  w.p1 = cv.take<double>(nb);
  w.a = cv.take<float>(C);
  w.b = cv.take<float>(C);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_batch_norm_train_workspace_bytes(int N, int C) {
  return batch_norm_layout(N, C, nullptr, nullptr);
}

extern "C" int d3f_batch_norm_train_forward(const float* x, int N, int C, const float* gamma, const float* beta,
                                            float* moving_mean, float* moving_var, float decay, float eps,
                                            const float* residual, float alpha, float* out, float* mean, float* invstd,
                                            void* workspace, size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N >= 0 && C >= 1 && (long long)N * C < (1ll << 31), D3F_ERR_INVALID,
              "batch_norm_train_forward: bad shape N=%d C=%d", N, C);
  D3F_REQUIRE(decay >= 0.f && decay <= 1.f && eps > 0.f, D3F_ERR_INVALID,
              "batch_norm_train_forward: 1 - momentum=%g outside [0, 1] or epsilon=%g not positive", (double)decay,
              (double)eps);
  D3F_REQUIRE(beta != nullptr && (gamma == nullptr || (moving_mean && moving_var && mean && invstd)),
              D3F_ERR_INVALID, "batch_norm_train_forward: null pointer");
  BatchNormWs w;
  const size_t need = batch_norm_layout(N, C, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "batch_norm_train_forward: workspace too small");
  if (N == 0) return D3F_OK;   // no batch statistics: the moving statistics stay as they are
  D3F_REQUIRE(x && out && workspace, D3F_ERR_INVALID, "batch_norm_train_forward: null pointer");
  const int nblk = row_blocks(N);
  double* p0 = w.p0;
  float *scale = w.a, *shift = w.b;
  const int cb = ceil_div(C, 256);
  if (gamma != nullptr) {
    const dim3 grid(ceil_div(C, 32), nblk);
    colsum_partial_kernel<kColSum><<<grid, 1024, 0, stream>>>(x, nullptr, nullptr, N, C, nullptr, nullptr, -1.f, p0,
                                                             nullptr);
    D3F_LAUNCH_CHECK("colsum_partial_kernel");
    bn_mean_kernel<<<cb, 256, 0, stream>>>(p0, nblk, N, C, mean);
    D3F_LAUNCH_CHECK("bn_mean_kernel");
    colsum_partial_kernel<kColSqDev><<<grid, 1024, 0, stream>>>(x, nullptr, nullptr, N, C, mean, nullptr, -1.f, p0,
                                                               nullptr);
    D3F_LAUNCH_CHECK("colsum_partial_kernel");
    bn_stats_kernel<<<cb, 256, 0, stream>>>(p0, nblk, N, C, gamma, beta, mean, decay, eps, moving_mean, moving_var,
                                            invstd, scale, shift);
    D3F_LAUNCH_CHECK("bn_stats_kernel");
  } else {
    offset_affine_kernel<<<cb, 256, 0, stream>>>(beta, C, scale, shift);
    D3F_LAUNCH_CHECK("offset_affine_kernel");
  }
  return d3f_affine_leaky(x, N, C, scale, shift, residual, alpha, out, stream, nullptr);
}

extern "C" int d3f_batch_norm_train_backward(const float* x, const float* out, const float* dout, int N, int C,
                                             const float* gamma, const float* mean, const float* invstd, float alpha,
                                             float* dx, float* dresidual, float* dgamma, float* dbeta, void* workspace,
                                             size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N >= 0 && C >= 1 && (long long)N * C < (1ll << 31), D3F_ERR_INVALID,
              "batch_norm_train_backward: bad shape N=%d C=%d", N, C);
  D3F_REQUIRE(gamma != nullptr || dgamma == nullptr, D3F_ERR_INVALID,
              "batch_norm_train_backward: dgamma without gamma (use_batch_norm = False has no gamma)");
  BatchNormWs w;
  const size_t need = batch_norm_layout(N, C, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "batch_norm_train_backward: workspace too small");
  if (dgamma) D3F_CUDA(cudaMemsetAsync(dgamma, 0, (size_t)C * sizeof(float), stream));
  if (dbeta) D3F_CUDA(cudaMemsetAsync(dbeta, 0, (size_t)C * sizeof(float), stream));
  if (N == 0) return D3F_OK;
  D3F_REQUIRE(x && out && dout && workspace && (gamma == nullptr || (mean && invstd)), D3F_ERR_INVALID,
              "batch_norm_train_backward: null pointer");
  const int nblk = row_blocks(N);
  double *p0 = w.p0, *p1 = w.p1;
  float *a = w.a, *b = w.b;
  const dim3 grid(ceil_div(C, 32), nblk);
  colsum_partial_kernel<kColBnGrad><<<grid, 1024, 0, stream>>>(x, out, dout, N, C, mean, invstd, alpha, p0, p1);
  D3F_LAUNCH_CHECK("colsum_partial_kernel");
  bn_grad_params_kernel<<<ceil_div(C, 256), 256, 0, stream>>>(p0, p1, nblk, N, C, dbeta, dgamma, a, b);
  D3F_LAUNCH_CHECK("bn_grad_params_kernel");
  if (dx || dresidual) {
    const int total = N * C;
    bn_dx_kernel<<<grid_1d(total), 256, 0, stream>>>(x, out, dout, total, C, gamma, mean, invstd, alpha, a, b, dx,
                                                     dresidual);
    D3F_LAUNCH_CHECK("bn_dx_kernel");
  }
  return D3F_OK;
}

namespace d3f {

// ---- ind_max_pool backward ----------------------------------------------------------------------------------------
// column minimum (ordered uint, preset 0xFFFFFFFF) or, with cmin given, the number of rows equal to it
__global__ void __launch_bounds__(256) colmin_pass_kernel(const float* __restrict__ x, int N, int C,
                                                          unsigned* __restrict__ cmin_ord, int* __restrict__ nmin) {
  __shared__ unsigned red[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  unsigned m = nmin ? 0u : 0xffffffffu;
  if (c < C) {
    const float target = nmin ? ord2f(cmin_ord[c]) : 0.f;
    for (int r = blockIdx.y * 8 + ty; r < N; r += gridDim.y * 8) {
      const float v = x[(size_t)r * C + c];
      if (nmin) m += v == target ? 1u : 0u;
      else m = min(m, f2ord(v));
    }
  }
  red[ty][tx] = m;
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int k = 1; k < 8; ++k) m = nmin ? m + red[k][tx] : min(m, red[k][tx]);
    if (nmin) atomicAdd(&nmin[c], (int)m);
    else atomicMin(&cmin_ord[c], m);
  }
}

// gs[q,c] = dout[q,c] / ties, ties = #{h : v(q,h,c) == out[q,c]}, v = x[id] for a real id, the column minimum else
__global__ void __launch_bounds__(256) maxpool_share_kernel(const float* __restrict__ x, const int* __restrict__ inds,
                                                            const float* __restrict__ out,
                                                            const float* __restrict__ dout, int N1, int N2, int H,
                                                            int C, const unsigned* __restrict__ cmin_ord,
                                                            float* __restrict__ gs) {
  const int total = N2 * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int q = i / C, c = i % C;
    const float o = out[i], shadow = ord2f(cmin_ord[c]);
    int ties = 0;
    for (int h = 0; h < H; ++h) {
      const int id = inds[(size_t)q * H + h];
      const float v = (id >= 0 && id < N1) ? x[(size_t)id * C + c] : shadow;
      ties += v == o ? 1 : 0;
    }
    gs[i] = ties > 0 ? dout[i] / (float)ties : 0.f;
  }
}

// partial[blk, c] = float64 sum over the shadow entries [offs[N1] + 2048 blk, ...) of gs[q,c] where the column
// minimum is the pooled maximum
__global__ void __launch_bounds__(256) shadow_partial_kernel(const uint32_t* __restrict__ sorted_q,
                                                             const int* __restrict__ offs, int N1, int E,
                                                             const float* __restrict__ out,
                                                             const float* __restrict__ gs, int C,
                                                             const unsigned* __restrict__ cmin_ord,
                                                             double* __restrict__ partial) {
  __shared__ double red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const long long eb = (long long)offs[N1] + (long long)blockIdx.y * kRowBlock;
  const long long ee = min((long long)E, eb + kRowBlock);
  double a = 0.0;
  if (c < C) {
    const float m = ord2f(cmin_ord[c]);
    for (long long e = eb + ty; e < ee; e += 8) {
      const size_t i = (size_t)sorted_q[e] * C + c;
      if (out[i] == m) a += (double)gs[i];
    }
  }
  red[ty][tx] = a;
  __syncthreads();
  if (ty == 0 && c < C) {
    for (int k = 1; k < 8; ++k) a += red[k][tx];
    partial[(size_t)blockIdx.y * C + c] = a;
  }
}

// share[c] = (sum of the shadow's gradient) / (number of rows equal to the column minimum): reduce_min's gradient
__global__ void shadow_share_kernel(const double* __restrict__ partial, int nblk, int C, const int* __restrict__ nmin,
                                    float* __restrict__ share) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float s = (float)block_order_sum(partial, nblk, C, c);
  share[c] = nmin[c] > 0 ? s / (float)nmin[c] : 0.f;
}

// dx[s,c] = sum over the entries of s, ascending (q, h), of gs[q,c] where x[s,c] is the pooled maximum (float64, one
// rounding), + share[c] where x[s,c] is the column minimum
__global__ void __launch_bounds__(256) maxpool_gather_kernel(const float* __restrict__ x,
                                                             const uint32_t* __restrict__ sorted_q,
                                                             const int* __restrict__ counts,
                                                             const int* __restrict__ offs,
                                                             const float* __restrict__ out,
                                                             const float* __restrict__ gs,
                                                             const unsigned* __restrict__ cmin_ord,
                                                             const float* __restrict__ share, int N1, int C,
                                                             float* __restrict__ dx) {
  const int total = N1 * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int s = i / C, c = i % C;
    const float v = x[i];
    double a = 0.0;
    for (int j = offs[s], e = offs[s] + counts[s]; j < e; ++j) {
      const size_t k = (size_t)sorted_q[j] * C + c;
      if (out[k] == v) a += (double)gs[k];
    }
    float r = (float)a;
    if (v == ord2f(cmin_ord[c])) r += share[c];
    dx[i] = r;
  }
}

struct MaxPoolBwd {
  Csr csr;
  unsigned* cmin;
  int* nmin;
  float *gs, *share;
  double* partial;
};

static size_t maxpool_backward_layout(int N1, int N2, int H, int C, void* base, MaxPoolBwd* w_out) {
  if (N1 < 1 || N2 < 0 || H < 0 || C < 1 || (long long)N2 * H >= (1ll << 31)) return 0;
  Carver cv(base);
  MaxPoolBwd w;
  w.csr = take_csr(cv, N2 * H, N1);
  w.cmin = cv.take<unsigned>(C);
  w.nmin = cv.take<int>(C);
  w.gs = cv.take<float>((size_t)N2 * C);
  w.share = cv.take<float>(C);
  w.partial = cv.take<double>((size_t)row_blocks((long long)N2 * H) * C);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

}  // namespace d3f

extern "C" size_t d3f_ind_max_pool_backward_workspace_bytes(int N1, int N2, int H, int C) {
  return maxpool_backward_layout(N1, N2, H, C, nullptr, nullptr);
}

extern "C" int d3f_ind_max_pool_backward(const float* x, const int* inds, const float* out, const float* dout, int N1,
                                         int N2, int H, int C, float* dx, void* workspace, size_t workspace_bytes,
                                         d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N1 >= 1 && N2 >= 0 && H >= 0 && C >= 1, D3F_ERR_INVALID,
              "ind_max_pool_backward: bad shape N1=%d N2=%d H=%d C=%d", N1, N2, H, C);
  D3F_REQUIRE((long long)N2 * max(H, C) < (1ll << 31) && (long long)N1 * C < (1ll << 31), D3F_ERR_INVALID,
              "ind_max_pool_backward: N2*H, N2*C or N1*C beyond int32");
  D3F_REQUIRE(x && dx && (N2 == 0 || (inds && out && dout && workspace)), D3F_ERR_INVALID,
              "ind_max_pool_backward: null pointer");
  MaxPoolBwd w;
  const size_t need = maxpool_backward_layout(N1, N2, H, C, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "ind_max_pool_backward: workspace too small");
  if (N2 == 0 || H == 0) {   // nothing was pooled (H = 0: every pooled row is the column minimum of no entry)
    D3F_CUDA(cudaMemsetAsync(dx, 0, (size_t)N1 * C * sizeof(float), stream));
    return D3F_OK;
  }
  const int E = N2 * H;
  D3F_CUDA(cudaMemsetAsync(w.cmin, 0xff, (size_t)C * sizeof(unsigned), stream));
  D3F_CUDA(cudaMemsetAsync(w.nmin, 0, (size_t)C * sizeof(int), stream));
  const dim3 cgrid(ceil_div(C, 32), min(ceil_div(N1, 64), 4 * kNumSMs));
  colmin_pass_kernel<<<cgrid, 256, 0, stream>>>(x, N1, C, w.cmin, nullptr);
  D3F_LAUNCH_CHECK("colmin_pass_kernel");
  colmin_pass_kernel<<<cgrid, 256, 0, stream>>>(x, N1, C, w.cmin, w.nmin);
  D3F_LAUNCH_CHECK("colmin_pass_kernel");
  maxpool_share_kernel<<<grid_1d((long long)N2 * C), 256, 0, stream>>>(x, inds, out, dout, N1, N2, H, C, w.cmin, w.gs);
  D3F_LAUNCH_CHECK("maxpool_share_kernel");
  const uint32_t* sorted_q = nullptr;
  int rc = reverse_csr(inds, N2, N1, H, nullptr, nullptr, w.csr.sb, w.csr.counts, w.csr.offs, w.csr.scan, &sorted_q,
                       stream);
  if (rc) return rc;
  const int nblk = row_blocks(E);
  shadow_partial_kernel<<<dim3(ceil_div(C, 32), nblk), 256, 0, stream>>>(sorted_q, w.csr.offs, N1, E, out, w.gs, C,
                                                                         w.cmin, w.partial);
  D3F_LAUNCH_CHECK("shadow_partial_kernel");
  shadow_share_kernel<<<ceil_div(C, 256), 256, 0, stream>>>(w.partial, nblk, C, w.nmin, w.share);
  D3F_LAUNCH_CHECK("shadow_share_kernel");
  maxpool_gather_kernel<<<grid_1d((long long)N1 * C), 256, 0, stream>>>(x, sorted_q, w.csr.counts, w.csr.offs, out,
                                                                        w.gs, w.cmin, w.share, N1, C, dx);
  D3F_LAUNCH_CHECK("maxpool_gather_kernel");
  return D3F_OK;
}

namespace d3f {

// ---- gather backward (closest_pool, tf.gather) --------------------------------------------------------------------
// dx[s,c] = sum of dout[q,c] over the q with inds[q] == s, ascending q, float64, one rounding
__global__ void __launch_bounds__(256) gather_rows_grad_kernel(const float* __restrict__ dout,
                                                               const uint32_t* __restrict__ sorted_q,
                                                               const int* __restrict__ counts,
                                                               const int* __restrict__ offs, int N1, int C,
                                                               float* __restrict__ dx) {
  const int total = N1 * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int s = i / C, c = i % C;
    double a = 0.0;
    for (int j = offs[s], e = offs[s] + counts[s]; j < e; ++j) a += (double)dout[(size_t)sorted_q[j] * C + c];
    dx[i] = (float)a;
  }
}

static size_t gather_rows_backward_layout(int N1, int N2, void* base, Csr* w_out) {
  if (N1 < 0 || N2 < 0) return 0;
  Carver cv(base);
  const Csr w = take_csr(cv, N2, N1);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

}  // namespace d3f

extern "C" size_t d3f_gather_rows_backward_workspace_bytes(int N1, int N2) {
  return gather_rows_backward_layout(N1, N2, nullptr, nullptr);
}

extern "C" int d3f_gather_rows_backward(const int* inds, const float* dout, int N1, int N2, int C, float* dx,
                                        void* workspace, size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N1 >= 0 && N2 >= 0 && C >= 1 && (long long)max(N1, N2) * C < (1ll << 31), D3F_ERR_INVALID,
              "gather_rows_backward: bad shape N1=%d N2=%d C=%d", N1, N2, C);
  D3F_REQUIRE(N1 == 0 || dx, D3F_ERR_INVALID, "gather_rows_backward: null pointer");
  D3F_REQUIRE(N1 == 0 || N2 == 0 || (inds && dout && workspace), D3F_ERR_INVALID,
              "gather_rows_backward: null pointer");
  Csr csr;
  const size_t need = gather_rows_backward_layout(N1, N2, workspace, &csr);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "gather_rows_backward: workspace too small");
  if (N1 == 0) return D3F_OK;
  if (N2 == 0) {
    D3F_CUDA(cudaMemsetAsync(dx, 0, (size_t)N1 * C * sizeof(float), stream));
    return D3F_OK;
  }
  const uint32_t* sorted_q = nullptr;
  int rc = reverse_csr(inds, N2, N1, 1, nullptr, nullptr, csr.sb, csr.counts, csr.offs, csr.scan, &sorted_q, stream);
  if (rc) return rc;
  gather_rows_grad_kernel<<<grid_1d((long long)N1 * C), 256, 0, stream>>>(dout, sorted_q, csr.counts, csr.offs, N1, C,
                                                                          dx);
  D3F_LAUNCH_CHECK("gather_rows_grad_kernel");
  return D3F_OK;
}

namespace d3f {

// ---- l2_normalize backward ------------------------------------------------------------------------------------------
// one warp per row; sum x^2 and the reciprocal norm exactly as the forward computes them. sum x^2 >= eps (Maximum's
// gradient goes to its first input on a tie): dx = (g - y (y.g)) * inv, else dx = g * inv
__global__ void __launch_bounds__(256) l2_normalize_grad_kernel(const float* __restrict__ x,
                                                                const float* __restrict__ dout, int N, int C,
                                                                float eps, float* __restrict__ dx) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  const float* xr = x + (size_t)warp * C;
  const float* gr = dout + (size_t)warp * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float v = xr[c];
    s = fmaf(v, v, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float m = fmaxf(s, eps);
  float inv = rsqrtf(m);
  inv = inv * (1.5f - 0.5f * m * inv * inv);
  float dot = 0.f;
  const bool through_norm = s >= eps;
  if (through_norm) {
    for (int c = lane; c < C; c += 32) dot = fmaf(xr[c] * inv, gr[c], dot);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  }
  for (int c = lane; c < C; c += 32) {
    const float g = gr[c];
    dx[(size_t)warp * C + c] = through_norm ? (g - xr[c] * inv * dot) * inv : g * inv;
  }
}

}  // namespace d3f

extern "C" int d3f_l2_normalize_backward(const float* x, const float* dout, int N, int C, float eps, float* dx,
                                         d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N >= 0 && C >= 1 && eps > 0.f, D3F_ERR_INVALID, "l2_normalize_backward: bad arguments N=%d C=%d eps=%g", N,
              C, (double)eps);
  if (N == 0) return D3F_OK;
  D3F_REQUIRE(x && dout && dx, D3F_ERR_INVALID, "l2_normalize_backward: null pointer");
  l2_normalize_grad_kernel<<<ceil_div(N * 32, 256), 256, 0, stream>>>(x, dout, N, C, eps, dx);
  D3F_LAUNCH_CHECK("l2_normalize_grad_kernel");
  return D3F_OK;
}

namespace d3f {

// ---- detection_scores backward ------------------------------------------------------------------------------------
// Forward (pool.cu), row i of cloud b, inv = 1/(M_b + 1e-6) with M_b the cloud's maximum, cnt = neighbours with a
// non-zero raw row sum (count_nonzero: no gradient):
//   f = x inv, mean = inv/cnt sum_h x[nb_h], d = f - mean, ratio = f / (1e-6 + max_c f), score = max_c softplus(d) ratio
// Rows of no cloud have inv = 0: constant score, no gradient.

// row maximum into the cloud maximum (ordered uint, exact), non-zero flag of the raw row sum: as the forward
__global__ void __launch_bounds__(256) det_rowmax_kernel(const float* __restrict__ x, int N, int D,
                                                         const int* __restrict__ start, int B,
                                                         unsigned* __restrict__ cmax, unsigned char* __restrict__ nz) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  float m = -kFltMax, s = 0.f;
  for (int c = lane; c < D; c += 32) {
    const float v = x[(size_t)warp * D + c];
    m = fmaxf(m, v);
    s += v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  if (lane == 0) {
    if (warp < start[B]) atomicMax(&cmax[batch_of(start, B, warp)], f2ord(m));
    nz[warp] = s != 0.f ? 1 : 0;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_isum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// one warp per row: the row's own terms. gx = dL/df * inv (the direct path), A = dL/dmean * inv / cnt (scattered to
// the neighbours by the gather pass), ginv = dL/dinv (summed per cloud), tm[b] += elements equal to the cloud maximum
__global__ void __launch_bounds__(256) det_row_grad_kernel(const float* __restrict__ x, const int* __restrict__ nb,
                                                           int N, int H, int D, const int* __restrict__ start, int B,
                                                           const unsigned* __restrict__ cmax,
                                                           const unsigned char* __restrict__ nz,
                                                           const float* __restrict__ gscore, float* __restrict__ mean_buf,
                                                           float* __restrict__ raw_buf, float* __restrict__ gx,
                                                           float* __restrict__ A, float* __restrict__ ginv,
                                                           int* __restrict__ tm) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  const size_t base = (size_t)warp * D;
  const bool in_cloud = warp < start[B];
  const int b = in_cloud ? batch_of(start, B, warp) : 0;
  const float M = in_cloud ? ord2f(cmax[b]) : 0.f;
  const float inv = in_cloud ? 1.f / (M + 1e-6f) : 0.f;
  const int* row = nb + (size_t)warp * H;
  int cnt = 0;
  for (int h = 0; h < H; ++h) {
    const int id = row[h];
    if (id >= 0 && id < N && nz[id]) ++cnt;
  }
  const float inv_cnt = 1.f / (float)max(cnt, 1);
  float dmax = -kFltMax;
  int ties_m = 0;
  for (int c = lane; c < D; c += 32) {
    const float v = x[base + c];
    dmax = fmaxf(dmax, v * inv);
    ties_m += (in_cloud && v == M) ? 1 : 0;
  }
  dmax = warp_max(dmax);
  ties_m = warp_isum(ties_m);
  if (lane == 0 && ties_m > 0) atomicAdd(&tm[b], ties_m);
  const float e = 1e-6f + dmax;
  float best = -kFltMax;
  for (int c = lane; c < D; c += 32) {
    const float f = x[base + c] * inv;
    float mean = 0.f, raw = 0.f;
    for (int h = 0; h < H; ++h) {
      const int id = row[h];
      if (id >= 0 && id < N) {
        const float v = x[(size_t)id * D + c];
        mean += v * inv;
        raw += v;
      }
    }
    mean *= inv_cnt;
    mean_buf[base + c] = mean;
    raw_buf[base + c] = raw;
    const float d = f - mean;
    const float softplus = d > 20.f ? d : log1pf(expf(d));
    best = fmaxf(best, softplus * (f / e));
  }
  best = warp_max(best);
  // the channel maxima: ties split evenly (reduce_max's gradient)
  int T = 0, Td = 0;
  for (int c = lane; c < D; c += 32) {
    const float f = x[base + c] * inv;
    const float d = f - mean_buf[base + c];
    const float softplus = d > 20.f ? d : log1pf(expf(d));
    T += softplus * (f / e) == best ? 1 : 0;
    Td += f == dmax ? 1 : 0;
  }
  T = warp_isum(T);
  Td = warp_isum(Td);
  const float gs = T > 0 ? gscore[warp] / (float)T : 0.f;
  float gdm = 0.f;   // dL/d dmax = -sum_c g_ratio f / e^2
  for (int c = lane; c < D; c += 32) {
    const float f = x[base + c] * inv;
    const float d = f - mean_buf[base + c];
    const float softplus = d > 20.f ? d : log1pf(expf(d));
    const float ratio = f / e;
    if (softplus * ratio == best) gdm -= gs * softplus * ratio / e;
  }
  gdm = warp_sum(gdm);
  const float gdm_share = Td > 0 ? gdm / (float)Td : 0.f;
  float gi = 0.f;
  for (int c = lane; c < D; c += 32) {
    const float xv = x[base + c];
    const float f = xv * inv;
    const float mean = mean_buf[base + c];
    const float d = f - mean;
    const float softplus = d > 20.f ? d : log1pf(expf(d));
    const float ratio = f / e;
    const float gp = softplus * ratio == best ? gs : 0.f;
    const float g_d = gp * ratio / (1.f + expf(-d));                  // softplus' = sigmoid
    const float g_f = gp * softplus / e + (f == dmax ? gdm_share : 0.f) + g_d;
    gx[base + c] = g_f * inv;
    A[base + c] = -g_d * inv * inv_cnt;
    gi += g_f * xv - g_d * raw_buf[base + c] * inv_cnt;
  }
  gi = warp_sum(gi);
  if (lane == 0) ginv[warp] = in_cloud ? gi : 0.f;
}

// one CTA per cloud: dL/dM_b = -inv^2 sum over the cloud's rows of ginv (fixed 2048-row chunks from the cloud's start,
// float64), split evenly over the cloud's elements equal to M_b (reduce_max's gradient)
__global__ void __launch_bounds__(256) det_cloud_grad_kernel(const float* __restrict__ ginv,
                                                             const int* __restrict__ start, int N,
                                                             const unsigned* __restrict__ cmax,
                                                             const int* __restrict__ tm, float* __restrict__ share) {
  __shared__ double red[256];
  const int b = blockIdx.x;
  const int a = min(start[b], N), e = min(start[b + 1], N);
  double tot = 0.0;
  for (int r0 = a; r0 < e; r0 += kRowBlock) {
    double s = 0.0;
    for (int r = r0 + threadIdx.x; r < min(e, r0 + kRowBlock); r += 256) s += (double)ginv[r];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
      __syncthreads();
    }
    tot += red[0];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double inv = (double)(1.f / (ord2f(cmax[b]) + 1e-6f));
    share[b] = tm[b] > 0 ? (float)(-tot * inv * inv / (double)tm[b]) : 0.f;
  }
}

// dx[r,c] = gx[r,c] + sum over the reverse entries of r, ascending (q, h), of A[q,c] (float64) + the cloud-max share
__global__ void __launch_bounds__(256) det_gather_kernel(const float* __restrict__ x, const float* __restrict__ gx,
                                                         const float* __restrict__ A,
                                                         const uint32_t* __restrict__ sorted_q,
                                                         const int* __restrict__ counts, const int* __restrict__ offs,
                                                         const int* __restrict__ start, int B,
                                                         const unsigned* __restrict__ cmax,
                                                         const float* __restrict__ share, int N, int D,
                                                         float* __restrict__ dx) {
  const int total = N * D;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int r = i / D, c = i % D;
    double a = (double)gx[i];
    for (int j = offs[r], e = offs[r] + counts[r]; j < e; ++j) a += (double)A[(size_t)sorted_q[j] * D + c];
    float v = (float)a;
    if (r < start[B]) {
      const int b = batch_of(start, B, r);
      if (x[i] == ord2f(cmax[b])) v += share[b];
    }
    dx[i] = v;
  }
}

struct DetBwd {
  Csr csr;
  int *start, *tm;
  unsigned* cmax;
  float *share, *mean, *raw, *gx, *A, *ginv;
  unsigned char* nz;
};

static size_t detection_backward_layout(int N, int H, int B, int D, void* base, DetBwd* w_out) {
  if (N < 0 || H < 0 || B < 1 || D < 1 || (long long)N * H >= (1ll << 31)) return 0;
  Carver cv(base);
  DetBwd w;
  w.csr = take_csr(cv, N * H, N);
  w.start = cv.take<int>((size_t)B + 1);
  w.tm = cv.take<int>(B);
  w.cmax = cv.take<unsigned>(B);
  w.share = cv.take<float>(B);
  const size_t ND = (size_t)N * D;
  w.mean = cv.take<float>(ND);
  w.raw = cv.take<float>(ND);
  w.gx = cv.take<float>(ND);
  w.A = cv.take<float>(ND);
  w.ginv = cv.take<float>(N);
  w.nz = cv.take<unsigned char>((size_t)N + 1);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

}  // namespace d3f

extern "C" size_t d3f_detection_scores_backward_workspace_bytes(int N, int H, int B, int D) {
  return detection_backward_layout(N, H, B, D, nullptr, nullptr);
}

extern "C" int d3f_detection_scores_backward(const float* feats, const int* neighbors, const int* lengths,
                                             const float* dscores, int B, int N, int H, int D, float* dfeats,
                                             void* workspace, size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch && N >= 0 && H >= 0 && D >= 1, D3F_ERR_INVALID,
              "detection_scores_backward: bad shape B=%d N=%d H=%d D=%d", B, N, H, D);
  D3F_REQUIRE((long long)N * max(H, D) < (1ll << 31), D3F_ERR_INVALID,
              "detection_scores_backward: N*H or N*D beyond int32");
  DetBwd w;
  const size_t need = detection_backward_layout(N, H, B, D, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "detection_scores_backward: workspace too small");
  if (N == 0) return D3F_OK;
  D3F_REQUIRE(feats && (neighbors || H == 0) && lengths && dscores && dfeats && workspace, D3F_ERR_INVALID,
              "detection_scores_backward: null pointer");
  int rc = launch_batch_start(lengths, B, w.start, stream);
  if (rc) return rc;
  D3F_CUDA(cudaMemsetAsync(w.cmax, 0, sizeof(unsigned) * B, stream));
  D3F_CUDA(cudaMemsetAsync(w.tm, 0, sizeof(int) * B, stream));
  const int wblocks = ceil_div(N * 32, 256);
  det_rowmax_kernel<<<wblocks, 256, 0, stream>>>(feats, N, D, w.start, B, w.cmax, w.nz);
  D3F_LAUNCH_CHECK("det_rowmax_kernel");
  det_row_grad_kernel<<<wblocks, 256, 0, stream>>>(feats, neighbors, N, H, D, w.start, B, w.cmax, w.nz, dscores,
                                                   w.mean, w.raw, w.gx, w.A, w.ginv, w.tm);
  D3F_LAUNCH_CHECK("det_row_grad_kernel");
  det_cloud_grad_kernel<<<B, 256, 0, stream>>>(w.ginv, w.start, N, w.cmax, w.tm, w.share);
  D3F_LAUNCH_CHECK("det_cloud_grad_kernel");
  const uint32_t* sorted_q = nullptr;
  if (H > 0) {
    rc = reverse_csr(neighbors, N, N, H, nullptr, nullptr, w.csr.sb, w.csr.counts, w.csr.offs, w.csr.scan, &sorted_q,
                     stream);
    if (rc) return rc;
  } else {
    D3F_CUDA(cudaMemsetAsync(w.csr.counts, 0, (size_t)(N + 1) * sizeof(int), stream));
    D3F_CUDA(cudaMemsetAsync(w.csr.offs, 0, (size_t)(N + 1) * sizeof(int), stream));
    sorted_q = w.csr.sb.vals[0];
  }
  det_gather_kernel<<<grid_1d((long long)N * D), 256, 0, stream>>>(feats, w.gx, w.A, sorted_q, w.csr.counts,
                                                                   w.csr.offs, w.start, B, w.cmax, w.share, N, D,
                                                                   dfeats);
  D3F_LAUNCH_CHECK("det_gather_kernel");
  return D3F_OK;
}

// Indexed pooling kernels of the encoder / decoder:
//   ind_max_pool  models/network_blocks.py:51-66   shadow row = column-wise minimum of x
//   closest_pool  models/network_blocks.py:69-83   shadow row = zeros, first index column only
//   l2_normalize  models/D3Feat.py:65              x * rsqrt(max(sum x^2, eps))
#include "ops.cuh"

namespace d3f {

// The shadow row of ind_max_pool is the column-wise minimum of x. A pooled row that has at least one real neighbour
// never needs it (the minimum cannot exceed a real value), and the pyramid guarantees one (a cell's barycenter lies
// within the pooling radius of one of the cell's points). So the pooling kernel runs first and raises a flag
// (colmin_ord[C] = 0) for rows WITHOUT a real neighbour; the full-matrix reduction and the fix-up pass below exit
// immediately while the flag is down, and produce the reference's result exactly when it is up.
//
// column-wise minimum via ordered-uint atomics; colmin_ord pre-set to 0xFFFFFFFF
__global__ void __launch_bounds__(256) colmin_kernel(const float* __restrict__ x, int Ncap, const int* __restrict__ n_dev,
                                                     int C, unsigned* __restrict__ colmin_ord) {
  const int N = dyn_rows(Ncap, n_dev);
  __shared__ unsigned red[8][32];
  if (colmin_ord[C] != 0u) return;   // no row asked for the shadow value
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  unsigned m = 0xffffffffu;
  if (c < C)
    for (int r = blockIdx.y * 8 + ty; r < N; r += gridDim.y * 8) m = min(m, f2ord(x[(size_t)r * C + c]));
  red[ty][tx] = m;
  __syncthreads();
  if (ty == 0 && c < C) {
#pragma unroll
    for (int k = 1; k < 8; ++k) m = min(m, red[k][tx]);
    atomicMin(&colmin_ord[c], m);
  }
}

// one warp per (pooled row, 128-channel slab): lanes own 4 consecutive channels (float4 when C % 4 == 0). Splitting the
// channels over warps matters at the deep levels (1204 rows x 1024 channels: one warp per row walked 8 slabs x 40
// dependent row loads; now 8 warps walk 40 each)
template <int VEC>
__global__ void __launch_bounds__(256)
ind_max_pool_kernel(const float* __restrict__ x, const int* __restrict__ inds, int N1cap, int N2cap,
                    const int* __restrict__ n1_dev, const int* __restrict__ n2_dev, int H, int C, int slabs,
                    unsigned* __restrict__ colmin_ord, float* __restrict__ out) {
  const int N1 = dyn_rows(N1cap, n1_dev), N2 = dyn_rows(N2cap, n2_dev);
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int warp = gw / slabs, slab = gw - warp * slabs;
  if (warp >= N2) return;
  const int* row = inds + (size_t)warp * H;
  const int c0 = slab * 32 * VEC + lane * VEC;
  if (c0 >= C) return;
  float best[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) best[v] = -3.402823466e38f;
  bool any_real = false;
  for (int h = 0; h < H; ++h) {
    int id = row[h];
    if (id < 0 || id >= N1) continue;
    any_real = true;
    const float* p = x + (size_t)id * C + c0;
    if (VEC == 4) {
      float4 t = *reinterpret_cast<const float4*>(p);
      best[0] = fmaxf(best[0], t.x); best[1 % VEC] = fmaxf(best[1 % VEC], t.y);
      best[2 % VEC] = fmaxf(best[2 % VEC], t.z); best[3 % VEC] = fmaxf(best[3 % VEC], t.w);
    } else {
      best[0] = fmaxf(best[0], *p);
    }
  }
  if (!any_real) {   // every neighbour is the shadow: the row is the column minimum, filled in by the fix-up pass
    if (lane == 0 && slab == 0) colmin_ord[C] = 0u;
    return;
  }
  if (VEC == 4) {
    *reinterpret_cast<float4*>(out + (size_t)warp * C + c0) =
        make_float4(best[0], best[1 % VEC], best[2 % VEC], best[3 % VEC]);
  } else {
    out[(size_t)warp * C + c0] = best[0];
  }
}

// rows without any real neighbour := column minimum (only runs its body when the pooling kernel raised the flag)
__global__ void __launch_bounds__(256)
ind_max_pool_fix_kernel(const int* __restrict__ inds, int N1cap, int N2cap, const int* __restrict__ n1_dev,
                        const int* __restrict__ n2_dev, int H, int C, const unsigned* __restrict__ colmin_ord,
                        float* __restrict__ out) {
  if (colmin_ord[C] != 0u) return;
  const int N1 = dyn_rows(N1cap, n1_dev), N2 = dyn_rows(N2cap, n2_dev);
  const int lane = threadIdx.x & 31;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < N2; r += (gridDim.x * blockDim.x) >> 5) {
    bool real = false;
    for (int h = lane; h < H; h += 32) {
      int id = inds[(size_t)r * H + h];
      real = real || (id >= 0 && id < N1);
    }
    if (__any_sync(0xffffffffu, real)) continue;
    for (int c = lane; c < C; c += 32) out[(size_t)r * C + c] = ord2f(colmin_ord[c]);
  }
}

// [C] ordered column minima + [1] flag (0xFFFFFFFF = not needed)
static size_t ind_max_pool_layout(int C, void* base, unsigned** colmin) {
  Carver cv(base);
  unsigned* c = cv.take<unsigned>((size_t)(C > 0 ? C : 1) + 1);
  if (colmin != nullptr) *colmin = c;
  return cv.off;
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_ind_max_pool_workspace_bytes(int C) { return ind_max_pool_layout(C, nullptr, nullptr); }

extern "C" int d3f_ind_max_pool(const float* x, const int* inds, int N1, int N2, int H, int C, float* out,
                                void* workspace, size_t workspace_bytes, d3f_stream_t stream_, const int* n1_dev,
                                const int* n2_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N2 == 0 || (x && inds && out && workspace), D3F_ERR_INVALID, "d3f_ind_max_pool: null pointer");
  D3F_REQUIRE(N1 >= 1 && N2 >= 0 && H >= 0 && C >= 1, D3F_ERR_INVALID, "ind_max_pool: bad shape N1=%d N2=%d H=%d C=%d",
              N1, N2, H, C);
  unsigned* colmin;
  const size_t need = ind_max_pool_layout(C, workspace, &colmin);
  D3F_REQUIRE(workspace_bytes >= need, D3F_ERR_WORKSPACE, "ind_max_pool: workspace too small");
  if (N2 == 0) return D3F_OK;
  D3F_CUDA(cudaMemsetAsync(colmin, 0xff, need, stream));
  int blocks = ceil_div(N2 * 32, 256);
  bool v4 = (C % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  const int slabs = ceil_div(C, v4 ? 128 : 32);
  const long long pool_blocks = ((long long)N2 * slabs * 32 + 255) / 256;
  D3F_REQUIRE(pool_blocks < (1ll << 31), D3F_ERR_CAPACITY, "ind_max_pool: %d rows x %d channels exceed the launch grid", N2, C);
  if (v4) ind_max_pool_kernel<4><<<(unsigned)pool_blocks, 256, 0, stream>>>(x, inds, N1, N2, n1_dev, n2_dev, H, C, slabs, colmin, out);
  else ind_max_pool_kernel<1><<<(unsigned)pool_blocks, 256, 0, stream>>>(x, inds, N1, N2, n1_dev, n2_dev, H, C, slabs, colmin, out);
  D3F_LAUNCH_CHECK("ind_max_pool_kernel");
  dim3 grid(ceil_div(C, 32), min(ceil_div(N1, 64), 4 * kNumSMs));
  colmin_kernel<<<grid, 256, 0, stream>>>(x, N1, n1_dev, C, colmin);
  D3F_LAUNCH_CHECK("colmin_kernel");
  ind_max_pool_fix_kernel<<<min(blocks, 4 * kNumSMs), 256, 0, stream>>>(inds, N1, N2, n1_dev, n2_dev, H, C, colmin, out);
  D3F_LAUNCH_CHECK("ind_max_pool_fix_kernel");
  return D3F_OK;
}

namespace d3f {

__global__ void __launch_bounds__(256)
closest_pool_kernel(const float* __restrict__ x, const int* __restrict__ inds, int N1cap, int N2cap,
                    const int* __restrict__ n1_dev, const int* __restrict__ n2_dev, int ld, int C,
                    float* __restrict__ out) {
  const int N1 = dyn_rows(N1cap, n1_dev), N2 = dyn_rows(N2cap, n2_dev);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N2) return;
  int id = inds[(size_t)warp * ld];
  bool shadow = id < 0 || id >= N1;
  for (int c = lane; c < C; c += 32) out[(size_t)warp * C + c] = shadow ? 0.f : x[(size_t)id * C + c];
}

}  // namespace d3f

extern "C" int d3f_closest_pool(const float* x, const int* inds, int N1, int N2, int ld_inds, int C, float* out,
                                d3f_stream_t stream_, const int* n1_dev, const int* n2_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N2 == 0 || (x && inds && out), D3F_ERR_INVALID, "d3f_closest_pool: null pointer");
  D3F_REQUIRE(N1 >= 0 && N2 >= 0 && ld_inds >= 1 && C >= 1, D3F_ERR_INVALID, "closest_pool: bad shape");
  if (N2 == 0) return D3F_OK;
  closest_pool_kernel<<<ceil_div(N2 * 32, 256), 256, 0, stream>>>(x, inds, N1, N2, n1_dev, n2_dev, ld_inds, C, out);
  D3F_LAUNCH_CHECK("closest_pool_kernel");
  return D3F_OK;
}

namespace d3f {

__global__ void __launch_bounds__(256) l2_normalize_kernel(const float* __restrict__ x, int Ncap,
                                                           const int* __restrict__ n_dev, int C, float eps,
                                                           float* __restrict__ out) {
  const int N = dyn_rows(Ncap, n_dev);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) {
    float v = x[(size_t)warp * C + c];
    s = fmaf(v, v, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  float inv = rsqrtf(fmaxf(s, eps));
  // one Newton step: rsqrtf is 2 ulp, the reference divides by an IEEE sqrt
  float m = fmaxf(s, eps);
  inv = inv * (1.5f - 0.5f * m * inv * inv);
  for (int c = lane; c < C; c += 32) out[(size_t)warp * C + c] = x[(size_t)warp * C + c] * inv;
}

}  // namespace d3f

extern "C" int d3f_l2_normalize(const float* x, int N, int C, float eps, float* out, d3f_stream_t stream_,
                                const int* n_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N == 0 || (x && out), D3F_ERR_INVALID, "d3f_l2_normalize: null pointer");
  D3F_REQUIRE(N >= 0 && C >= 1, D3F_ERR_INVALID, "l2_normalize: bad shape");
  if (N == 0) return D3F_OK;
  l2_normalize_kernel<<<ceil_div(N * 32, 256), 256, 0, stream>>>(x, N, n_dev, C, eps, out);
  D3F_LAUNCH_CHECK("l2_normalize_kernel");
  return D3F_OK;
}

namespace d3f {

// ---------------------------------------------------------------------------------------------------
// Detection score of D3Feat (models/D3Feat.py:67-115), generalised from the reference's hard-coded pair of clouds to
// B stacked clouds: per-cloud max normalisation, density-invariant saliency softplus(x - mean of the neighbours whose
// feature-row sum is non-zero), channel-max ratio, max over channels. Rows at or past start[B] (lengths summing to less
// than the row count) belong to no cloud: they take no part in any cloud's maximum, and their own score is unspecified.
__global__ void __launch_bounds__(256)
cloud_max_kernel(const float* __restrict__ x, int Ncap, const int* __restrict__ n_dev, int D,
                 const int* __restrict__ start, int B, unsigned* __restrict__ cloud_max_ord,
                 unsigned char* __restrict__ nonzero) {
  const int N = dyn_rows(Ncap, n_dev);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  float m = -3.402823466e38f, s = 0.f;
  for (int c = lane; c < D; c += 32) {
    float v = x[(size_t)warp * D + c];
    m = fmaxf(m, v);
    s += v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  if (lane == 0) {
    if (warp < start[B]) atomicMax(&cloud_max_ord[batch_of(start, B, warp)], f2ord(m));
    nonzero[warp] = s != 0.f ? 1 : 0;   // tf.count_nonzero of the neighbour's channel sum (:91-92)
  }
}

__global__ void __launch_bounds__(256)
detection_score_kernel(const float* __restrict__ x, const int* __restrict__ nb, int Ncap,
                       const int* __restrict__ n_dev, int H, int D, const int* __restrict__ start, int B,
                       const unsigned* __restrict__ cloud_max_ord, const unsigned char* __restrict__ nonzero,
                       float* __restrict__ score) {
  const int N = dyn_rows(Ncap, n_dev);
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= N) return;
  // all neighbours of a point lie in its own cloud, so one scale serves the point and its neighbourhood; a row of no
  // cloud gets scale 0
  const float inv = warp < start[B] ? 1.f / (ord2f(cloud_max_ord[batch_of(start, B, warp)]) + 1e-6f) : 0.f;
  const int* row = nb + (size_t)warp * H;
  int cnt = 0;
  for (int h = 0; h < H; ++h) {
    int id = row[h];
    if (id >= 0 && id < N && nonzero[id]) ++cnt;
  }
  const float inv_cnt = 1.f / (float)max(cnt, 1);
  float dmax = -3.402823466e38f;
  for (int c = lane; c < D; c += 32) dmax = fmaxf(dmax, x[(size_t)warp * D + c] * inv);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dmax = fmaxf(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
  float best = -3.402823466e38f;
  for (int c = lane; c < D; c += 32) {
    const float f = x[(size_t)warp * D + c] * inv;
    float mean = 0.f;
    for (int h = 0; h < H; ++h) {
      int id = row[h];
      if (id >= 0 && id < N) mean += x[(size_t)id * D + c] * inv;   // the shadow row is zero
    }
    mean *= inv_cnt;
    const float d = f - mean;
    const float softplus = d > 20.f ? d : log1pf(expf(d));
    best = fmaxf(best, softplus * (f / (1e-6f + dmax)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) score[warp] = best;
}

struct DetectionWs {
  int* start;
  unsigned* cmax;
  unsigned char* nonzero;
};

static size_t detection_layout(int N, int B, void* base, DetectionWs* w_out) {
  Carver cv(base);
  DetectionWs w;
  w.start = cv.take<int>((size_t)B + 1);
  w.cmax = cv.take<unsigned>(B);
  w.nonzero = cv.take<unsigned char>((size_t)N + 1);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

}  // namespace d3f

extern "C" size_t d3f_detection_scores_workspace_bytes(int N, int B) { return detection_layout(N, B, nullptr, nullptr); }

extern "C" int d3f_detection_scores(const float* feats, const int* neighbors, const int* lengths, int B, int N, int H,
                                    int D, float* out_scores, void* workspace, size_t workspace_bytes,
                                    d3f_stream_t stream_, const int* n_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N == 0 || (feats && (neighbors || H == 0) && lengths && out_scores && workspace), D3F_ERR_INVALID,
              "d3f_detection_scores: null pointer");
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch && N >= 0 && H >= 0 && D >= 1, D3F_ERR_INVALID, "detection_scores: bad shape");
  DetectionWs w;
  const size_t need = detection_layout(N, B, workspace, &w);
  D3F_REQUIRE(workspace_bytes >= need, D3F_ERR_WORKSPACE, "detection_scores: workspace too small");
  if (N == 0) return D3F_OK;
  int* start = w.start;
  unsigned* cmax = w.cmax;
  unsigned char* nonzero = w.nonzero;
  int rc = launch_batch_start(lengths, B, start, stream);
  if (rc) return rc;
  D3F_CUDA(cudaMemsetAsync(cmax, 0, sizeof(unsigned) * B, stream));
  cloud_max_kernel<<<ceil_div(N * 32, 256), 256, 0, stream>>>(feats, N, n_dev, D, start, B, cmax, nonzero);
  D3F_LAUNCH_CHECK("cloud_max_kernel");
  detection_score_kernel<<<ceil_div(N * 32, 256), 256, 0, stream>>>(feats, neighbors, N, n_dev, H, D, start, B, cmax, nonzero, out_scores);
  D3F_LAUNCH_CHECK("detection_score_kernel");
  return D3F_OK;
}

namespace d3f {

__global__ void __launch_bounds__(256)
affine_leaky_kernel(const float* __restrict__ x, long long total_cap, const int* __restrict__ n_dev, int C,
                    const float* __restrict__ scale, const float* __restrict__ shift,
                    const float* __restrict__ residual, float alpha, float* __restrict__ out) {
  const long long total = n_dev ? min(total_cap, (long long)max(__ldg(n_dev), 0) * C) : total_cap;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    float y = x[i];
    if (scale) y = fmaf(y, scale[c], shift[c]);
    if (residual) y += residual[i];
    if (alpha >= 0.f) y = y > 0.f ? y : y * alpha;
    out[i] = y;
  }
}

}  // namespace d3f

extern "C" int d3f_affine_leaky(const float* x, int N, int C, const float* scale, const float* shift,
                                const float* residual, float alpha, float* out, d3f_stream_t stream_,
                                const int* n_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(N == 0 || (x && out), D3F_ERR_INVALID, "d3f_affine_leaky: null pointer");
  D3F_REQUIRE(N >= 0 && C >= 1 && (scale == nullptr) == (shift == nullptr), D3F_ERR_INVALID, "affine_leaky: bad arguments");
  long long total = (long long)N * C;
  if (total == 0) return D3F_OK;
  int blocks = (int)min((total + 255) / 256, (long long)kNumSMs * 16);
  affine_leaky_kernel<<<blocks, 256, 0, stream>>>(x, total, n_dev, C, scale, shift, residual, alpha, out);
  D3F_LAUNCH_CHECK("affine_leaky_kernel");
  return D3F_OK;
}

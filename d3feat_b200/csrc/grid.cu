// Grid subsampling (voxel barycenters) as a sort-based hash grid, bit-exact with the reference:
//   tf_custom_ops/tf_subsampling/grid_subsampling/grid_subsampling.cpp:5-97, 101-149
//   cpp_wrappers/cpp_subsampling/grid_subsampling/grid_subsampling.cpp:5-105
//
// Pipeline (all on the caller's stream, no host round trip):
//   batch starts -> per-cloud bbox (ordered-uint atomics) -> reference cell key per point
//   -> stable radix sort of (cloud, key | point index) -> segment heads -> exclusive scan
//   -> one thread per cell sums its points IN INPUT ORDER (fp32, like SampledData::update_points)
//      and multiplies by (float)(1.0/count).
#include "ops.cuh"
#include "sort.cuh"

namespace d3f {

// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) batch_start_kernel(const int* __restrict__ len, int B,
                                                           int* __restrict__ start) {
  // B <= 1024: warp-shuffle scan in one CTA; start[B] = total
  __shared__ int ws[32];
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int v = threadIdx.x < B ? len[threadIdx.x] : 0;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) ws[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = ws[lane], winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    ws[lane] = winc - w;
  }
  __syncthreads();
  int excl = ws[warp] + inc - v;
  if (threadIdx.x < B) start[threadIdx.x] = excl;
  if (threadIdx.x == B - 1) start[B] = excl + v;
  if (B == 0 && threadIdx.x == 0) start[0] = 0;
}

int launch_batch_start(const int* len, int B, int* start, cudaStream_t stream) {
  batch_start_kernel<<<1, 1024, 0, stream>>>(len, B, start);
  D3F_LAUNCH_CHECK("batch_start_kernel");
  return 0;
}

// bbox_ord[b*6 + {0,1,2}] = min (ordered uint), [3,4,5] = max. Must be pre-set to 0xFF.. / 0.
// With `start`, only the rows that belong to a cloud are visited, and their number goes to *n_rows (the row count of
// every later kernel of the subsampling).
__global__ void __launch_bounds__(256) bbox_batch_kernel(const float* __restrict__ pts, int Ncap,
                                                         const int* __restrict__ n_dev,
                                                         const int* __restrict__ start, int B,
                                                         unsigned* __restrict__ bbox_ord, int* __restrict__ n_rows) {
  const int N = start != nullptr ? cloud_rows(Ncap, n_dev, start, B) : dyn_rows(Ncap, n_dev);
  if (n_rows != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *n_rows = N;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ceil_div(N, 32) * 32; i += gridDim.x * blockDim.x) {
    bool valid = i < N;
    int b = valid ? batch_of(start, B, i) : -1;
    float x = 0.f, y = 0.f, z = 0.f;
    if (valid) { x = pts[3 * (size_t)i]; y = pts[3 * (size_t)i + 1]; z = pts[3 * (size_t)i + 2]; }
    unsigned mn[3] = {valid ? f2ord(x) : 0xffffffffu, valid ? f2ord(y) : 0xffffffffu, valid ? f2ord(z) : 0xffffffffu};
    unsigned mx[3] = {valid ? f2ord(x) : 0u, valid ? f2ord(y) : 0u, valid ? f2ord(z) : 0u};
    int b0 = __shfl_sync(0xffffffffu, b, 0);
    bool uniform = __all_sync(0xffffffffu, b == b0 || !valid) && b0 >= 0;
    if (uniform) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
          mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
      }
      if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          atomicMin(&bbox_ord[b0 * 6 + a], mn[a]);
          atomicMax(&bbox_ord[b0 * 6 + 3 + a], mx[a]);
        }
      }
    } else if (valid) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        atomicMin(&bbox_ord[b * 6 + a], mn[a]);
        atomicMax(&bbox_ord[b * 6 + 3 + a], mx[a]);
      }
    }
  }
}

__global__ void bbox_decode_kernel(const unsigned* __restrict__ ord, float* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ord2f(ord[i]);
}

}  // namespace d3f

using namespace d3f;

// Whole-cloud bbox (B = 1) into 6 device floats. Uses out_bbox itself as the ordered-uint scratch.
extern "C" int d3f_bbox(const float* pts, int N, float* out_bbox, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(pts != nullptr || N == 0, D3F_ERR_INVALID, "d3f_bbox: null points");
  D3F_REQUIRE(out_bbox != nullptr && N >= 0, D3F_ERR_INVALID, "d3f_bbox: bad arguments");
  unsigned* ord = (unsigned*)out_bbox;
  D3F_CUDA(cudaMemsetAsync(ord, 0xff, 3 * sizeof(unsigned), stream));
  D3F_CUDA(cudaMemsetAsync(ord + 3, 0, 3 * sizeof(unsigned), stream));
  if (N > 0) {
    int blocks = min(ceil_div(N, 256), kNumSMs * 4);
    bbox_batch_kernel<<<blocks, 256, 0, stream>>>(pts, N, nullptr, nullptr, 1, ord, nullptr);
    D3F_LAUNCH_CHECK("bbox_batch_kernel");
  }
  bbox_decode_kernel<<<1, 32, 0, stream>>>(ord, out_bbox, 6);
  D3F_LAUNCH_CHECK("bbox_decode_kernel");
  return 0;
}

namespace d3f {

// ---------------------------------------------------------------------------------------------------
// Reference grid geometry of one cloud (grid_subsampling.cpp:25-31), from its ordered-uint bbox.
struct CloudGrid {
  float ox, oy, oz;
  long long NX, NY;
};

__device__ __forceinline__ CloudGrid cloud_grid(const unsigned* __restrict__ bbox_ord, int b, float dl) {
  CloudGrid g;
  float inv = __fdiv_rn(1.0f, dl);  // (1/sampleDl)
  float mnx = ord2f(bbox_ord[b * 6 + 0]), mny = ord2f(bbox_ord[b * 6 + 1]), mnz = ord2f(bbox_ord[b * 6 + 2]);
  float mxx = ord2f(bbox_ord[b * 6 + 3]), mxy = ord2f(bbox_ord[b * 6 + 4]);
  g.ox = __fmul_rn(floorf(__fmul_rn(mnx, inv)), dl);  // floor(minCorner * (1/dl)) * dl
  g.oy = __fmul_rn(floorf(__fmul_rn(mny, inv)), dl);
  g.oz = __fmul_rn(floorf(__fmul_rn(mnz, inv)), dl);
  g.NX = (long long)floorf(__fdiv_rn(__fsub_rn(mxx, g.ox), dl)) + 1;
  g.NY = (long long)floorf(__fdiv_rn(__fsub_rn(mxy, g.oy), dl)) + 1;
  return g;
}

// sort key = cloud << (cell_bits+1) | folded reference key. err[0] is raised if a key needs more than
// cell_bits bits (host bbox too small).
__global__ void __launch_bounds__(256)
cell_key_kernel(const float* __restrict__ pts, int Ncap, const int* __restrict__ n_dev, const int* __restrict__ start,
                int B, const unsigned* __restrict__ bbox_ord, float dl, int cell_bits, uint64_t* __restrict__ keys,
                uint32_t* __restrict__ vals, int* __restrict__ err) {
  const int N = dyn_rows(Ncap, n_dev);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int b = batch_of(start, B, i);
  CloudGrid g = cloud_grid(bbox_ord, b, dl);
  float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
  long long ix = (long long)floorf(__fdiv_rn(__fsub_rn(x, g.ox), dl));
  long long iy = (long long)floorf(__fdiv_rn(__fsub_rn(y, g.oy), dl));
  long long iz = (long long)floorf(__fdiv_rn(__fsub_rn(z, g.oz), dl));
  // reference: size_t arithmetic mod 2^64; identical to this signed value whenever it is >= 0
  long long k = ix + g.NX * iy + g.NX * g.NY * iz;
  long long lim = 1ll << cell_bits;
  if (k >= lim || k < -lim) {
    atomicExch(err, 1);
    k = k < 0 ? -lim : lim - 1;
  }
  // negative keys (origin rounded above the minimum) wrap to the top of the u64 range in the reference:
  // keep them after all non-negative keys, in ascending order
  uint64_t folded = k >= 0 ? (uint64_t)k : (uint64_t)(lim + (k + lim));
  keys[i] = ((uint64_t)b << (cell_bits + 1)) | folded;
  vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) segment_head_kernel(const uint64_t* __restrict__ keys, int Ncap,
                                                           const int* __restrict__ n_dev, int* __restrict__ flags) {
  const int N = dyn_rows(Ncap, n_dev);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

// One thread per sorted position; heads reduce their segment in input order.
__global__ void __launch_bounds__(128)
cell_reduce_kernel(const float* __restrict__ pts, const uint64_t* __restrict__ keys,
                   const uint32_t* __restrict__ vals, const int* __restrict__ flags,
                   const int* __restrict__ cell_of, int Ncap, const int* __restrict__ n_dev, int out_cap, int cell_bits,
                   const int* __restrict__ classes, int ldim, float* __restrict__ out_pts,
                   int* __restrict__ out_classes, int* __restrict__ out_batch_len, int* __restrict__ cell_first,
                   int* __restrict__ cell_count) {
  const int N = dyn_rows(Ncap, n_dev);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || !flags[i]) return;
  uint64_t key = keys[i];
  int m = cell_of[i];
  if (m >= out_cap) return;   // more cells than the caller's output capacity: reported through out_M (status kernel)
  float sx = 0.f, sy = 0.f, sz = 0.f;
  int count = 0;
  int j = i;
  while (j < N && keys[j] == key) {
    size_t p = vals[j];
    sx = __fadd_rn(sx, pts[3 * p]);
    sy = __fadd_rn(sy, pts[3 * p + 1]);
    sz = __fadd_rn(sz, pts[3 * p + 2]);
    for (int c = 0; c < ldim; ++c) {
      int l = classes[p * ldim + c];
      int cur = (count == 0) ? l : out_classes[(size_t)m * ldim + c];
      out_classes[(size_t)m * ldim + c] = l > cur ? l : cur;  // largest label present (see header)
    }
    ++count;
    ++j;
  }
  float r = (float)(1.0 / (double)count);  // (1.0 / v.second.count) narrowed by operator*(PointXYZ, float)
  out_pts[3 * (size_t)m] = __fmul_rn(sx, r);
  out_pts[3 * (size_t)m + 1] = __fmul_rn(sy, r);
  out_pts[3 * (size_t)m + 2] = __fmul_rn(sz, r);
  cell_first[m] = i;
  cell_count[m] = count;
  atomicAdd(&out_batch_len[(int)(key >> (cell_bits + 1))], 1);
}

// features: one thread per (cell, channel); fp32 sum in input order then / (float)count
__global__ void __launch_bounds__(256)
cell_feature_kernel(const float* __restrict__ feats, int fdim, const uint32_t* __restrict__ vals,
                    const int* __restrict__ cell_first, const int* __restrict__ cell_count,
                    const int* __restrict__ M_ptr, float* __restrict__ out_feats) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int M = *M_ptr;
  if (t >= (long long)M * fdim) return;
  int m = (int)(t / fdim), c = (int)(t % fdim);
  int first = cell_first[m], count = cell_count[m];
  float s = 0.f;
  for (int j = 0; j < count; ++j) s = __fadd_rn(s, feats[(size_t)vals[first + j] * fdim + c]);
  out_feats[(size_t)m * fdim + c] = __fdiv_rn(s, (float)count);
}

// a sort-key overflow (a cloud wider than the host bbox allows) is reported to the caller as out_M = -1, more cells than the
// output capacity as out_M = -2; `status` (optional) accumulates the same conditions as bits 1 / 2 for callers that
// never read out_M on the host (the graph-replayed pyramid)
__global__ void subsample_status_kernel(const int* __restrict__ err, int* __restrict__ out_M, int out_cap,
                                        int* __restrict__ status) {
  if (*err) {
    *out_M = -1;
    if (status) atomicOr(status, 1);
  } else if (*out_M > out_cap) {
    *out_M = -2;
    if (status) atomicOr(status, 2);
  }
}

// ---------------------------------------------------------------------------------------------------
static int cell_bits_from_bbox(const float* host_bbox, float dl) {
  double cells = 1.0;
  for (int a = 0; a < 3; ++a) {
    double ext = (double)host_bbox[3 + a] - (double)host_bbox[a];
    if (!(ext >= 0)) ext = 0;
    cells *= (floor(ext / (double)dl) + 3.0);
  }
  int bits = 1;
  while (bits < 62 && (double)(1ull << bits) < cells) ++bits;
  return bits;
}

struct SubsampleWs {
  SortBuffers sort;
  int* start;
  unsigned* bbox_ord;
  int* flags;
  int* cell_of;
  int* scan_scratch;
  int* cell_first;
  int* cell_count;
  int* err;
  int* n_rows;   // rows that belong to a cloud: min(row count, start[B]), written by bbox_batch_kernel
};

static size_t subsample_layout(int N, int B, void* base, SubsampleWs* w_out) {
  int n = N > 0 ? N : 1;
  Carver cv(base);
  SubsampleWs w;
  w.sort.keys[0] = cv.take<uint64_t>(n);
  w.sort.keys[1] = cv.take<uint64_t>(n);
  w.sort.vals[0] = cv.take<uint32_t>(n);
  w.sort.vals[1] = cv.take<uint32_t>(n);
  w.sort.block_hist = cv.take<int>(256 * (size_t)sort_num_blocks(n));
  w.start = cv.take<int>(B + 1);
  w.bbox_ord = cv.take<unsigned>(6 * (size_t)(B > 0 ? B : 1));
  w.flags = cv.take<int>(n);
  w.cell_of = cv.take<int>(n);
  w.scan_scratch = cv.take<int>(scan_num_blocks(n) + 1);
  w.cell_first = cv.take<int>(n);
  w.cell_count = cv.take<int>(n);
  w.err = cv.take<int>(1);
  w.n_rows = cv.take<int>(1);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

int grid_subsample(const float* pts, const int* batch_len, int B, int N, float dl, const float* feats, int fdim,
                   const int* classes, int ldim, const float* host_bbox, float* out_pts, float* out_feats,
                   int* out_classes, int* out_batch_len, int* out_M, void* workspace, size_t workspace_bytes,
                   cudaStream_t stream, const int* n_dev, int out_capacity, int* status, const int* start_pre) {
  if (out_capacity < 0) out_capacity = N;   // a subsampled cloud never has more points than its parent
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "grid_subsample: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(N >= 0 && dl > 0.f, D3F_ERR_INVALID, "grid_subsample: N=%d, dl=%g invalid", N, (double)dl);
  D3F_REQUIRE(host_bbox != nullptr, D3F_ERR_INVALID, "grid_subsample: host_bbox is required");
  D3F_REQUIRE((feats == nullptr) == (fdim == 0) && (classes == nullptr) == (ldim == 0), D3F_ERR_INVALID,
              "grid_subsample: feats/fdim or classes/ldim mismatch");
  SubsampleWs w;
  const size_t need = subsample_layout(N, B, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "grid_subsample: workspace too small");

  D3F_CUDA(cudaMemsetAsync(out_batch_len, 0, sizeof(int) * B, stream));
  D3F_CUDA(cudaMemsetAsync(out_M, 0, sizeof(int), stream));
  if (N == 0) return D3F_OK;

  int bbits = 0;
  while ((1 << bbits) < B) ++bbits;
  int cell_bits = cell_bits_from_bbox(host_bbox, dl);
  D3F_REQUIRE(cell_bits + 1 + bbits <= 62, D3F_ERR_CAPACITY,
              "grid_subsample: grid of 2^%d cells x %d clouds exceeds the 62-bit sort key", cell_bits, B);

  if (start_pre != nullptr) w.start = const_cast<int*>(start_pre);   // the caller already scanned these lengths
  else if (launch_batch_start(batch_len, B, w.start, stream)) return D3F_ERR_CUDA;
  D3F_CUDA(cudaMemsetAsync(w.err, 0, sizeof(int), stream));
  // per-cloud bbox: min slots 0xFFFFFFFF, max slots 0
  D3F_CUDA(cudaMemsetAsync(w.bbox_ord, 0, sizeof(unsigned) * 6 * B, stream));
  {
    // min slots to 0xFFFFFFFF via a strided 2D memset: rows of 6 uints, first 3 set
    D3F_CUDA(cudaMemset2DAsync(w.bbox_ord, 6 * sizeof(unsigned), 0xff, 3 * sizeof(unsigned), B, stream));
  }
  // rows at or past start[B] belong to no cloud: from here on every kernel's row count is w.n_rows
  int blocks = min(ceil_div(N, 256), kNumSMs * 8);
  bbox_batch_kernel<<<blocks, 256, 0, stream>>>(pts, N, n_dev, w.start, B, w.bbox_ord, w.n_rows);
  D3F_LAUNCH_CHECK("bbox_batch_kernel");
  cell_key_kernel<<<ceil_div(N, 256), 256, 0, stream>>>(pts, N, w.n_rows, w.start, B, w.bbox_ord, dl, cell_bits,
                                                        w.sort.keys[0], w.sort.vals[0], w.err);
  D3F_LAUNCH_CHECK("cell_key_kernel");
  int cur = radix_sort_pairs(w.sort, N, cell_bits + 1 + bbits, stream, w.n_rows);
  if (cur < 0) return cur;
  segment_head_kernel<<<ceil_div(N, 256), 256, 0, stream>>>(w.sort.keys[cur], N, w.n_rows, w.flags);
  D3F_LAUNCH_CHECK("segment_head_kernel");
  int rc = exclusive_scan_i32(w.flags, w.cell_of, N, out_M, w.scan_scratch, stream, w.n_rows);
  if (rc) return rc;
  cell_reduce_kernel<<<ceil_div(N, 128), 128, 0, stream>>>(pts, w.sort.keys[cur], w.sort.vals[cur], w.flags,
                                                           w.cell_of, N, w.n_rows, out_capacity, cell_bits, classes,
                                                           ldim, out_pts, out_classes, out_batch_len, w.cell_first,
                                                           w.cell_count);
  D3F_LAUNCH_CHECK("cell_reduce_kernel");
  if (fdim > 0) {
    long long work = (long long)N * fdim;  // upper bound on M * fdim
    cell_feature_kernel<<<(unsigned)((work + 255) / 256), 256, 0, stream>>>(feats, fdim, w.sort.vals[cur],
                                                                            w.cell_first, w.cell_count, out_M,
                                                                            out_feats);
    D3F_LAUNCH_CHECK("cell_feature_kernel");
  }
  subsample_status_kernel<<<1, 1, 0, stream>>>(w.err, out_M, out_capacity, status);
  D3F_LAUNCH_CHECK("subsample_status_kernel");
  return D3F_OK;
}

int grid_subsample_error_flag(const void* workspace, size_t workspace_bytes, int N, int B, int** flag) {
  SubsampleWs w;
  subsample_layout(N, B, const_cast<void*>(workspace), &w);
  *flag = w.err;
  return 0;
}

}  // namespace d3f

extern "C" size_t d3f_grid_subsample_workspace_bytes(int N, int B) { return subsample_layout(N, B, nullptr, nullptr); }

extern "C" int d3f_grid_subsample(const float* pts, const int* batch_len, int B, int N, float dl, const float* feats,
                                  int fdim, const int* classes, int ldim, const float* host_bbox, float* out_pts,
                                  float* out_feats, int* out_classes, int* out_batch_len, int* out_M, void* workspace,
                                  size_t workspace_bytes, d3f_stream_t stream) {
  D3F_REQUIRE((pts != nullptr || N == 0) && batch_len != nullptr && out_pts != nullptr && out_batch_len != nullptr &&
                  out_M != nullptr && workspace != nullptr,
              D3F_ERR_INVALID, "d3f_grid_subsample: null pointer");
  D3F_REQUIRE((fdim == 0 || out_feats != nullptr) && (ldim == 0 || out_classes != nullptr), D3F_ERR_INVALID,
              "d3f_grid_subsample: missing feature / class output");
  return grid_subsample(pts, batch_len, B, N, dl, feats, fdim, classes, ldim, host_bbox, out_pts, out_feats,
                        out_classes, out_batch_len, out_M, workspace, workspace_bytes, (cudaStream_t)stream);
}

// Voxel down-sampling of raw scans, Open3D 0.7's VoxelDownSample (Geometry/DownSample.cpp) as every reference entry
// point runs it before the network (datasets/ThreeDMatch.py:349, datasets/ETH.py:169, datasets/KITTI.py:314-315,
// demo_registration.py:24), bit-exact in fp64:
//   min_b = min over the cloud's finite rows - v * 0.5;  i_a = (int)floor((p_a - min_b,a) / v)  (one IEEE fp64 op each)
//   voxel point = (sum of its rows in fp64, sequentially in input order) / (double)count, rounded to fp32.
//
// Pipeline (all on the caller's stream, no host round trip):
//   batch starts -> per-cloud minimum of the finite rows (ordered-uint atomics) -> fp64 voxel index and sort key
//   (cloud, iz, iy, ix) per row -> stable radix sort of (key, row) -> voxel heads -> exclusive scan
//   -> one thread per voxel sums its rows in input order (the stable sort keeps it) and divides.
#include <math.h>

#include "ops.cuh"
#include "sort.cuh"

namespace d3f {

__device__ __forceinline__ bool finite3(float x, float y, float z) {
  return isfinite(x) && isfinite(y) && isfinite(z);
}

// bmin_ord[b*3 + a] = ordered-uint minimum of axis a over the finite rows of cloud b (pre-set to 0xFF..). Rows with a
// non-finite coordinate are in no bound. *n_rows = the rows that belong to a cloud (the row count of later kernels).
__global__ void __launch_bounds__(256) voxel_bounds_kernel(const float* __restrict__ pts, int Ncap,
                                                           const int* __restrict__ n_dev, const int* __restrict__ start,
                                                           int B, unsigned* __restrict__ bmin_ord,
                                                           int* __restrict__ n_rows) {
  const int N = cloud_rows(Ncap, n_dev, start, B);
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_rows = N;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ceil_div(N, 32) * 32; i += gridDim.x * blockDim.x) {
    float x = 0.f, y = 0.f, z = 0.f;
    if (i < N) { x = pts[3 * (size_t)i]; y = pts[3 * (size_t)i + 1]; z = pts[3 * (size_t)i + 2]; }
    const bool valid = i < N && finite3(x, y, z);
    const int b = valid ? batch_of(start, B, i) : -1;
    unsigned mn[3] = {valid ? f2ord(x) : 0xffffffffu, valid ? f2ord(y) : 0xffffffffu, valid ? f2ord(z) : 0xffffffffu};
    const int b0 = __shfl_sync(0xffffffffu, b, 0);
    if (__all_sync(0xffffffffu, b == b0 || b < 0) && b0 >= 0) {
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int a = 0; a < 3; ++a) atomicMin(&bmin_ord[b0 * 3 + a], mn[a]);
    } else if (valid) {
#pragma unroll
      for (int a = 0; a < 3; ++a) atomicMin(&bmin_ord[b * 3 + a], mn[a]);
    }
  }
}

struct VoxelBits {
  int x, y, z;   // per-axis index widths
  int cloud;     // shift of the cloud id: x + y + z
};

// One axis: floor((p - (min - v * 0.5)) / v) with each operation one IEEE fp64 operation. Returns the index, or
// `lim` when it does not fit in the axis width (the cloud is wider than host_bbox allows).
__device__ __forceinline__ unsigned long long voxel_axis(float p, unsigned min_ord, double v, unsigned long long lim) {
  const double lo = __dsub_rn((double)ord2f(min_ord), __dmul_rn(v, 0.5));
  const double f = floor(__ddiv_rn(__dsub_rn((double)p, lo), v));
  return f < (double)lim ? (unsigned long long)f : lim;   // f >= 0: p >= min > lo
}

// key = cloud << bits.cloud | iz << (x + y) | iy << x | ix; rows with a non-finite coordinate get cloud = B, after
// every cloud. err[0] is raised (and the index clamped) when an index needs more than its axis width.
__global__ void __launch_bounds__(256)
voxel_key_kernel(const float* __restrict__ pts, int Ncap, const int* __restrict__ n_rows, const int* __restrict__ start,
                 int B, const unsigned* __restrict__ bmin_ord, double v, VoxelBits bits, uint64_t* __restrict__ keys,
                 uint32_t* __restrict__ vals, int* __restrict__ err) {
  const int N = dyn_rows(Ncap, n_rows);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
  uint64_t key = (uint64_t)B << bits.cloud;
  if (finite3(x, y, z)) {
    const int b = batch_of(start, B, i);
    const unsigned long long lx = 1ull << bits.x, ly = 1ull << bits.y, lz = 1ull << bits.z;
    unsigned long long ix = voxel_axis(x, bmin_ord[b * 3 + 0], v, lx);
    unsigned long long iy = voxel_axis(y, bmin_ord[b * 3 + 1], v, ly);
    unsigned long long iz = voxel_axis(z, bmin_ord[b * 3 + 2], v, lz);
    if (ix == lx || iy == ly || iz == lz) {
      atomicExch(err, 1);
      ix = min(ix, lx - 1);
      iy = min(iy, ly - 1);
      iz = min(iz, lz - 1);
    }
    key = ((uint64_t)b << bits.cloud) | (iz << (bits.x + bits.y)) | (iy << bits.x) | ix;
  }
  keys[i] = key;
  vals[i] = (uint32_t)i;
}

// flags[i] = 1 where a voxel starts in the sorted keys (dropped rows start none)
__global__ void __launch_bounds__(256) voxel_head_kernel(const uint64_t* __restrict__ keys, int Ncap,
                                                         const int* __restrict__ n_rows, int B, int cloud_shift,
                                                         int* __restrict__ flags) {
  const int N = dyn_rows(Ncap, n_rows);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const uint64_t k = keys[i];
  flags[i] = (i == 0 || k != keys[i - 1]) && (k >> cloud_shift) < (uint64_t)B ? 1 : 0;
}

// One thread per sorted position; each voxel head sums its rows in input order in fp64 and writes voxel m < out_cap.
__global__ void __launch_bounds__(128)
voxel_reduce_kernel(const float* __restrict__ pts, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                    const int* __restrict__ flags, const int* __restrict__ voxel_of, int Ncap,
                    const int* __restrict__ n_rows, int out_cap, int cloud_shift, float* __restrict__ out_pts,
                    int* __restrict__ out_len) {
  const int N = dyn_rows(Ncap, n_rows);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || !flags[i]) return;
  const int m = voxel_of[i];
  if (m >= out_cap) return;   // more voxels than the output holds: reported by voxel_status_kernel
  const uint64_t key = keys[i];
  double sx = 0.0, sy = 0.0, sz = 0.0;
  int count = 0;
  for (int j = i; j < N && keys[j] == key; ++j, ++count) {
    const size_t p = vals[j];
    sx = __dadd_rn(sx, (double)pts[3 * p]);
    sy = __dadd_rn(sy, (double)pts[3 * p + 1]);
    sz = __dadd_rn(sz, (double)pts[3 * p + 2]);
  }
  const double c = (double)count;
  out_pts[3 * (size_t)m] = __double2float_rn(__ddiv_rn(sx, c));
  out_pts[3 * (size_t)m + 1] = __double2float_rn(__ddiv_rn(sy, c));
  out_pts[3 * (size_t)m + 2] = __double2float_rn(__ddiv_rn(sz, c));
  atomicAdd(&out_len[(int)(key >> cloud_shift)], 1);
}

// Exact form (status == nullptr): *out_M = M, or -1 for a key overflow, -2 for more voxels than out_cap.
// Static form: *out_M = min(M, out_cap); bit 0 / bit 1 of *status for the same two conditions.
__global__ void voxel_status_kernel(const int* __restrict__ err, const int* __restrict__ total, int out_cap,
                                    int* __restrict__ out_M, int* __restrict__ status) {
  const int M = *total;
  if (status != nullptr) {
    const int bits = (*err ? 1 : 0) | (M > out_cap ? 2 : 0);
    if (bits) atomicOr(status, bits);
    *out_M = M < out_cap ? M : out_cap;
  } else {
    *out_M = *err ? -1 : (M > out_cap ? -2 : M);
  }
}

// ---------------------------------------------------------------------------------------------------
// Index width of one axis: a cloud of extent e (<= the host_bbox extent) has indices <= floor(e / v + 0.5); two cells of
// margin cover the rounding of the fp64 division.
static int voxel_axis_bits(double extent, double v) {
  if (!(extent >= 0)) extent = 0;
  const double cells = floor(extent / v) + 3.0;
  int bits = 1;
  while (bits < 31 && (double)(1ull << bits) < cells) ++bits;
  return (double)(1ull << bits) < cells ? 31 : bits;   // 31: more than kMaxAxisBits, refused by the caller
}

constexpr int kMaxAxisBits = 30;

struct VoxelWs {
  SortBuffers sort;
  int* start;
  unsigned* bmin_ord;
  int* flags;
  int* voxel_of;
  int* scan_scratch;
  int* err;
  int* n_rows;
  int* total;
};

static size_t voxel_layout(int N, int B, void* base, VoxelWs* w_out) {
  if (N < 0 || B < 1 || B > kMaxBatch) return 0;
  const int n = N > 0 ? N : 1;
  Carver cv(base);
  VoxelWs w;
  w.sort.keys[0] = cv.take<uint64_t>(n);
  w.sort.keys[1] = cv.take<uint64_t>(n);
  w.sort.vals[0] = cv.take<uint32_t>(n);
  w.sort.vals[1] = cv.take<uint32_t>(n);
  w.sort.block_hist = cv.take<int>(256 * (size_t)sort_num_blocks(n));
  w.start = cv.take<int>((size_t)B + 1);
  w.bmin_ord = cv.take<unsigned>(3 * (size_t)(B > 0 ? B : 1));
  w.flags = cv.take<int>(n);
  w.voxel_of = cv.take<int>(n);
  w.scan_scratch = cv.take<int>(scan_num_blocks(n) + 1);
  w.err = cv.take<int>(1);
  w.n_rows = cv.take<int>(1);
  w.total = cv.take<int>(1);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_voxel_down_sample_workspace_bytes(int N, int B) { return voxel_layout(N, B, nullptr, nullptr); }

extern "C" int d3f_voxel_down_sample(const float* pts, const int* lengths, int B, int N, const int* n_dev,
                                     double voxel_size, const float* host_bbox, float* out_pts, int* out_lengths,
                                     int* out_M, int out_capacity, int* d_status, void* workspace,
                                     size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "voxel_down_sample: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(N >= 0, D3F_ERR_INVALID, "voxel_down_sample: N=%d", N);
  D3F_REQUIRE(isfinite(voxel_size) && voxel_size > 0.0, D3F_ERR_INVALID,
              "voxel_down_sample: voxel_size=%g must be finite and > 0", voxel_size);
  if (out_capacity < 0) out_capacity = N;   // a voxelised cloud never has more points than its rows
  D3F_REQUIRE((pts != nullptr || N == 0) && lengths != nullptr && out_lengths != nullptr && out_M != nullptr &&
                  workspace != nullptr && (out_pts != nullptr || out_capacity == 0),
              D3F_ERR_INVALID, "voxel_down_sample: null pointer");
  D3F_REQUIRE(host_bbox != nullptr, D3F_ERR_INVALID, "voxel_down_sample: host_bbox is required");
  for (int a = 0; a < 6; ++a)
    D3F_REQUIRE(isfinite(host_bbox[a]), D3F_ERR_INVALID, "voxel_down_sample: host_bbox[%d]=%g is not finite", a,
                (double)host_bbox[a]);
  VoxelWs w;
  const size_t need = voxel_layout(N, B, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "voxel_down_sample: workspace too small");
  VoxelBits bits;
  bits.x = voxel_axis_bits((double)host_bbox[3] - (double)host_bbox[0], voxel_size);
  bits.y = voxel_axis_bits((double)host_bbox[4] - (double)host_bbox[1], voxel_size);
  bits.z = voxel_axis_bits((double)host_bbox[5] - (double)host_bbox[2], voxel_size);
  bits.cloud = bits.x + bits.y + bits.z;
  int bbits = 0;
  while ((1 << bbits) < B + 1) ++bbits;   // cloud ids 0 .. B (B = dropped rows)
  D3F_REQUIRE(bits.x <= kMaxAxisBits && bits.y <= kMaxAxisBits && bits.z <= kMaxAxisBits &&
                  bits.cloud + bbits <= 62,
              D3F_ERR_CAPACITY, "voxel_down_sample: a grid of 2^%d x 2^%d x 2^%d voxels x %d clouds exceeds the sort key",
              bits.x, bits.y, bits.z, B);

  D3F_CUDA(cudaMemsetAsync(out_lengths, 0, sizeof(int) * B, stream));
  if (N == 0) {
    D3F_CUDA(cudaMemsetAsync(out_M, 0, sizeof(int), stream));
    return D3F_OK;
  }
  if (launch_batch_start(lengths, B, w.start, stream)) return D3F_ERR_CUDA;
  D3F_CUDA(cudaMemsetAsync(w.err, 0, sizeof(int), stream));
  D3F_CUDA(cudaMemsetAsync(w.bmin_ord, 0xff, sizeof(unsigned) * 3 * B, stream));
  voxel_bounds_kernel<<<min(ceil_div(N, 256), kNumSMs * 8), 256, 0, stream>>>(pts, N, n_dev, w.start, B, w.bmin_ord,
                                                                              w.n_rows);
  D3F_LAUNCH_CHECK("voxel_bounds_kernel");
  voxel_key_kernel<<<ceil_div(N, 256), 256, 0, stream>>>(pts, N, w.n_rows, w.start, B, w.bmin_ord, voxel_size, bits,
                                                         w.sort.keys[0], w.sort.vals[0], w.err);
  D3F_LAUNCH_CHECK("voxel_key_kernel");
  const int cur = radix_sort_pairs(w.sort, N, bits.cloud + bbits, stream, w.n_rows);
  if (cur < 0) return cur;
  voxel_head_kernel<<<ceil_div(N, 256), 256, 0, stream>>>(w.sort.keys[cur], N, w.n_rows, B, bits.cloud, w.flags);
  D3F_LAUNCH_CHECK("voxel_head_kernel");
  const int rc = exclusive_scan_i32(w.flags, w.voxel_of, N, w.total, w.scan_scratch, stream, w.n_rows);
  if (rc) return rc;
  voxel_reduce_kernel<<<ceil_div(N, 128), 128, 0, stream>>>(pts, w.sort.keys[cur], w.sort.vals[cur], w.flags,
                                                            w.voxel_of, N, w.n_rows, out_capacity, bits.cloud, out_pts,
                                                            out_lengths);
  D3F_LAUNCH_CHECK("voxel_reduce_kernel");
  voxel_status_kernel<<<1, 1, 0, stream>>>(w.err, w.total, out_capacity, out_M, d_status);
  D3F_LAUNCH_CHECK("voxel_status_kernel");
  return D3F_OK;
}

// Keypoint selection by detection score for B stacked clouds -- the selection the reference's testers run on the host:
//   utils/tester.py:209-213   3DMatch: every point of a fragment in ascending score order (evaluate.py keeps the last 250)
//   utils/tester.py:281-290   KITTI: the top k of each cloud, ascending
//
// One stable LSD radix sort of (cloud << 32 | ord(score), row) pairs orders every cloud at once; cloud b then occupies
// the sorted positions [start_b, start_b + len_b), the same offsets as its input rows, and its top k are the last
// min(k, len_b) of them. Canonicalising the scores first (every NaN -> one positive quiet NaN, -0.0 -> +0.0) makes
// the order that of np.argsort(kind="stable"): NaNs above +inf, ties by ascending row. All launches are sized by the
// capacity and read the row count from n_dev, so the whole selection can be captured in a CUDA graph.
//
// Random keypoints for the same layout -- the testers' `-rand` arm: np.random.choice(len, k) per cloud, with
// replacement (utils/tester.py:238-279, geometric_registration/evaluate.py:45-54) -- are counter-based draws of
// rng.cuh, one per output slot (d3f_sample_keypoints).
#include <climits>

#include "ops.cuh"
#include "rng.cuh"
#include "sort.cuh"

namespace d3f {

// keys[i] = cloud(i) << 32 | ord(score[i]), vals[i] = i. Rows past the last cloud (lengths summing to less than n) get
// cloud id B and sort behind every cloud.
__global__ void __launch_bounds__(256)
keypoint_key_kernel(const float* __restrict__ scores, int Ncap, const int* __restrict__ n_dev,
                    const int* __restrict__ start, int B, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int N = dyn_rows(Ncap, n_dev);
  const int end = start[B];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    const int b = i < end ? batch_of(start, B, i) : B;
    keys[i] = ((uint64_t)b << 32) | score_ord(scores[i]);
    vals[i] = (uint32_t)i;
  }
}

__global__ void __launch_bounds__(256)
keypoint_order_kernel(const uint32_t* __restrict__ sorted, int Ncap, const int* __restrict__ n_dev,
                      int* __restrict__ order) {
  const int N = dyn_rows(Ncap, n_dev);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) order[i] = (int)sorted[i];
}

// One warp per output slot (b, j), j < k. Cloud b's sorted range is cut at n, so no row >= n is ever read, whatever
// the lengths say. Slots j >= count_b get index -1 and zero rows.
__global__ void __launch_bounds__(256)
keypoint_gather_kernel(const uint32_t* __restrict__ sorted, int Ncap, const int* __restrict__ n_dev,
                       const int* __restrict__ start, int B, int k, const float* __restrict__ scores,
                       const float* __restrict__ points, const float* __restrict__ desc, int D,
                       int* __restrict__ out_index, int* __restrict__ out_count, float* __restrict__ out_points,
                       float* __restrict__ out_desc, float* __restrict__ out_scores) {
  const int N = dyn_rows(Ncap, n_dev);
  const int lane = threadIdx.x & 31;
  const long long slots = (long long)B * k;
  const long long stride = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < slots; w += stride) {
    const int b = (int)(w / k), j = (int)(w - (long long)b * k);
    const int s = min(max(start[b], 0), N);
    const int e = min(max(start[b + 1], s), N);
    const int cnt = min(k, e - s);
    const bool real = j < cnt;
    const int idx = real ? (int)sorted[e - cnt + j] : -1;
    if (lane == 0) {
      if (out_index) out_index[w] = idx;
      if (out_scores) out_scores[w] = real ? scores[idx] : 0.f;
      if (out_count && j == 0) out_count[b] = cnt;
    }
    if (out_points && lane < 3) out_points[w * 3 + lane] = real ? points[(size_t)idx * 3 + lane] : 0.f;
    if (out_desc)
      for (int c = lane; c < D; c += 32) out_desc[w * D + c] = real ? desc[(size_t)idx * D + c] : 0.f;
  }
}

// Uniform random keypoints, with replacement: slot j of cloud b holds row s_b + draw_index(z, n_b) with
// z = splitmix64(seed + ((b << 32) | j) * golden), so a slot's row depends only on (seed, b, j, n_b) and the first c
// slots of a k-slot draw are the c-slot draw. One warp per output slot, as keypoint_gather_kernel; the clouds are cut
// at n as there, and an empty cloud gets count 0, index -1 and zero rows.
__global__ void __launch_bounds__(256)
keypoint_sample_kernel(int Ncap, const int* __restrict__ n_dev, const int* __restrict__ start, int B, int k,
                       unsigned long long seed, const float* __restrict__ scores, const float* __restrict__ points,
                       const float* __restrict__ desc, int D, int* __restrict__ out_index, int* __restrict__ out_count,
                       float* __restrict__ out_points, float* __restrict__ out_desc, float* __restrict__ out_scores) {
  const int N = dyn_rows(Ncap, n_dev);
  const int lane = threadIdx.x & 31;
  const long long slots = (long long)B * k;
  const long long stride = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < slots; w += stride) {
    const int b = (int)(w / k), j = (int)(w - (long long)b * k);
    const int s = min(max(start[b], 0), N);
    const int e = min(max(start[b + 1], s), N);
    const bool real = e > s;
    const unsigned long long c = ((unsigned long long)(unsigned)b << 32) | (unsigned)j;
    const int idx = real ? s + draw_index(splitmix64(seed + c * kGolden), e - s) : -1;
    if (lane == 0) {
      if (out_index) out_index[w] = idx;
      if (out_scores) out_scores[w] = real ? scores[idx] : 0.f;
      if (out_count && j == 0) out_count[b] = real ? k : 0;
    }
    if (out_points && lane < 3) out_points[w * 3 + lane] = real ? points[(size_t)idx * 3 + lane] : 0.f;
    if (out_desc)
      for (int ch = lane; ch < D; ch += 32) out_desc[w * D + ch] = real ? desc[(size_t)idx * D + ch] : 0.f;
  }
}

// cloud ids 0..B (B = rows past the last cloud) above the 32 score bits
static int keypoint_key_bits(int B) {
  int bits = 0;
  while ((1 << bits) <= B) ++bits;
  return 32 + bits;
}

static size_t select_layout(int N, int B, void* base, int** start, SortBuffers* sb) {
  if (N < 0 || B < 1) return 0;
  Carver cv(base);
  int* s = cv.take<int>((size_t)B + 1);
  SortBuffers x;
  x.keys[0] = cv.take<uint64_t>(N);
  x.keys[1] = cv.take<uint64_t>(N);
  x.vals[0] = cv.take<uint32_t>(N);
  x.vals[1] = cv.take<uint32_t>(N);
  x.block_hist = cv.take<int>(256 * (size_t)sort_num_blocks(N));
  if (start != nullptr) *start = s;
  if (sb != nullptr) *sb = x;
  return cv.off;
}

static size_t sample_layout(int B, void* base, int** start) {
  if (B < 1) return 0;
  Carver cv(base);
  int* s = cv.take<int>((size_t)B + 1);
  if (start != nullptr) *start = s;
  return cv.off;
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_select_keypoints_workspace_bytes(int N, int B) { return select_layout(N, B, nullptr, nullptr, nullptr); }

extern "C" int d3f_select_keypoints(const float* scores, const int* lengths, int B, int N, int k, const float* points,
                                    const float* descriptors, int D, int* out_order, int* out_index, int* out_count,
                                    float* out_points, float* out_descriptors, float* out_scores, void* workspace,
                                    size_t workspace_bytes, d3f_stream_t stream_, const int* n_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const bool per_cloud = out_index || out_count || out_points || out_descriptors || out_scores;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "select_keypoints: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(N >= 0, D3F_ERR_INVALID, "select_keypoints: bad shape N=%d", N);
  D3F_REQUIRE(per_cloud || out_order, D3F_ERR_INVALID, "select_keypoints: no output requested");
  D3F_REQUIRE(!per_cloud || k >= 1, D3F_ERR_INVALID, "select_keypoints: k=%d must be >= 1 for per-cloud outputs", k);
  D3F_REQUIRE(descriptors == nullptr || D >= 1, D3F_ERR_INVALID, "select_keypoints: D=%d must be >= 1", D);
  D3F_REQUIRE(out_points == nullptr || points != nullptr, D3F_ERR_INVALID,
              "select_keypoints: gathered points requested without points");
  D3F_REQUIRE(out_descriptors == nullptr || descriptors != nullptr, D3F_ERR_INVALID,
              "select_keypoints: gathered descriptors requested without descriptors");
  D3F_REQUIRE(lengths != nullptr && workspace != nullptr && (scores != nullptr || N == 0), D3F_ERR_INVALID,
              "select_keypoints: null pointer");
  int* start;
  SortBuffers sb;
  const size_t need = select_layout(N, B, workspace, &start, &sb);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "select_keypoints: workspace too small");
  int rc = launch_batch_start(lengths, B, start, stream);
  if (rc) return rc;
  int cur = 0;
  if (N > 0) {
    const int blocks = min(ceil_div(N, 256), 8 * kNumSMs);
    keypoint_key_kernel<<<blocks, 256, 0, stream>>>(scores, N, n_dev, start, B, sb.keys[0], sb.vals[0]);
    D3F_LAUNCH_CHECK("keypoint_key_kernel");
    cur = radix_sort_pairs(sb, N, keypoint_key_bits(B), stream, n_dev);
    if (cur < 0) return cur;
    if (out_order) {
      keypoint_order_kernel<<<blocks, 256, 0, stream>>>(sb.vals[cur], N, n_dev, out_order);
      D3F_LAUNCH_CHECK("keypoint_order_kernel");
    }
  }
  if (per_cloud) {   // also with N == 0: counts and padding are still written
    const long long slots = (long long)B * k;
    const int blocks = (int)min((slots + 7) / 8, (long long)16 * kNumSMs);
    keypoint_gather_kernel<<<blocks, 256, 0, stream>>>(sb.vals[cur], N, n_dev, start, B, k, scores, points, descriptors,
                                                       D, out_index, out_count, out_points, out_descriptors, out_scores);
    D3F_LAUNCH_CHECK("keypoint_gather_kernel");
  }
  return D3F_OK;
}

extern "C" size_t d3f_sample_keypoints_workspace_bytes(int B) { return sample_layout(B, nullptr, nullptr); }

extern "C" int d3f_sample_keypoints(const int* lengths, int B, int N, int k, uint64_t seed, const float* points,
                                    const float* descriptors, int D, const float* scores, int* out_index,
                                    int* out_count, float* out_points, float* out_descriptors, float* out_scores,
                                    void* workspace, size_t workspace_bytes, d3f_stream_t stream_, const int* n_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "sample_keypoints: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(N >= 0, D3F_ERR_INVALID, "sample_keypoints: bad shape N=%d", N);
  D3F_REQUIRE(k >= 1 && (long long)B * k <= INT_MAX, D3F_ERR_INVALID,
              "sample_keypoints: k=%d must be >= 1 with B*k=%lld within int32", k, (long long)B * k);
  D3F_REQUIRE(out_index || out_count || out_points || out_descriptors || out_scores, D3F_ERR_INVALID,
              "sample_keypoints: no output requested");
  D3F_REQUIRE(descriptors == nullptr || D >= 1, D3F_ERR_INVALID, "sample_keypoints: D=%d must be >= 1", D);
  D3F_REQUIRE(out_points == nullptr || points != nullptr, D3F_ERR_INVALID,
              "sample_keypoints: gathered points requested without points");
  D3F_REQUIRE(out_descriptors == nullptr || descriptors != nullptr, D3F_ERR_INVALID,
              "sample_keypoints: gathered descriptors requested without descriptors");
  D3F_REQUIRE(out_scores == nullptr || scores != nullptr, D3F_ERR_INVALID,
              "sample_keypoints: gathered scores requested without scores");
  D3F_REQUIRE(lengths != nullptr && workspace != nullptr, D3F_ERR_INVALID, "sample_keypoints: null pointer");
  int* start;
  const size_t need = sample_layout(B, workspace, &start);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "sample_keypoints: workspace too small");
  int rc = launch_batch_start(lengths, B, start, stream);
  if (rc) return rc;
  const long long slots = (long long)B * k;
  const int blocks = (int)min((slots + 7) / 8, (long long)16 * kNumSMs);
  keypoint_sample_kernel<<<blocks, 256, 0, stream>>>(N, n_dev, start, B, k, (unsigned long long)seed, scores, points,
                                                     descriptors, D, out_index, out_count, out_points, out_descriptors,
                                                     out_scores);
  D3F_LAUNCH_CHECK("keypoint_sample_kernel");
  return D3F_OK;
}

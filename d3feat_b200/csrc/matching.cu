// Descriptor matching between keypoint sets of cloud pairs -- the host step every consumer of the keypoints runs:
//   geometric_registration/evaluate.py:11-27   build_correspondence: argmin of sqrt(2 - 2 a.b) both ways, mutual pairs
//   utils/tester.py:281-314, demo_registration.py:184-192   Open3D feature matching: source -> target nearest neighbour
//
// Similarity, exactly: s_ij = 0.0f, then for c = 0 .. D-1 in ascending order s_ij = fadd_rn(s_ij, fmul_rn(a_ic, b_jc))
// (no FMA contraction). nn_st[i] = argmax_j s_ij and nn_ts[j] = argmax_i s_ij with numpy's semantics: NaN above
// everything, -0.0 equal to +0.0, ties to the smallest slot. On unit descriptors argmax s is the reference's
// argmin sqrt(2 - 2s), except where the rounding of 2 - 2s merges distinct similarities.
//
// match_tile_kernel: one 64 x 64 tile of (source slot, target slot) per iteration of a CTA, D in chunks of 32 channels
// through shared memory, a 4 x 4 register block per thread. Each row's and each column's best is a 64-bit key
// (score_ord(s) << 32 | ~index): the largest key is the exact argmax with the smallest index on ties, whatever the
// tile split and the order in which CTAs run, so partial results combine with atomicMax. match_finalize_kernel unpacks
// the keys of one pair and compacts the mutual matches in ascending source slot with a block scan. Launches are sized
// by (P, k, D); counts and pair ids are read from the device, so the op can be captured in a CUDA graph.
#include "ops.cuh"

namespace d3f {

namespace {

constexpr int kTile = 64;             // slots per tile side
constexpr int kChunk = 32;            // channels per shared-memory chunk
constexpr int kLd = kTile + 4;        // padded row of the transposed tiles (keeps float4 alignment)
constexpr int kTileThreads = 256;     // 16 x 16 threads, 4 x 4 results each
constexpr int kFinalizeThreads = 256;

// slots of cloud b that hold keypoints; 0 for an id outside [0, B)
__device__ __forceinline__ int slots_of(const int* __restrict__ count, int B, int k, int b) {
  if (b < 0 || b >= B) return 0;
  const int n = __ldg(count + b);
  return n < 0 ? 0 : (n < k ? n : k);
}

__device__ __forceinline__ unsigned long long match_key(float s, int idx) {
  return ((unsigned long long)score_ord(s) << 32) | (unsigned)~idx;
}

// one chunk of a descriptor tile, transposed into smem[c][slot]; slots >= n are not read
__device__ __forceinline__ void load_chunk(float (*dst)[kLd], const float* __restrict__ desc, int cloud, int k, int D,
                                           int slot0, int n, int c0, int dc) {
  for (int e = threadIdx.x; e < kTile * kChunk; e += kTileThreads) {
    const int r = e / kChunk, c = e - r * kChunk;
    float v = 0.f;
    if (c < dc && slot0 + r < n) v = __ldg(desc + ((size_t)cloud * k + slot0 + r) * D + c0 + c);
    dst[c][r] = v;
  }
}

__global__ void __launch_bounds__(kTileThreads)
match_tile_kernel(const float* __restrict__ desc, const int* __restrict__ count, int B, int k, int D,
                  const int* __restrict__ pairs, int P, unsigned long long* __restrict__ row_key,
                  unsigned long long* __restrict__ col_key) {
  __shared__ __align__(16) float As[kChunk][kLd];
  __shared__ __align__(16) float Bs[kChunk][kLd];
  __shared__ unsigned long long rk[kTile], ck[kTile];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int T = (k + kTile - 1) / kTile;
  const long long tiles = (long long)P * T * T;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int p = (int)(t / ((long long)T * T));
    const int rem = (int)(t - (long long)p * T * T);
    const int i0 = (rem / T) * kTile, j0 = (rem % T) * kTile;
    const int src = __ldg(pairs + 2 * p), tgt = __ldg(pairs + 2 * p + 1);
    int ns = slots_of(count, B, k, src), nt = slots_of(count, B, k, tgt);
    if (ns == 0 || nt == 0) ns = nt = 0;             // a pair naming no cloud, or an empty one, matches nothing
    if (i0 >= ns || j0 >= nt) continue;              // uniform across the CTA
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
    for (int c0 = 0; c0 < D; c0 += kChunk) {
      const int dc = min(kChunk, D - c0);
      __syncthreads();                               // previous chunk (or tile) fully consumed
      load_chunk(As, desc, src, k, D, i0, ns, c0, dc);
      load_chunk(Bs, desc, tgt, k, D, j0, nt, c0, dc);
      __syncthreads();
#pragma unroll 4
      for (int c = 0; c < dc; ++c) {
        const float4 a = *reinterpret_cast<const float4*>(&As[c][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[c][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[r][q] = __fadd_rn(acc[r][q], __fmul_rn(av[r], bv[q]));
      }
    }
    if (threadIdx.x < kTile) ck[threadIdx.x] = 0ull;
    __syncthreads();
    // a row's 64 columns live in the 16 lanes of one half-warp: a shuffle reduction gives its tile best
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = i0 + ty * 4 + r;
      unsigned long long best = 0ull;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int j = j0 + tx * 4 + q;
        if (i < ns && j < nt) best = max(best, match_key(acc[r][q], j));
      }
#pragma unroll
      for (int o = 8; o >= 1; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
      if (tx == 0) rk[ty * 4 + r] = best;
    }
    // a column's 64 rows span both half-warps of all 8 warps: shuffle across the halves, then one atomic per warp
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + tx * 4 + q;
      unsigned long long best = 0ull;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = i0 + ty * 4 + r;
        if (i < ns && j < nt) best = max(best, match_key(acc[r][q], i));
      }
      best = max(best, __shfl_xor_sync(0xffffffffu, best, 16));
      if ((ty & 1) == 0 && best) atomicMax(&ck[tx * 4 + q], best);
    }
    __syncthreads();
    if (threadIdx.x < kTile) {
      const int i = i0 + threadIdx.x;
      if (i < ns) atomicMax(row_key + (size_t)p * k + i, rk[threadIdx.x]);
    } else if (threadIdx.x < 2 * kTile) {
      const int j = j0 + threadIdx.x - kTile;
      if (j < nt) atomicMax(col_key + (size_t)p * k + j, ck[threadIdx.x - kTile]);
    }
  }
}

// exclusive block scan of one flag per thread; *total receives the sum
__device__ __forceinline__ int block_exclusive_scan(int flag, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int v = flag;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) warp_sums[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int w = lane < kFinalizeThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    if (lane < kFinalizeThreads / 32) warp_sums[lane] = w;   // inclusive
    if (lane == 31) *total = w;
  }
  __syncthreads();
  const int before = warp == 0 ? 0 : warp_sums[warp - 1];
  const int r = before + v - flag;
  __syncthreads();                                   // warp_sums is reused by the next call
  return r;
}

__global__ void __launch_bounds__(kFinalizeThreads)
match_finalize_kernel(const int* __restrict__ count, int B, int k, const int* __restrict__ pairs, int P,
                      const unsigned long long* __restrict__ row_key, const unsigned long long* __restrict__ col_key,
                      int* __restrict__ nn_st, float* __restrict__ sim_st, int* __restrict__ nn_ts,
                      float* __restrict__ sim_ts, int* __restrict__ matches, int* __restrict__ n_matches) {
  __shared__ int warp_sums[kFinalizeThreads / 32];
  __shared__ int chunk_total;
  for (int p = blockIdx.x; p < P; p += gridDim.x) {
    const int src = __ldg(pairs + 2 * p), tgt = __ldg(pairs + 2 * p + 1);
    int ns = slots_of(count, B, k, src), nt = slots_of(count, B, k, tgt);
    if (ns == 0 || nt == 0) ns = nt = 0;
    const size_t base = (size_t)p * k;
    for (int j = threadIdx.x; j < k; j += kFinalizeThreads) {
      const unsigned long long key = j < nt ? col_key[base + j] : 0ull;
      nn_ts[base + j] = key ? (int)~(unsigned)key : -1;
      sim_ts[base + j] = key ? ord2f((unsigned)(key >> 32)) : 0.f;
    }
    int n_out = 0;
    for (int i0 = 0; i0 < k; i0 += kFinalizeThreads) {   // uniform trip count: every thread reaches the scans
      const int i = i0 + threadIdx.x;
      const unsigned long long key = i < ns ? row_key[base + i] : 0ull;
      const int j = key ? (int)~(unsigned)key : -1;
      if (i < k) {
        nn_st[base + i] = j;
        sim_st[base + i] = key ? ord2f((unsigned)(key >> 32)) : 0.f;
      }
      const int mutual = j >= 0 && (int)~(unsigned)col_key[base + j] == i;
      const int pos = n_out + block_exclusive_scan(mutual, warp_sums, &chunk_total);
      if (mutual) {
        matches[2 * (base + pos)] = i;
        matches[2 * (base + pos) + 1] = j;
      }
      n_out += chunk_total;
    }
    for (int r = n_out + threadIdx.x; r < k; r += kFinalizeThreads) {
      matches[2 * (base + r)] = -1;
      matches[2 * (base + r) + 1] = -1;
    }
    if (threadIdx.x == 0) n_matches[p] = n_out;
  }
}

// the best key of every row and every column of each pair's k x k similarity matrix
size_t match_layout(int k, int P, void* base, unsigned long long** row_key, unsigned long long** col_key) {
  if (k < 1 || P < 1 || (long long)P * k > INT32_MAX) return 0;
  Carver cv(base);
  unsigned long long* r = cv.take<unsigned long long>((size_t)P * k);
  unsigned long long* c = cv.take<unsigned long long>((size_t)P * k);
  if (row_key != nullptr) *row_key = r;
  if (col_key != nullptr) *col_key = c;
  return cv.off;
}

}  // namespace
}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_match_descriptors_workspace_bytes(int k, int P) {
  return match_layout(k, P, nullptr, nullptr, nullptr);
}

extern "C" int d3f_match_descriptors(const float* desc, const int* count, int B, int k, int D, const int* pairs, int P,
                                     int* nn_st, float* sim_st, int* nn_ts, float* sim_ts, int* matches, int* n_matches,
                                     void* workspace, size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "match_descriptors: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(k >= 1 && D >= 1 && P >= 1, D3F_ERR_INVALID, "match_descriptors: bad shape k=%d D=%d P=%d", k, D, P);
  D3F_REQUIRE((long long)P * k <= INT32_MAX, D3F_ERR_INVALID, "match_descriptors: P*k=%lld exceeds int32",
              (long long)P * k);
  D3F_REQUIRE(desc && count && pairs && nn_st && sim_st && nn_ts && sim_ts && matches && n_matches && workspace,
              D3F_ERR_INVALID, "match_descriptors: null pointer");
  unsigned long long *row_key, *col_key;
  const size_t need = match_layout(k, P, workspace, &row_key, &col_key);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "match_descriptors: workspace too small");
  // key 0 is below every real key (score_ord is never 0): "no candidate yet". One memset over both key arrays.
  D3F_CUDA(cudaMemsetAsync(row_key, 0, need, stream));
  const int T = ceil_div(k, kTile);
  const long long tiles = (long long)P * T * T;
  const int blocks = (int)min(tiles, (long long)32 * kNumSMs);
  match_tile_kernel<<<blocks, kTileThreads, 0, stream>>>(desc, count, B, k, D, pairs, P, row_key, col_key);
  D3F_LAUNCH_CHECK("match_tile_kernel");
  match_finalize_kernel<<<min(P, 8 * kNumSMs), kFinalizeThreads, 0, stream>>>(count, B, k, pairs, P, row_key, col_key,
                                                                             nn_st, sim_st, nn_ts, sim_ts, matches,
                                                                             n_matches);
  D3F_LAUNCH_CHECK("match_finalize_kernel");
  return D3F_OK;
}

// The training update and the data-parallel reduction (contract: include/d3feat_b200.h, restated in
// oracle/optim_np.py):
//
//   momentum_clip_update   utils/trainer.py:116-156: tf.clip_by_norm on each gradient on its own (TF 1.12), then
//                          ApplyMomentum (accum = accum*momentum + g; var -= accum*lr), for every tensor of a table
//   rank_mean              out[p] = (sum over ranks of x[r, p], in rank order, fp64) / R
//
// The update is two launches for all tensors together. momentum_l2_partial_kernel sums the squares of every 2048-element
// block of every gradient sequentially in fp64, one lane per block. momentum_update_kernel gives each CTA a
// contiguous run of blocks; for each tensor of its run it adds the tensor's block partials in block order (every CTA
// that touches a tensor computes the same norm) and updates its elements. Each CTA derives the block layout from the
// table itself (a prefix over the tensors' block counts in shared memory), so the host never reads the table back. No
// float atomics: the results are bitwise identical run to run and across streams.
#include "ops.cuh"

namespace d3f {

constexpr int kOptBlock = 2048;          // elements per partial of a tensor's sum of squares
constexpr int kOptMaxTensors = 1024;     // tensors per call: the block prefix (T + 1 entries) lives in shared memory
constexpr int kPartialThreads = 64;      // a warp per 32 consecutive 2048-element blocks
constexpr int kUpdateThreads = 256;
constexpr long long kMaxTensorBlocks = 1ll << 40;   // a garbage numel cannot overflow the prefix

__device__ __forceinline__ long long tensor_blocks(long long n) {
  return n > 0 ? min((n + kOptBlock - 1) / kOptBlock, kMaxTensorBlocks) : 0;
}

// first[t] = blocks of tensors 0..t-1, first[T] = all blocks: each thread counts a contiguous run of tensors, then a
// block-wide exclusive scan (warp shuffles, one warp over the warp totals). warp_tot[32] is scratch.
__device__ void block_prefix(const d3f_momentum_tensor* __restrict__ table, int T, long long* first,
                             long long* warp_tot) {
  const int per = (T + (int)blockDim.x - 1) / (int)blockDim.x;
  const int lo = min(T, (int)threadIdx.x * per), hi = min(T, lo + per);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (int)blockDim.x >> 5;
  long long v = 0;
  for (int t = lo; t < hi; ++t) v += tensor_blocks(table[t].numel);
  long long x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[w] = x;
  __syncthreads();
  if (w == 0) {
    long long t = lane < nw ? warp_tot[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    if (lane < nw) warp_tot[lane] = t;
  }
  __syncthreads();
  long long a = (w > 0 ? warp_tot[w - 1] : 0) + x - v;
  for (int t = lo; t < hi; ++t) {
    first[t] = a;
    a += tensor_blocks(table[t].numel);
  }
  if (threadIdx.x == 0) first[T] = warp_tot[nw - 1];
  __syncthreads();
}

// the tensor of global block b < first[T]: the largest t with first[t] <= b (empty tensors are skipped over)
__device__ __forceinline__ int tensor_of(const long long* first, int T, long long b) {
  int lo = 0, hi = T - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// partial[b] = sum of g^2 over global block b, sequentially in fp64 (blocks at or past cap, the workspace's capacity,
// are not written). A warp takes 32 consecutive blocks, one per lane, so every instruction of the sequential sums does
// 32 blocks' work. The blocks pass through shared memory in chunks of kChunk elements: the warp loads a chunk of all 32
// blocks coalesced (each block's kChunk elements are one 256-byte row), then each lane adds its own row in order while
// the next chunk's loads are already in flight in registers. g^2 of an fp32 value is exact in fp64 (24-bit
// significands, exponents well inside fp64's range), so fma(v, v, acc) rounds once per addition, as acc + v*v does;
// elements past a block's end are read as zeros, and adding +0 to a sum >= 0 changes nothing.
constexpr int kChunk = 64;
constexpr int kChunkPerLane = 32 * kChunk / 32;   // elements of one chunk each lane loads (two per block row)

__global__ void __launch_bounds__(kPartialThreads) momentum_l2_partial_kernel(
    const d3f_momentum_tensor* __restrict__ table, int T, long long cap, double* __restrict__ partial) {
  __shared__ float tile[kPartialThreads / 32][32][kChunk + 1];   // +1: the row-per-lane reads are conflict-free
  __shared__ const float* row_g[kPartialThreads / 32][32];
  __shared__ int row_n[kPartialThreads / 32][32];
  __shared__ long long warp_tot[32];
  extern __shared__ long long prefix_smem[];   // first[T + 1]
  long long* first = prefix_smem;
  block_prefix(table, T, first, warp_tot);
  const long long nblk = min(first[T], cap);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long groups = (nblk + 31) / 32;
  const long long stride = (long long)gridDim.x * (kPartialThreads / 32);
  for (long long grp = (long long)blockIdx.x * (kPartialThreads / 32) + w; grp < groups; grp += stride) {
    const long long b = grp * 32 + lane;
    int n = 0;
    const float* g = nullptr;
    if (b < nblk) {
      const int t = tensor_of(first, T, b);
      const long long e0 = (b - first[t]) * kOptBlock;
      n = (int)min(table[t].numel - e0, (long long)kOptBlock);
      g = table[t].grad + e0;
    }
    row_g[w][lane] = g;
    row_n[w][lane] = n;
    int nmax = n;
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    const int chunks = (nmax + kChunk - 1) / kChunk;
    __syncwarp();
    float next[kChunkPerLane];
    auto load = [&](int k) {
#pragma unroll
      for (int r = 0; r < 32; ++r) {
#pragma unroll
        for (int h = 0; h < kChunk / 32; ++h) {
          const int i = k * kChunk + h * 32 + lane;
          next[r * (kChunk / 32) + h] = i < row_n[w][r] ? __ldg(row_g[w][r] + i) : 0.f;
        }
      }
    };
    double acc = 0.0;
    if (chunks > 0) load(0);
    for (int k = 0; k < chunks; ++k) {
      __syncwarp();                      // the previous chunk's rows have been read
#pragma unroll
      for (int r = 0; r < 32; ++r) {
#pragma unroll
        for (int h = 0; h < kChunk / 32; ++h) tile[w][r][h * 32 + lane] = next[r * (kChunk / 32) + h];
      }
      __syncwarp();
      if (k + 1 < chunks) load(k + 1);   // in flight while the lanes add this chunk
#pragma unroll 16
      for (int j = 0; j < kChunk; ++j) {
        const double v = (double)tile[w][lane][j];
        acc = fma(v, v, acc);
      }
    }
    if (b < nblk) partial[b] = acc;
    __syncwarp();                        // row_g / row_n are rewritten for the next group
  }
}

__device__ __forceinline__ void momentum_element(float g, float& accum, float& var, float lr, float momentum, float c,
                                                 float M) {
  if (c > 0.f) g = __fdiv_rn(__fmul_rn(g, c), M);
  accum = __fadd_rn(__fmul_rn(accum, momentum), g);
  var = __fsub_rn(var, __fmul_rn(accum, lr));
}

// clip (c > 0) and the momentum update over this CTA's contiguous run of blocks
__global__ void __launch_bounds__(kUpdateThreads, 4) momentum_update_kernel(
    const d3f_momentum_tensor* __restrict__ table, int T, long long cap, const double* __restrict__ partial, float lr,
    float momentum, float c) {
  extern __shared__ long long prefix_smem[];   // first[T + 1]
  __shared__ long long warp_tot[32];
  __shared__ float s_max;
  long long* first = prefix_smem;
  block_prefix(table, T, first, warp_tot);
  const long long nblk = min(first[T], cap);
  const long long per = (nblk + gridDim.x - 1) / gridDim.x;
  const long long b1 = min(nblk, (long long)blockIdx.x * per + per);
  for (long long b = (long long)blockIdx.x * per; b < b1;) {
    const int t = tensor_of(first, T, b);
    const long long be = min(b1, first[t + 1]);
    float M = 0.f;
    if (c > 0.f) {
      if (threadIdx.x == 0) {
        double l2 = 0.0;
        const long long ke = min(first[t + 1], cap);
#pragma unroll 8
        for (long long k = first[t]; k < ke; ++k) l2 += partial[k];
        // TF: l2norm = where(l2sum > 0, sqrt(l2sum), l2sum); maximum(l2norm, clip_norm)
        const float norm = l2 > 0.0 ? (float)sqrt(l2) : (float)l2;
        s_max = norm < c ? c : norm;
      }
      __syncthreads();
      M = s_max;
    }
    const float* __restrict__ g = table[t].grad;
    float* __restrict__ accum = table[t].accum;
    float* __restrict__ var = table[t].var;
    const long long hi = min(table[t].numel, (be - first[t]) * kOptBlock);
    long long i = (b - first[t]) * kOptBlock + threadIdx.x;
    constexpr int U = 4;   // four elements per thread in flight
    for (; i + (U - 1) * kUpdateThreads < hi; i += U * kUpdateThreads) {
      float gv[U], av[U], vv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        gv[u] = __ldg(g + i + u * kUpdateThreads);
        av[u] = accum[i + u * kUpdateThreads];
        vv[u] = var[i + u * kUpdateThreads];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        momentum_element(gv[u], av[u], vv[u], lr, momentum, c, M);
        accum[i + u * kUpdateThreads] = av[u];
        var[i + u * kUpdateThreads] = vv[u];
      }
    }
    for (; i < hi; i += kUpdateThreads) {
      float av = accum[i], vv = var[i];
      momentum_element(__ldg(g + i), av, vv, lr, momentum, c, M);
      accum[i] = av;
      var[i] = vv;
    }
    __syncthreads();   // s_max is rewritten for the next tensor
    b = be;
  }
}

// out may be x's row 0: each element's rank-0 value is read before it is written, by the same thread. R = 1 copies
// (the fp64 round trip would canonicalise a NaN's payload).
__global__ void __launch_bounds__(256) rank_mean_kernel(const float* x, int R, long long P, float* out) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
    if (R == 1) {
      out[p] = x[p];
      continue;
    }
    double s = (double)x[p];
#pragma unroll 4
    for (int r = 1; r < R; ++r) s += (double)x[(size_t)r * P + p];
    out[p] = (float)(s / (double)R);
  }
}

static size_t prefix_smem_bytes(int T) { return (size_t)(T + 1) * sizeof(long long); }

static long long partial_capacity(int T, long long numel_total) {
  return (numel_total + kOptBlock - 1) / kOptBlock + T;   // every tensor ends at most one partial block early
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_momentum_clip_workspace_bytes(int T, long long numel_total) {
  if (T < 0 || T > kOptMaxTensors || numel_total < 0) return 0;
  return align_up((size_t)partial_capacity(T, numel_total) * sizeof(double), 256) + 256;
}

extern "C" int d3f_momentum_clip_update(const d3f_momentum_tensor* table, int T, long long numel_total, float lr,
                                        float momentum, float clip_norm, void* workspace, size_t workspace_bytes,
                                        d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(T >= 0 && T <= kOptMaxTensors && numel_total >= 0, D3F_ERR_INVALID,
              "momentum_clip_update: bad shape T=%d numel_total=%lld (T in [0, %d])", T, numel_total, kOptMaxTensors);
  D3F_REQUIRE(isfinite(lr) && isfinite(momentum) && isfinite(clip_norm), D3F_ERR_INVALID,
              "momentum_clip_update: lr=%g momentum=%g clip_norm=%g must be finite", (double)lr, (double)momentum,
              (double)clip_norm);
  if (T == 0 || numel_total == 0) return D3F_OK;
  D3F_REQUIRE(table != nullptr && workspace != nullptr, D3F_ERR_INVALID, "momentum_clip_update: null pointer");
  D3F_REQUIRE(workspace_bytes >= d3f_momentum_clip_workspace_bytes(T, numel_total), D3F_ERR_WORKSPACE,
              "momentum_clip_update: workspace too small");
  const long long cap = partial_capacity(T, numel_total);
  double* partial = (double*)workspace;
  if (clip_norm > 0.f) {
    const long long warps = (cap + 31) / 32;            // a warp per 32 blocks
    const long long per_cta = kPartialThreads / 32;
    const long long g = min((warps + per_cta - 1) / per_cta, (long long)kNumSMs * 8);
    momentum_l2_partial_kernel<<<(int)g, kPartialThreads, prefix_smem_bytes(T), stream>>>(
        table, T, cap, partial);
    D3F_LAUNCH_CHECK("momentum_l2_partial_kernel");
  }
  const int grid = (int)min(cap, (long long)kNumSMs * 4);   // one wave
  momentum_update_kernel<<<grid, kUpdateThreads, prefix_smem_bytes(T), stream>>>(
      table, T, cap, partial, lr, momentum, clip_norm);
  D3F_LAUNCH_CHECK("momentum_update_kernel");
  return D3F_OK;
}

extern "C" int d3f_rank_mean(const float* x, int R, long long P, float* out, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(R >= 1 && P >= 0 && (double)R * (double)P < 9.0e18, D3F_ERR_INVALID,
              "rank_mean: bad shape R=%d P=%lld", R, P);
  if (P == 0) return D3F_OK;
  D3F_REQUIRE(x != nullptr && out != nullptr, D3F_ERR_INVALID, "rank_mean: null pointer");
  const int grid = (int)min((P + 255) / 256, (long long)kNumSMs * 16);
  rank_mean_kernel<<<grid, 256, 0, stream>>>(x, R, P, out);
  D3F_LAUNCH_CHECK("rank_mean_kernel");
  return D3F_OK;
}

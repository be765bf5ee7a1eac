// Backward pass of rigid KPConv (kernels/convolution_ops.py:161-255) and of the unary convolution (:90-99).
//
//   out[q,o] = (1/nn_q) sum_h sum_k w(q,h,k) sum_c f[idx[q,h],c] W[k,c,o]          (nn_q held constant)
//   G[q,o]   = dout[q,o] / nn_q
//   dW[k,c,o] = sum_q wf[q,k,c] G[q,o]                  wf = stage 1 of the forward, recomputed chunk by chunk
//   df[s,c]   = sum_{(q,h): idx[q,h] = s} sum_k w(q,h,k) sum_o G[q,o] W[k,c,o]
//
// The feature gradient is a forward KPConv over the transposed neighbourhood: queries and supports swap roles, the
// reverse table rev[s,:] lists the queries that reach s (ascending (q, h), padded with the shadow index), the kernel
// points are -Kp (fl(q - s) = -fl(s - q) and fl(x + kp) = -fl(-x - kp), so every d^2, weight and closest-point choice
// is the forward's own), the features are G and the weights W^T = W.permute(0, 2, 1), without normalisation. So it
// runs through kpconv_forward_impl and its tensor-core kernels.
//
// The weight gradient is A^T B with the reduction over rows (A = wf or x, B = G or dout): fixed 2048-row blocks, each
// with fresh accumulators folded every 64 rows, partial tiles written per block and summed in float64 in block order
// by a second pass. No float atomics: the gradients are bitwise identical run to run.
#include "ops.cuh"
#include "sort.cuh"

namespace d3f {

constexpr int kWgRowBlock = 2048;   // rows per partial of the weight gradient
constexpr int kWgFold = 64;         // rows per fresh accumulator inside a block
constexpr int kWgStage = 16;        // rows per shared-memory stage

// ---- reverse neighbour table -------------------------------------------------------------------------------------
// Entry i = q*H + h of idx is real when q < rows_q and 0 <= idx < rows_s. keys: the support (rows past it: Ns, sorted
// last), vals: the query; counts[s] += 1 per real entry (integer atomics: exact in any order).
__global__ void __launch_bounds__(256) reverse_keys_kernel(const int* __restrict__ idx, int Nq, int Ns, int H,
                                                           const int* __restrict__ nq_dev, const int* __restrict__ ns_dev,
                                                           uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                           int* __restrict__ counts) {
  const int nq = dyn_rows(Nq, nq_dev), ns = dyn_rows(Ns, ns_dev);
  const long long E = (long long)Nq * H;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < E; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i / H);
    const int s = idx[i];
    const bool real = q < nq && s >= 0 && s < ns;
    if (real) atomicAdd(&counts[s], 1);
    if (keys != nullptr) {
      keys[i] = real ? (uint64_t)s : (uint64_t)Ns;
      vals[i] = (uint32_t)q;
    }
  }
}

__global__ void __launch_bounds__(1024) max_count_kernel(const int* __restrict__ counts, int n, int* __restrict__ out) {
  __shared__ int wmax[32];
  int m = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = max(m, counts[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = wmax[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) *out = m;
  }
}

// rev[s, j] = j-th query reaching s (sorted vals from offs[s]), or `pad` (the shadow of the transposed problem)
__global__ void __launch_bounds__(256) reverse_fill_kernel(const int* __restrict__ counts, const int* __restrict__ offs,
                                                           const uint32_t* __restrict__ sorted_q, int Ns, int Hr, int pad,
                                                           int* __restrict__ rev) {
  const long long total = (long long)Ns * Hr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(i / Hr), j = (int)(i % Hr);
    rev[i] = j < counts[s] ? (int)sorted_q[offs[s] + j] : pad;
  }
}

// ---- G = dout / nn, from the forward's support pack (same clamp of the index, same flag) --------------------------
__global__ void __launch_bounds__(256) grad_rowscale_kernel(const float* __restrict__ dout, const int* __restrict__ idx,
                                                            const float4* __restrict__ s4, int Nq, int Ns, int H, int Cout,
                                                            int normalize, const int* __restrict__ nq_dev,
                                                            const int* __restrict__ ns_dev, float* __restrict__ G) {
  const int nq = dyn_rows(Nq, nq_dev), ns = dyn_rows(Ns, ns_dev);
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= Nq) return;
  float* g = G + (size_t)q * Cout;
  if (q >= nq) {                     // rows past the count: dout is never read there
    for (int o = lane; o < Cout; o += 32) g[o] = 0.f;
    return;
  }
  float inv = 1.f;
  if (normalize) {
    int nn = 0;
    for (int h = lane; h < H; h += 32) {
      int id = idx[(size_t)q * H + h];
      if (id < 0 || id > ns) id = ns;
      nn += s4[id].w > 0.f ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nn += __shfl_xor_sync(0xffffffffu, nn, o);
    inv = 1.f / (float)max(nn, 1);
  }
  for (int o = lane; o < Cout; o += 32) g[o] = dout[(size_t)q * Cout + o] * inv;
}

// WT[k][o][c] = W[k][c][o]
__global__ void __launch_bounds__(256) transpose_weights_kernel(const float* __restrict__ W, int K, int Cin, int Cout,
                                                                float* __restrict__ WT) {
  const long long total = (long long)K * Cin * Cout;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cin);
    const long long r = i / Cin;
    const int o = (int)(r % Cout), k = (int)(r / Cout);
    WT[i] = W[((size_t)k * Cin + c) * Cout + o];
  }
}

__global__ void negate_kernel(const float* __restrict__ x, int n, float* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = -x[i];
}

// ---- weight gradient: partial[blk, m, n] = sum over the rows r of block blk of A[r, m] B[r, n] ----------------------
// BM x BN output tile per CTA (BM * BN = 4096), 4 x 4 per thread, rows staged 16 at a time through shared memory. Rows
// at or past min(R, *r_dev - r_off) are not read. Every (blk, m, n) of the grid is written (zero for an empty block).
template <int BN>
__global__ void __launch_bounds__(256) wgrad_partial_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                            int R, int M, int N, const int* __restrict__ r_dev, int r_off,
                                                            float* __restrict__ partial) {
  constexpr int BM = 4096 / BN;
  constexpr int TNT = BN / 4;        // threads along n
  __shared__ __align__(16) float As[kWgStage][BM];
  __shared__ __align__(16) float Bs[kWgStage][BN];
  const int rows = r_dev ? min(R, max(__ldg(r_dev) - r_off, 0)) : R;
  const int tn = threadIdx.x % TNT, tm = threadIdx.x / TNT;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int rb = blockIdx.z * kWgRowBlock, re = min(rows, rb + kWgRowBlock);
  float acc[4][4], tot[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = tot[i][j] = 0.f;
  for (int r0 = rb; r0 < re; r0 += kWgStage) {
#pragma unroll
    for (int e = threadIdx.x; e < kWgStage * BM; e += 256) {
      const int rr = e / BM, mm = e % BM;
      const int r = r0 + rr, m = m0 + mm;
      As[rr][mm] = (r < re && m < M) ? A[(size_t)r * M + m] : 0.f;
    }
#pragma unroll
    for (int e = threadIdx.x; e < kWgStage * BN; e += 256) {
      const int rr = e / BN, nn = e % BN;
      const int r = r0 + rr, n = n0 + nn;
      Bs[rr][nn] = (r < re && n < N) ? B[(size_t)r * N + n] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < kWgStage; ++rr) {
      const float4 a = *reinterpret_cast<const float4*>(&As[rr][tm * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[rr][tn * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
    if (((r0 - rb) / kWgStage + 1) % (kWgFold / kWgStage) == 0) {   // fresh accumulators every 64 rows
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          tot[i][j] += acc[i][j];
          acc[i][j] = 0.f;
        }
    }
  }
  float* out = partial + (size_t)blockIdx.z * M * N;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + tm * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tn * 4 + j;
      if (n < N) out[(size_t)m * N + n] = tot[i][j] + acc[i][j];
    }
  }
}

// out[i] = sum over the blocks b in ascending order of partial[b, i], in float64, rounded once
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ partial, int nblk, long long MN,
                                                           float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < MN; i += (long long)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < nblk; ++b) s += (double)partial[(size_t)b * MN + i];
    out[i] = (float)s;
  }
}

static int grid_for(long long n, int threads = 256) {
  long long b = (n + threads - 1) / threads;
  return (int)max(1ll, min(b, (long long)kNumSMs * 16));
}

int reverse_csr(const int* idx, int Nq, int Ns, int H, const int* nq_dev, const int* ns_dev, const SortBuffers& sb,
                int* counts, int* offs, int* scan_scratch, const uint32_t** sorted_q, cudaStream_t stream) {
  // a stable sort of the (q, h)-ordered entries by support gives ascending (s, q, h)
  const int E = Nq * H;
  D3F_CUDA(cudaMemsetAsync(counts, 0, (size_t)(Ns + 1) * sizeof(int), stream));
  reverse_keys_kernel<<<grid_for((long long)E), 256, 0, stream>>>(idx, Nq, Ns, H, nq_dev, ns_dev, sb.keys[0],
                                                                   sb.vals[0], counts);
  D3F_LAUNCH_CHECK("reverse_keys_kernel");
  int nbits = 1;
  while (nbits < 31 && (1 << nbits) <= Ns) ++nbits;   // keys are in [0, Ns]
  const int cur = radix_sort_pairs(sb, E, nbits, stream);
  if (cur < 0) return cur;
  const int rc = exclusive_scan_i32(counts, offs, Ns + 1, nullptr, scan_scratch, stream);   // counts[Ns] = 0
  if (rc) return rc;
  *sorted_q = sb.vals[cur];
  return D3F_OK;
}

static int wgrad_blocks(int rows) { return rows > 0 ? ceil_div(rows, kWgRowBlock) : 1; }

static int launch_wgrad_partial(const float* A, const float* B, int R, int M, int N, const int* r_dev, int r_off,
                                int nblk, float* partial, cudaStream_t stream) {
  if (N <= 32) {
    dim3 grid(ceil_div(M, 128), ceil_div(N, 32), nblk);
    wgrad_partial_kernel<32><<<grid, 256, 0, stream>>>(A, B, R, M, N, r_dev, r_off, partial);
  } else {
    dim3 grid(ceil_div(M, 64), ceil_div(N, 64), nblk);
    wgrad_partial_kernel<64><<<grid, 256, 0, stream>>>(A, B, R, M, N, r_dev, r_off, partial);
  }
  D3F_LAUNCH_CHECK("wgrad_partial_kernel");
  return D3F_OK;
}

static int launch_wgrad_reduce(const float* partial, int nblk, long long MN, float* out, cudaStream_t stream) {
  wgrad_reduce_kernel<<<grid_for(MN), 256, 0, stream>>>(partial, nblk, MN, out);
  D3F_LAUNCH_CHECK("wgrad_reduce_kernel");
  return D3F_OK;
}

// ---- KPConv --------------------------------------------------------------------------------------------------------
struct BackwardLayout {
  // persistent
  size_t s4, G, rev, nKp, WT, WTp;
  // phase region (reused: reverse table build, then the transposed forward, then the weight gradient)
  size_t region;
  size_t counts, offs, scan, keys0, keys1, vals0, vals1, hist, width;   // inside region, table build
  size_t fwd_bytes;                                                    // inside region, transposed forward
  size_t wf, partial;                                                  // inside region, weight gradient
  size_t total;
  int chunk, bpc, n_chunks;
};

static BackwardLayout backward_layout(int Nq, int Ns, int H, int K, int Cin, int Cout, int Hr) {
  BackwardLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) { off = align_up(off, 256); size_t r = off; off += bytes; return r; };
  L.s4 = take((size_t)(Ns + 1) * sizeof(float4));
  L.G = take((size_t)Nq * Cout * sizeof(float));
  L.rev = take((size_t)Ns * (Hr > 0 ? Hr : 1) * sizeof(int));
  L.nKp = take((size_t)K * 3 * sizeof(float));
  L.WT = take((size_t)K * Cout * Cin * sizeof(float));
  L.WTp = take(tc_packed_floats(K * Cout, Cin) * sizeof(float));
  L.region = align_up(off, 256);
  // table build
  const long long E = (long long)Nq * H;
  size_t r = 0;
  auto rtake = [&](size_t bytes) { r = align_up(r, 256); size_t o = r; r += bytes; return o; };
  L.counts = rtake((size_t)(Ns + 1) * sizeof(int));
  L.offs = rtake((size_t)(Ns + 1) * sizeof(int));
  L.scan = rtake((size_t)(scan_num_blocks(Ns + 1) + 1) * sizeof(int));
  L.width = rtake(sizeof(int));
  L.keys0 = rtake((size_t)E * sizeof(uint64_t));
  L.keys1 = rtake((size_t)E * sizeof(uint64_t));
  L.vals0 = rtake((size_t)E * sizeof(uint32_t));
  L.vals1 = rtake((size_t)E * sizeof(uint32_t));
  L.hist = rtake((size_t)256 * sort_num_blocks((int)E) * sizeof(int));
  const size_t build = align_up(r, 256);
  // transposed forward: Ns queries, Nq supports, Hr neighbours, Cout -> Cin channels
  L.fwd_bytes = kpconv_workspace_bytes(Ns, Nq, Hr, K, Cout, Cin);
  // weight gradient
  L.chunk = kpconv_chunk_queries(K, Cin);
  if (L.chunk > Nq) L.chunk = Nq > 0 ? Nq : 1;
  L.n_chunks = Nq > 0 ? ceil_div(Nq, L.chunk) : 0;
  L.bpc = wgrad_blocks(L.chunk);
  r = 0;
  L.wf = rtake((size_t)L.chunk * K * Cin * sizeof(float));
  L.partial = rtake((size_t)(L.n_chunks > 0 ? L.n_chunks : 1) * L.bpc * K * Cin * Cout * sizeof(float));
  const size_t wgrad = align_up(r, 256);
  size_t region = build;
  if (L.fwd_bytes > region) region = L.fwd_bytes;
  if (wgrad > region) region = wgrad;
  L.total = L.region + region + 1024;
  return L;
}

size_t kpconv_backward_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout, int Hr) {
  if (Nq < 0 || Ns < 0 || H < 0 || K < 1 || Cin < 1 || Cout < 1 || Hr < 0) return 0;
  return backward_layout(Nq, Ns, H, K, Cin, Cout, Hr).total;
}

int kpconv_reverse_width(const int* idx, int Nq, int Ns, int H, int* width, void* workspace, size_t workspace_bytes,
                         cudaStream_t stream, const int* nq_dev, const int* ns_dev) {
  D3F_REQUIRE(Nq >= 0 && Ns >= 0 && H >= 0 && width != nullptr, D3F_ERR_INVALID,
              "kpconv_reverse_width: bad arguments Nq=%d Ns=%d H=%d", Nq, Ns, H);
  *width = 0;
  if (Nq == 0 || Ns == 0 || H == 0) return D3F_OK;
  D3F_REQUIRE(idx != nullptr && workspace != nullptr, D3F_ERR_INVALID, "kpconv_reverse_width: null pointer");
  const BackwardLayout L = backward_layout(Nq, Ns, H, 1, 1, 1, 0);
  D3F_REQUIRE(workspace_bytes >= L.region + L.width + sizeof(int), D3F_ERR_WORKSPACE,
              "kpconv_reverse_width: workspace too small");
  char* reg = static_cast<char*>(workspace) + L.region;
  int* counts = reinterpret_cast<int*>(reg + L.counts);
  int* dwidth = reinterpret_cast<int*>(reg + L.width);
  D3F_CUDA(cudaMemsetAsync(counts, 0, (size_t)Ns * sizeof(int), stream));
  reverse_keys_kernel<<<grid_for((long long)Nq * H), 256, 0, stream>>>(idx, Nq, Ns, H, nq_dev, ns_dev, nullptr, nullptr,
                                                                       counts);
  D3F_LAUNCH_CHECK("reverse_keys_kernel");
  max_count_kernel<<<1, 1024, 0, stream>>>(counts, Ns, dwidth);
  D3F_LAUNCH_CHECK("max_count_kernel");
  D3F_CUDA(cudaMemcpyAsync(width, dwidth, sizeof(int), cudaMemcpyDeviceToHost, stream));
  D3F_CUDA(cudaStreamSynchronize(stream));
  return D3F_OK;
}

int kpconv_backward(const float* q, const float* s, const int* idx, const float* feat, const float* Kp, const float* W,
                    const float* dout, int Nq, int Ns, int H, int Hr, int K, int Cin, int Cout, float extent,
                    int influence, int mode, int normalize, int tensor_cores, float* dfeat, float* dW, void* workspace,
                    size_t workspace_bytes, cudaStream_t stream, const int* nq_dev, const int* ns_dev) {
  D3F_REQUIRE(Nq >= 0 && Ns >= 0 && H >= 0 && Hr >= 0 && Cin >= 1 && Cout >= 1, D3F_ERR_INVALID,
              "kpconv_backward: bad shape Nq=%d Ns=%d H=%d Hr=%d Cin=%d Cout=%d", Nq, Ns, H, Hr, Cin, Cout);
  D3F_REQUIRE(K >= 1 && K <= 64, D3F_ERR_INVALID, "kpconv_backward: num_kernel_points=%d outside [1, 64]", K);
  D3F_REQUIRE(influence >= 0 && influence <= 2, D3F_ERR_INVALID,
              "Unknown influence function type (config.KP_influence)");
  D3F_REQUIRE(mode == D3F_MODE_SUM || mode == D3F_MODE_CLOSEST, D3F_ERR_INVALID,
              "Unknown convolution mode. Should be 'closest' or 'sum'");
  D3F_REQUIRE(extent > 0.f, D3F_ERR_INVALID, "kpconv_backward: KP_extent=%g", (double)extent);
  D3F_REQUIRE((long long)Nq * H < (1ll << 31), D3F_ERR_INVALID, "kpconv_backward: Nq*H=%lld beyond int32",
              (long long)Nq * H);
  const BackwardLayout L = backward_layout(Nq, Ns, H, K, Cin, Cout, Hr);
  D3F_REQUIRE(workspace_bytes >= L.total, D3F_ERR_WORKSPACE, "kpconv_backward: workspace too small");
  if (dfeat != nullptr && Ns > 0) D3F_CUDA(cudaMemsetAsync(dfeat, 0, (size_t)Ns * Cin * sizeof(float), stream));
  if (dW != nullptr) D3F_CUDA(cudaMemsetAsync(dW, 0, (size_t)K * Cin * Cout * sizeof(float), stream));
  if (Nq == 0 || Ns == 0 || (dfeat == nullptr && dW == nullptr)) return D3F_OK;

  char* ws = static_cast<char*>(workspace);
  char* reg = ws + L.region;
  float4* s4 = reinterpret_cast<float4*>(ws + L.s4);
  float* G = reinterpret_cast<float*>(ws + L.G);
  int rc = kpconv_prep_supports(false, s, feat, Ns, ns_dev, K, Cin, normalize, s4, stream);
  if (rc) return rc;
  grad_rowscale_kernel<<<ceil_div(Nq * 32, 256), 256, 0, stream>>>(dout, idx, s4, Nq, Ns, H, Cout, normalize != 0,
                                                                     nq_dev, ns_dev, G);
  D3F_LAUNCH_CHECK("grad_rowscale_kernel");

  if (dfeat != nullptr && Hr > 0 && H > 0) {
    int* counts = reinterpret_cast<int*>(reg + L.counts);
    int* offs = reinterpret_cast<int*>(reg + L.offs);
    int* rev = reinterpret_cast<int*>(ws + L.rev);
    SortBuffers sb;
    sb.keys[0] = reinterpret_cast<uint64_t*>(reg + L.keys0);
    sb.keys[1] = reinterpret_cast<uint64_t*>(reg + L.keys1);
    sb.vals[0] = reinterpret_cast<uint32_t*>(reg + L.vals0);
    sb.vals[1] = reinterpret_cast<uint32_t*>(reg + L.vals1);
    sb.block_hist = reinterpret_cast<int*>(reg + L.hist);
    const uint32_t* sorted_q = nullptr;
    rc = reverse_csr(idx, Nq, Ns, H, nq_dev, ns_dev, sb, counts, offs, reinterpret_cast<int*>(reg + L.scan), &sorted_q,
                     stream);
    if (rc) return rc;
    reverse_fill_kernel<<<grid_for((long long)Ns * Hr), 256, 0, stream>>>(counts, offs, sorted_q, Ns, Hr, Nq, rev);
    D3F_LAUNCH_CHECK("reverse_fill_kernel");
    // W^T [K, Cout, Cin] (packed for the tensor-core contraction), -Kp
    float* WT = reinterpret_cast<float*>(ws + L.WT);
    float* nKp = reinterpret_cast<float*>(ws + L.nKp);
    transpose_weights_kernel<<<grid_for((long long)K * Cin * Cout), 256, 0, stream>>>(W, K, Cin, Cout, WT);
    D3F_LAUNCH_CHECK("transpose_weights_kernel");
    negate_kernel<<<1, 256, 0, stream>>>(Kp, K * 3, nKp);
    D3F_LAUNCH_CHECK("negate_kernel");
    float* WTp = nullptr;
    if (tensor_cores) {
      WTp = reinterpret_cast<float*>(ws + L.WTp);
      rc = tc_pack_weight(WT, K * Cout, Cin, WTp, stream);
      if (rc) return rc;
    }
    rc = kpconv_forward_impl(false, s, q, rev, G, nKp, nullptr, nullptr, WT, WTp, nullptr, Ns, Nq, Hr, K, Cout, Cin,
                             extent, influence, mode, 0, nullptr, nullptr, nullptr, -1.f, dfeat, reg, L.fwd_bytes,
                             stream, ns_dev, nq_dev);
    if (rc) return rc;
  }

  if (dW != nullptr) {
    float* wf = reinterpret_cast<float*>(reg + L.wf);
    float* partial = reinterpret_cast<float*>(reg + L.partial);
    const int M = K * Cin;
    for (int ci = 0, n0 = 0; n0 < Nq; n0 += L.chunk, ++ci) {
      const int n1 = min(Nq, n0 + L.chunk);
      rc = kpconv_stage1_wf(q, s4, idx, feat, Kp, Nq, Ns, H, K, Cin, extent, influence, mode, n0, n1, wf, stream,
                            nq_dev, ns_dev);
      if (rc) return rc;
      rc = launch_wgrad_partial(wf, G + (size_t)n0 * Cout, n1 - n0, M, Cout, nq_dev, n0, L.bpc,
                                partial + (size_t)ci * L.bpc * M * Cout, stream);
      if (rc) return rc;
    }
    rc = launch_wgrad_reduce(partial, L.n_chunks * L.bpc, (long long)M * Cout, dW, stream);
    if (rc) return rc;
  }
  return D3F_OK;
}

// ---- unary ----------------------------------------------------------------------------------------------------------
size_t unary_backward_workspace_bytes(int N, int Cin, int Cout) {
  if (N < 0 || Cin < 1 || Cout < 1) return 0;
  size_t b = align_up((size_t)Cin * Cout * sizeof(float), 256);
  b += align_up(tc_packed_floats(Cout, Cin) * sizeof(float), 256);
  b += align_up((size_t)wgrad_blocks(N) * Cin * Cout * sizeof(float), 256);
  return b + 1024;
}

int unary_backward(const float* x, const float* W, const float* dout, int N, int Cin, int Cout, int tensor_cores,
                   float* dx, float* dW, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                   const int* n_dev) {
  D3F_REQUIRE(N >= 0 && Cin >= 1 && Cout >= 1, D3F_ERR_INVALID, "unary_backward: bad shape N=%d Cin=%d Cout=%d", N,
              Cin, Cout);
  D3F_REQUIRE(workspace_bytes >= unary_backward_workspace_bytes(N, Cin, Cout), D3F_ERR_WORKSPACE,
              "unary_backward: workspace too small");
  if (dx != nullptr && N > 0) D3F_CUDA(cudaMemsetAsync(dx, 0, (size_t)N * Cin * sizeof(float), stream));
  if (dW != nullptr) D3F_CUDA(cudaMemsetAsync(dW, 0, (size_t)Cin * Cout * sizeof(float), stream));
  if (N == 0) return D3F_OK;
  Carver cv(workspace, workspace_bytes);
  float* WT = cv.take<float>((size_t)Cin * Cout);
  float* WTp = cv.take<float>(tc_packed_floats(Cout, Cin));
  float* partial = cv.take<float>((size_t)wgrad_blocks(N) * Cin * Cout);
  int rc;
  if (dx != nullptr) {   // dx = dout @ W^T through the forward GEMM
    transpose_weights_kernel<<<grid_for((long long)Cin * Cout), 256, 0, stream>>>(W, 1, Cin, Cout, WT);
    D3F_LAUNCH_CHECK("transpose_weights_kernel");
    Epilogue ep;
    ep.rowscale = nullptr;
    ep.bn_scale = nullptr;
    ep.bn_shift = nullptr;
    ep.bias = nullptr;
    ep.residual = nullptr;
    ep.leaky_alpha = -1.f;
    ep.row_map = nullptr;
    ep.m_dev = n_dev;
    if (tensor_cores && tc_gemm_supported(dout, Cout)) {
      rc = tc_pack_weight(WT, Cout, Cin, WTp, stream);
      if (rc) return rc;
      rc = tc_gemm(dout, WTp, dx, N, Cin, Cout, ep, stream);
    } else {
      rc = gemm_f32(dout, WT, dx, N, Cin, Cout, ep, stream);
    }
    if (rc) return rc;
  }
  if (dW != nullptr) {
    const int nblk = wgrad_blocks(N);
    rc = launch_wgrad_partial(x, dout, N, Cin, Cout, n_dev, 0, nblk, partial, stream);
    if (rc) return rc;
    rc = launch_wgrad_reduce(partial, nblk, (long long)Cin * Cout, dW, stream);
    if (rc) return rc;
  }
  return D3F_OK;
}

}  // namespace d3f

// fp32 GEMM with the fused block epilogue (CUDA-core FFMA path).
//   C[M,N] = epilogue( rowscale[m] * (A[M,K] @ B[K,N]) )
//   epilogue: * bn_scale[n] + bn_shift[n]  ->  + bias[n]  ->  + residual[m,n]  ->  LeakyReLU(alpha)
// Used by the unary convolutions (kernels/convolution_ops.py:90-99 + models/network_blocks.py:149-165,
// 185-186, 343-368) and by the second stage of KPConv (sum_k wf_k @ W_k == [Nq, K*Cin] @ [K*Cin, Cout]).
#include "ops.cuh"

namespace d3f {


template <int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
gemm_f32_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C, int Mcap, int N, int K,
                Epilogue ep) {
  const int M = ep.m_dev ? min(Mcap, max(__ldg(ep.m_dev) - ep.m_off, 0)) : Mcap;
  if ((int)blockIdx.y * BM >= M) return;   // CTA-uniform: tiles beyond the actual row count
  constexpr int THREADS = (BM / TM) * (BN / TN);
  __shared__ float As[2][BK][BM + 4];
  __shared__ float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const bool a_vec = (K % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  const bool b_vec = (N % 4 == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  constexpr int A_VECS = BM * BK / 4, B_VECS = BK * BN / 4;
  constexpr int A_PER = (A_VECS + THREADS - 1) / THREADS, B_PER = (B_VECS + THREADS - 1) / THREADS;
  float4 a_reg[A_PER], b_reg[B_PER];

  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int r = 0; r < A_PER; ++r) {
      int v = tid + r * THREADS;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (v < A_VECS) {
        int row = v / (BK / 4), kq = (v % (BK / 4)) * 4;
        int gm = m0 + row, gk = k0 + kq;
        if (gm < M) {
          const float* p = A + (size_t)gm * K + gk;
          if (a_vec && gk + 3 < K) {
            x = *reinterpret_cast<const float4*>(p);
          } else {
            if (gk < K) x.x = p[0];
            if (gk + 1 < K) x.y = p[1];
            if (gk + 2 < K) x.z = p[2];
            if (gk + 3 < K) x.w = p[3];
          }
        }
      }
      a_reg[r] = x;
    }
#pragma unroll
    for (int r = 0; r < B_PER; ++r) {
      int v = tid + r * THREADS;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (v < B_VECS) {
        int row = v / (BN / 4), nq = (v % (BN / 4)) * 4;
        int gk = k0 + row, gn = n0 + nq;
        if (gk < K) {
          const float* p = B + (size_t)gk * N + gn;
          if (b_vec && gn + 3 < N) {
            x = *reinterpret_cast<const float4*>(p);
          } else {
            if (gn < N) x.x = p[0];
            if (gn + 1 < N) x.y = p[1];
            if (gn + 2 < N) x.z = p[2];
            if (gn + 3 < N) x.w = p[3];
          }
        }
      }
      b_reg[r] = x;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int r = 0; r < A_PER; ++r) {
      int v = tid + r * THREADS;
      if (v < A_VECS) {
        int row = v / (BK / 4), kq = (v % (BK / 4)) * 4;
        As[buf][kq + 0][row] = a_reg[r].x;
        As[buf][kq + 1][row] = a_reg[r].y;
        As[buf][kq + 2][row] = a_reg[r].z;
        As[buf][kq + 3][row] = a_reg[r].w;
      }
    }
#pragma unroll
    for (int r = 0; r < B_PER; ++r) {
      int v = tid + r * THREADS;
      if (v < B_VECS) {
        int row = v / (BN / 4), nq = (v % (BN / 4)) * 4;
        *reinterpret_cast<float4*>(&Bs[buf][row][nq]) = b_reg[r];
      }
    }
  };

  const int nk = (K + BK - 1) / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 t = *reinterpret_cast<const float4*>(&As[buf][kk][ty * TM + i]);
        a[i] = t.x; a[i + 1] = t.y; a[i + 2] = t.z; a[i + 3] = t.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        float4 t = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * TN + j]);
        b[j] = t.x; b[j + 1] = t.y; b[j + 2] = t.z; b[j + 3] = t.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int gm = m0 + ty * TM + i;
    if (gm >= M) continue;
    float rs = ep.rowscale ? ep.rowscale[gm] : 1.f;
    const size_t orow = ep.row_map ? (size_t)ep.row_map[gm] : (size_t)gm;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int gn = n0 + tx * TN + j;
      if (gn >= N) continue;
      float y = acc[i][j] * rs;
      if (ep.bn_scale) y = fmaf(y, ep.bn_scale[gn], ep.bn_shift[gn]);
      if (ep.bias) y += ep.bias[gn];
      if (ep.residual) y += ep.residual[orow * N + gn];
      if (ep.leaky_alpha >= 0.f) y = y > 0.f ? y : y * ep.leaky_alpha;
      C[orow * N + gn] = y;
    }
  }
}

int gemm_f32(const float* A, const float* B, float* C, int M, int N, int K, const Epilogue& ep, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return D3F_OK;
  D3F_REQUIRE(K > 0, D3F_ERR_INVALID, "gemm: K=%d", K);
  // small-M (deep pyramid levels) use 64-row tiles so that more CTAs are in flight
  long long ctas128 = (long long)ceil_div(M, 128) * ceil_div(N, 128);
  if (ctas128 >= 2 * kNumSMs && N >= 128) {
    dim3 grid(ceil_div(N, 128), ceil_div(M, 128));
    gemm_f32_kernel<128, 128, 8, 8, 8><<<grid, 256, 0, stream>>>(A, B, C, M, N, K, ep);
  } else if (N >= 64) {
    dim3 grid(ceil_div(N, 64), ceil_div(M, 64));
    gemm_f32_kernel<64, 64, 16, 4, 4><<<grid, 256, 0, stream>>>(A, B, C, M, N, K, ep);
  } else {
    dim3 grid(ceil_div(N, 32), ceil_div(M, 128));
    gemm_f32_kernel<128, 32, 16, 4, 4><<<grid, 256, 0, stream>>>(A, B, C, M, N, K, ep);
  }
  D3F_LAUNCH_CHECK("gemm_f32_kernel");
  return D3F_OK;
}

}  // namespace d3f

using namespace d3f;

extern "C" int d3f_unary_forward(const float* x, const float* W, const float* W_packed, int N, int Cin, int Cout,
                                 const float* bn_scale, const float* bn_shift, const float* bias, const float* residual,
                                 float leaky_alpha, float* out, d3f_stream_t stream, const int* n_dev) {
  D3F_REQUIRE(N >= 0 && Cin >= 1 && Cout >= 1, D3F_ERR_INVALID, "d3f_unary_forward: bad shape N=%d Cin=%d Cout=%d", N,
              Cin, Cout);
  D3F_REQUIRE(N == 0 || (x && W && out), D3F_ERR_INVALID, "d3f_unary_forward: null pointer");
  D3F_REQUIRE((bn_scale == nullptr) == (bn_shift == nullptr), D3F_ERR_INVALID,
              "d3f_unary_forward: bn_scale/bn_shift mismatch");
  Epilogue ep;
  ep.rowscale = nullptr;
  ep.bn_scale = bn_scale;
  ep.bn_shift = bn_shift;
  ep.bias = bias;
  ep.residual = residual;
  ep.leaky_alpha = leaky_alpha;
  ep.row_map = nullptr;
  ep.m_dev = n_dev;
  if (W_packed != nullptr && tc_gemm_supported(x, Cin))
    return tc_gemm(x, W_packed, out, N, Cout, Cin, ep, (cudaStream_t)stream);
  return gemm_f32(x, W, out, N, Cout, Cin, ep, (cudaStream_t)stream);
}

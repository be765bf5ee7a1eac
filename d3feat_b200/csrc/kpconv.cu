// KPConv forward (kernels/convolution_ops.py:161-255 rigid, :379-499 deformable).
//
// Stage 1 (this file): one warp per query point gathers the neighbour feature rows, evaluates the kernel-point
// correlation weights w[h,k] and accumulates
//        wf[n,k,:] = sum_h w[n,h,k] * feat[idx[n,h],:]            (:240 / :486)
// Kernels, most specialised first (launch_stage1 picks):
//   kpconv_stage1_fast_kernel<NT>    K = 15, rigid, linear influence, sum aggregation (every D3Feat model): weights in
//                                    mma.sync A-fragment layout, rows loaded in B-fragment layout, 3xTF32 on the tensor
//                                    pipe, nothing in shared memory; wide layers as 64-channel passes over gridDim.y
//   kpconv_stage1_staged_kernel<NT>  the same with the gathers staged through shared memory (opt-in, same bits)
//   kpconv_stage1_mma_kernel<...>    the general mma.sync kernel: deformable, gaussian / constant influence, closest mode
//   kpconv_cin1_kernel<FAST>         first layer (Cin = 1), whole operator in one kernel
//   kpconv_stage1_anyk_kernel, _v2_kernel, _kernel   CUDA-core paths: any number of kernel points, odd widths
// Stage 2 is the dense contraction  out[n,:] = (sum_k wf[n,k,:] @ W[k]) / nn[n]  ==  [Nq, K*Cin] @ [K*Cin, Cout] on
// wgmma with the block epilogue fused (tc_gemm.cu; gemm.cu without tensor cores). The [N,H,K,3], [N,H,K], [N,H,Cin]
// intermediates of the TF graph are never materialised; wf is one buffer per layer (chunks beyond 512 MB).
// kpconv_fused.cu holds the single persistent kernel (stage 1 + contraction) for the Cin = Cout = 32 layers (opt-in).
#include <stdlib.h>

#include "ops.cuh"

namespace d3f {


constexpr int kS1Warps = 4;      // queries per CTA
constexpr int kWStride = 20;     // floats per neighbour in the weight tile (16 B aligned, 4-way write conflicts)
constexpr int kKMax = 16;        // kernel points are padded to 16 in shared memory

struct Stage1Params {
  const float* q;
  const float4* s4;           // [Ns+1] supports as (x, y, z, flag): flag = 1 if the feature-row sum > 0
                              // (normalisation, :249-253); entry Ns is the shadow point (flag 0)
  const int* idx;
  const float* feat;
  int count_nn;               // accumulate the normalisation count
  const float* Kp;            // [K,3]
  const float* offsets;       // [Nq,K,3] or null (deformable)
  const float* modulations;   // [Nq,K] or null
  int Nq, Ns, H, Cin;
  int n0, n1;                 // query chunk [n0, n1) (slots; slot i is query order[i] when order != null)
  const int* order;           // optional visiting order of the queries (hash-grid cell order)
  float extent;               // KP_extent of this layer
  float inv_scale;            // 1/(2 extent) rigid (:215), 1/extent deformable (:461)
  float gauss_inv;            // 1/(2 sigma^2 + 1e-9), sigma = 0.3 extent (:218-222)
  int influence, closest;
  float shadow;               // coordinate of the shadow support point (1e6 / 1000)
  float* wf;                  // [n1-n0, K*Cin]
  float* inv_nn;              // [n1-n0] or null
  const int* nq_dev;          // optional: actual query / support counts in device memory (Nq / Ns are capacities)
  const int* ns_dev;
};

// One warp per support point: pack (x, y, z, flag) so that phase A needs ONE 16-byte load per neighbour instead of
// three scattered 4-byte loads plus a flag byte; entry Ns is the shadow point. mode 0: flag = 0, 1: flag = (row sum
// of the features > 0) (:250-251), 2: flag slot carries the scalar feature itself (Cin = 1 kernel).
__global__ void __launch_bounds__(256) prep_supports_kernel(const float* __restrict__ s, const float* __restrict__ feat,
                                                            int Ns_cap, const int* __restrict__ ns_dev, int Cin,
                                                            int mode, float shadow, float4* __restrict__ s4) {
  const int Ns = dyn_rows(Ns_cap, ns_dev);
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp > Ns) return;
  if (warp == Ns) {
    if (lane == 0) s4[Ns] = make_float4(shadow, shadow, shadow, 0.f);
    return;
  }
  float w = 0.f;
  if (mode == 1) {
    float sum = 0.f;
    for (int c = lane; c < Cin; c += 32) sum += feat[(size_t)warp * Cin + c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    w = sum > 0.f ? 1.f : 0.f;
  } else if (mode == 2) {
    w = feat[warp];
  }
  if (lane == 0) s4[warp] = make_float4(s[3 * (size_t)warp], s[3 * (size_t)warp + 1], s[3 * (size_t)warp + 2], w);
}

// mode 1 with Cin % 4 == 0: G lanes per support (G = 8 / 16 / 32 for Cin = 32 / 64 / >= 128) read the feature row as
// float4, so a warp packs 32 / G supports per pass instead of one.
template <int G>
__global__ void __launch_bounds__(256) prep_supports_vec_kernel(const float* __restrict__ s,
                                                                const float* __restrict__ feat, int Ns_cap,
                                                                const int* __restrict__ ns_dev, int Cin,
                                                                float shadow, float4* __restrict__ s4) {
  const int Ns = dyn_rows(Ns_cap, ns_dev);
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = t / G, gl = t % G;
  float sum = 0.f;
  if (row < Ns) {
    const float4* fr = reinterpret_cast<const float4*>(feat + (size_t)row * Cin);
    for (int c4 = gl; c4 < Cin / 4; c4 += G) {
      float4 v = fr[c4];
      sum += (v.x + v.y) + (v.z + v.w);
    }
  }
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (gl == 0) {
    if (row < Ns)
      s4[row] = make_float4(s[3 * (size_t)row], s[3 * (size_t)row + 1], s[3 * (size_t)row + 2], sum > 0.f ? 1.f : 0.f);
    else if (row == Ns)
      s4[Ns] = make_float4(shadow, shadow, shadow, 0.f);
  }
}

template <int K, int VEC, bool DEFORM>
__global__ void __launch_bounds__(kS1Warps * 32) kpconv_stage1_kernel(Stage1Params p) {
  const int Ns_ = dyn_rows(p.Ns, p.ns_dev), n1_ = min(p.n1, dyn_rows(p.Nq, p.nq_dev));
  static_assert(K <= kKMax, "K too large");
  __shared__ __align__(16) float wts[kS1Warps][32 * kWStride];
  __shared__ float kp_s[kS1Warps][kKMax * 3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = p.n0 + blockIdx.x * kS1Warps + warp;
  if (n >= n1_) return;  // warp-uniform
  const int qid = p.order ? p.order[n] : n;

  // kernel points of this query (rigid: shared by all queries; deformable: Kp + offsets[n])
  for (int t = lane; t < K * 3; t += 32) {
    float v = p.Kp[t];
    if (DEFORM) v += p.offsets[(size_t)qid * K * 3 + t];
    kp_s[warp][t] = v;
  }
  for (int t = K * 3 + lane; t < kKMax * 3; t += 32) kp_s[warp][t] = 0.f;
  const float qx = p.q[3 * (size_t)qid], qy = p.q[3 * (size_t)qid + 1], qz = p.q[3 * (size_t)qid + 2];
  const int* row = p.idx + (size_t)qid * p.H;
  const float ext2 = p.extent * p.extent;
  __syncwarp();

  int nn_count = 0;
  const int c_step = 32 * VEC;
  for (int c0 = 0; c0 < p.Cin; c0 += c_step) {
    float acc[K][VEC];
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[k][v] = 0.f;
    const int c = c0 + lane * VEC;
    const bool c_ok = c < p.Cin;

    for (int h0 = 0; h0 < p.H; h0 += 32) {
      // ---- phase A: lane <-> neighbour h0+lane: correlation weights to the K kernel points ------------
      const int h = h0 + lane;
      int id = (h < p.H) ? row[h] : Ns_;
      if (id < 0 || id > Ns_) id = Ns_;  // -1 padding of the non-batch op behaves like the shadow
      const bool real = id < Ns_;
      const float4 sp = __ldg(&p.s4[id]);   // entry Ns = shadow point
      const float rx = sp.x - qx, ry = sp.y - qy, rz = sp.z - qz;
      float w[kKMax];
      float dmin = 3.0e38f;
      int kmin = 0;
      bool in_range = false;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        float dx = rx - kp_s[warp][3 * k], dy = ry - kp_s[warp][3 * k + 1], dz = rz - kp_s[warp][3 * k + 2];
        float d2 = dx * dx + dy * dy + dz * dz;
        if (d2 < dmin) { dmin = d2; kmin = k; }
        in_range = in_range || (d2 < ext2);
        float wk;
        if (p.influence == D3F_INFLUENCE_LINEAR) wk = fmaxf(1.f - sqrtf(d2 + 1e-10f) * p.inv_scale, 0.f);
        else if (p.influence == D3F_INFLUENCE_GAUSSIAN) wk = expf(-d2 * p.gauss_inv);
        else wk = DEFORM ? (d2 < ext2 ? 1.f : 0.f) : 1.f;
        w[k] = wk;
      }
      if (p.closest) {
#pragma unroll
        for (int k = 0; k < K; ++k) w[k] = (k == kmin) ? w[k] : 0.f;
      }
      const bool keep = real && (!DEFORM || in_range);
#pragma unroll
      for (int k = 0; k < kKMax; ++k) wts[warp][lane * kWStride + k] = (keep && k < K) ? w[k] : 0.f;
      if (c0 == 0 && p.count_nn) nn_count += __popc(__ballot_sync(0xffffffffu, sp.w > 0.f));
      const unsigned keep_mask = __ballot_sync(0xffffffffu, keep);
      __syncwarp();

      // ---- phase B: accumulate the kept neighbours of this chunk -------------------------------------
      unsigned m = keep_mask;
      while (m) {
        // up to 4 neighbours per step: issue the row loads first (memory-level parallelism)
        int hh[4];
        float f[4][VEC];
        int cnt = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (m) {
            hh[u] = __ffs(m) - 1;
            m &= m - 1;
            ++cnt;
          } else {
            hh[u] = -1;
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (hh[u] >= 0) {
            int idh = __shfl_sync(0xffffffffu, id, hh[u]);
            const float* fp = p.feat + (size_t)idh * p.Cin + c;
            if (VEC == 4) {
              float4 t = c_ok ? *reinterpret_cast<const float4*>(fp) : make_float4(0.f, 0.f, 0.f, 0.f);
              f[u][0] = t.x; f[u][1 % VEC] = t.y; f[u][2 % VEC] = t.z; f[u][3 % VEC] = t.w;
            } else if (VEC == 2) {
              float2 t = c_ok ? *reinterpret_cast<const float2*>(fp) : make_float2(0.f, 0.f);
              f[u][0] = t.x; f[u][1 % VEC] = t.y;
            } else {
              f[u][0] = c_ok ? *fp : 0.f;
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (hh[u] >= 0) {
            const float4* wp = reinterpret_cast<const float4*>(&wts[warp][hh[u] * kWStride]);
            float wv[kKMax];
#pragma unroll
            for (int kq = 0; kq < (K + 3) / 4; ++kq) {
              float4 t = wp[kq];
              wv[4 * kq] = t.x; wv[4 * kq + 1] = t.y; wv[4 * kq + 2] = t.z; wv[4 * kq + 3] = t.w;
            }
#pragma unroll
            for (int k = 0; k < K; ++k)
#pragma unroll
              for (int v = 0; v < VEC; ++v) acc[k][v] = fmaf(wv[k], f[u][v], acc[k][v]);
          }
        }
        (void)cnt;
      }
      __syncwarp();
    }

    // ---- write wf[n, k, c0 + lane*VEC ..] (optionally modulated, :489-490) ----------------------------
    if (c_ok) {
      float* dst = p.wf + (size_t)(n - p.n0) * K * p.Cin + c;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        float mod = (DEFORM && p.modulations) ? p.modulations[(size_t)qid * K + k] : 1.f;
        if (VEC == 4) {
          *reinterpret_cast<float4*>(dst + (size_t)k * p.Cin) =
              make_float4(acc[k][0] * mod, acc[k][1 % VEC] * mod, acc[k][2 % VEC] * mod, acc[k][3 % VEC] * mod);
        } else if (VEC == 2) {
          *reinterpret_cast<float2*>(dst + (size_t)k * p.Cin) = make_float2(acc[k][0] * mod, acc[k][1 % VEC] * mod);
        } else {
          dst[(size_t)k * p.Cin] = acc[k][0] * mod;
        }
      }
    }
  }
  if (p.inv_nn != nullptr && lane == 0) p.inv_nn[n - p.n0] = 1.f / (float)max(nn_count, 1);
}

// ---------------------------------------------------------------------------------------------------
// Stage 1, paired-kernel-point version (the one the encoder's layers use): the K = 15 kernel points are padded to 16
// and handled as 8 PAIRS, so one ffma2 updates (wf[2j], wf[2j+1]) of a channel, fed by four broadcast LDS.128 that
// deliver the pairs already packed. For Cin = 32 a warp serves TWO queries (one per half-warp, 2 channels per lane) so
// that the weight reads and the row loads are amortised over both.
// sm_90 has no packed fp32 FMA: a pair is two FFMA with the same round-to-nearest result per element.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// MUFU.SQRT: one instruction instead of the ~10-instruction IEEE sequence (max error ~1 ulp; tolerance 1e-4). The
// .ftz form matters: without it ptxas wraps the MUFU in a denormal rescue (FSETP + FMUL 2^24 + FMUL 2^-12, four
// instructions per root); every argument here is d^2 + 1e-10 >= 1e-10, never subnormal.
__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

template <int CPL, int QPW, bool DEFORM>
__global__ void __launch_bounds__(kS1Warps * 32, CPL == 4 ? 4 : 6) kpconv_stage1_v2_kernel(Stage1Params p) {
  const int Ns_ = dyn_rows(p.Ns, p.ns_dev), n1_ = min(p.n1, dyn_rows(p.Nq, p.nq_dev));
  constexpr int K = 15, KP = 16;
  constexpr int LPQ = 32 / QPW;  // lanes (= neighbour slots per pass) per query
  static_assert(CPL == 2 || CPL == 4, "channels per lane");
  __shared__ __align__(16) float wts[kS1Warps][32 * kWStride];
  __shared__ float kp_s[kS1Warps][QPW][KP * 3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = lane / LPQ, sl = lane % LPQ;
  const int nfirst = p.n0 + (blockIdx.x * kS1Warps + warp) * QPW;
  if (nfirst >= n1_) return;  // warp-uniform
  const int n = nfirst + sub;
  const bool qvalid = n < n1_;
  const int nslot = qvalid ? n : nfirst;  // invalid half-warps shadow the first query (results discarded)
  const int nq = p.order ? p.order[nslot] : nslot;

  for (int t = sl; t < KP * 3; t += LPQ) {
    float v = t < K * 3 ? p.Kp[t] : 0.f;
    if (DEFORM && t < K * 3) v += p.offsets[(size_t)nq * K * 3 + t];
    kp_s[warp][sub][t] = v;
  }
  const float qx = p.q[3 * (size_t)nq], qy = p.q[3 * (size_t)nq + 1], qz = p.q[3 * (size_t)nq + 2];
  const int* row = p.idx + (size_t)nq * p.H;
  const float ext2 = p.extent * p.extent;
  const unsigned gshift = (unsigned)(sub * LPQ);
  const unsigned gmask = LPQ == 32 ? 0xffffffffu : ((1u << LPQ) - 1u);
  float* wq = &wts[warp][sub * LPQ * kWStride];
  __syncwarp();

  int nn_count = 0;
  constexpr int c_step = LPQ * CPL;
  for (int c0 = 0; c0 < p.Cin; c0 += c_step) {
    float2 acc[KP / 2][CPL];
#pragma unroll
    for (int j = 0; j < KP / 2; ++j)
#pragma unroll
      for (int v = 0; v < CPL; ++v) acc[j][v] = make_float2(0.f, 0.f);
    const int c = c0 + sl * CPL;   // Cin is a multiple of c_step for every instantiation dispatched here

    for (int h0 = 0; h0 < p.H; h0 += LPQ) {
      // ---- phase A: lane <-> neighbour h0+sl of this lane's query ---------------------------------------
      const int h = h0 + sl;
      int id = (h < p.H) ? row[h] : Ns_;
      if (id < 0 || id > Ns_) id = Ns_;
      const bool real = id < Ns_;
      const float4 sp = __ldg(&p.s4[id]);   // entry Ns = shadow point
      const float rx = sp.x - qx, ry = sp.y - qy, rz = sp.z - qz;
      float w[KP];
      float dmin = 3.0e38f;
      int kmin = 0;
      bool in_range = false;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        float dx = rx - kp_s[warp][sub][3 * k], dy = ry - kp_s[warp][sub][3 * k + 1], dz = rz - kp_s[warp][sub][3 * k + 2];
        float d2 = dx * dx + dy * dy + dz * dz;
        if (d2 < dmin) { dmin = d2; kmin = k; }
        in_range = in_range || (d2 < ext2);
        float wk;
        if (p.influence == D3F_INFLUENCE_LINEAR) wk = fmaxf(1.f - sqrt_approx(d2 + 1e-10f) * p.inv_scale, 0.f);
        else if (p.influence == D3F_INFLUENCE_GAUSSIAN) wk = __expf(-d2 * p.gauss_inv);
        else wk = DEFORM ? (d2 < ext2 ? 1.f : 0.f) : 1.f;
        w[k] = wk;
      }
      w[K] = 0.f;
      if (p.closest) {
#pragma unroll
        for (int k = 0; k < K; ++k) w[k] = (k == kmin) ? w[k] : 0.f;
      }
      const bool keep = real && qvalid && (!DEFORM || in_range);
#pragma unroll
      for (int kq = 0; kq < KP / 4; ++kq)
        *reinterpret_cast<float4*>(&wq[sl * kWStride + 4 * kq]) =
            keep ? make_float4(w[4 * kq], w[4 * kq + 1], w[4 * kq + 2], w[4 * kq + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (c0 == 0 && p.count_nn) nn_count += __popc((__ballot_sync(0xffffffffu, sp.w > 0.f) >> gshift) & gmask);
      unsigned m = (__ballot_sync(0xffffffffu, keep) >> gshift) & gmask;
      int cnt = __popc(m);
      if (QPW >= 2) cnt = max(cnt, __shfl_xor_sync(0xffffffffu, cnt, 16));
      if (QPW >= 4) cnt = max(cnt, __shfl_xor_sync(0xffffffffu, cnt, 8));
      __syncwarp();

      // ---- phase B: both half-warps walk their kept neighbours in lockstep, kUnroll per step: all row loads
      //      of a step are issued before the first FMA consumes one (memory-level parallelism) -------------
      constexpr int kUnroll = CPL == 4 ? 2 : 4;
      for (int it = 0; it < cnt; it += kUnroll) {
        int hh[kUnroll];
        float f[kUnroll][CPL];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const bool act = m != 0;
          hh[u] = act ? __ffs(m) - 1 : 0;
          m &= m - 1;
          const int idh = __shfl_sync(0xffffffffu, id, (int)gshift + hh[u]);
          const float* fp = p.feat + (size_t)idh * p.Cin + c;
          if (CPL == 4) {
            float4 t = act ? __ldg(reinterpret_cast<const float4*>(fp)) : make_float4(0.f, 0.f, 0.f, 0.f);
            f[u][0] = t.x; f[u][1] = t.y; f[u][2 % CPL] = t.z; f[u][3 % CPL] = t.w;
          } else {
            float2 t = act ? __ldg(reinterpret_cast<const float2*>(fp)) : make_float2(0.f, 0.f);
            f[u][0] = t.x; f[u][1] = t.y;
          }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          // an inactive slot reads slot 0's weights with f = 0: contributes nothing
          const float4* wp = reinterpret_cast<const float4*>(&wq[hh[u] * kWStride]);
          float2 wpair[KP / 2];
#pragma unroll
          for (int kq = 0; kq < KP / 4; ++kq) {
            float4 t = wp[kq];
            wpair[2 * kq] = make_float2(t.x, t.y);
            wpair[2 * kq + 1] = make_float2(t.z, t.w);
          }
#pragma unroll
          for (int v = 0; v < CPL; ++v) {
            const float2 fd = make_float2(f[u][v], f[u][v]);
#pragma unroll
            for (int j = 0; j < KP / 2; ++j) acc[j][v] = ffma2(wpair[j], fd, acc[j][v]);
          }
        }
      }
      __syncwarp();
    }

    // ---- write wf[n, k, c .. c+CPL) (optionally modulated, :489-490) ------------------------------------
    if (qvalid) {
      float* dst = p.wf + (size_t)(n - p.n0) * K * p.Cin + c;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const float mod = (DEFORM && p.modulations) ? p.modulations[(size_t)nq * K + k] : 1.f;
        float o[CPL];
#pragma unroll
        for (int v = 0; v < CPL; ++v) o[v] = ((k & 1) ? acc[k / 2][v].y : acc[k / 2][v].x) * mod;
        if (CPL == 4) *reinterpret_cast<float4*>(dst + (size_t)k * p.Cin) = make_float4(o[0], o[1], o[2 % CPL], o[3 % CPL]);
        else *reinterpret_cast<float2*>(dst + (size_t)k * p.Cin) = make_float2(o[0], o[1]);
      }
    }
  }
  if (p.inv_nn != nullptr && qvalid && sl == 0) p.inv_nn[n - p.n0] = 1.f / (float)max(nn_count, 1);
}

// ---------------------------------------------------------------------------------------------------
// Stage 1 on the tensor pipe (warp-level mma.sync.m16n8k8 TF32, 3xTF32 split: even three TF32 products per fp32 one
// run well above the CUDA-core fp32 rate). Per query and 8-neighbour step:
//     wf[16 kernel pts, channels] += W^T[16 x 8 neighbours] . F[8 neighbours x channels]
// * A (correlation weights) is computed DIRECTLY in fragment layout: lane (g = lane/4, t = lane%4) evaluates the
//   weights of neighbours {8s+t, 8s+t+4} against kernel points {g, g+8} -- they live in registers, no shared memory.
// * B (gathered features) is loaded DIRECTLY in fragment layout. Column j of n-tile n is mapped to channel NT*j + n,
//   so a lane's B elements over the NT n-tiles are NT consecutive floats of its neighbour's row: one 16-byte load
//   per 4 channels, four full 128-byte rows per warp instruction.
// * Accumulators: NT x 4 registers per lane = kernel points {g, g+8} x channels [2*NT*t, 2*NT*(t+1)).
__device__ __forceinline__ void mma_tf32(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void split3(float x, unsigned& hi, unsigned& lo) {
  hi = (__float_as_uint(x) + 0x1000u) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

// ---------------------------------------------------------------------------------------------------
// The same stage 1 with the instruction stream pared down for the configuration every D3Feat model runs (rigid, linear
// influence, sum aggregation). The general kernel is issue bound, and less than half of its instructions per
// 8-neighbour step are the correlation / split / MMA work. What is removed here:
//  * the shadow test on the weights: the rigid shadow point sits at 1e6 (:190), its linear influence is
//    max(1 - ~1e7, 0) = 0 on its own; the same trick parks the 16th (non-existent) kernel point of lanes g = 7 at 1e6;
//  * the ballot / popc chain of the neighbour count: every lane counts its own two neighbours, lanes 0-3 are reduced
//    with two shuffles at the end;
//  * the per-step re-derivation of the feature base pointer (ptxas rematerialised it from %tid every step: nine
//    instructions per row load) -- the pointer is made opaque and rows are addressed with one IMAD.WIDE;
//  * the epsilon add (folded into the first FMA of d^2), 64-bit index arithmetic (rows are addressed with 32-bit
//    element offsets; the host routes layers beyond 2^31 elements to the general kernel).
// (cvt.rna.tf32.f32 would be the natural split, but ptxas expands it to four instructions with an Inf/NaN guard; the
//  integer add-and-mask of split3 is two)

template <int NT>
__global__ void __launch_bounds__(kS1Warps * 32, NT == 4 ? 8 : (NT == 8 ? 5 : 3))
kpconv_stage1_fast_kernel(Stage1Params p) {
  const int Ns_ = dyn_rows(p.Ns, p.ns_dev), n1_ = min(p.n1, dyn_rows(p.Nq, p.nq_dev));
  constexpr int K = 15;
  static_assert(NT % 4 == 0, "one float4 per four n-tiles");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int n = p.n0 + blockIdx.x * kS1Warps + warp;
  if (n >= n1_) return;  // warp-uniform
  const int kA = g, kB = g + 8;
  const bool validB = kB < K;
  const float kax = p.Kp[3 * kA], kay = p.Kp[3 * kA + 1], kaz = p.Kp[3 * kA + 2];
  const float kbx = validB ? p.Kp[3 * kB] : 1e6f, kby = validB ? p.Kp[3 * kB + 1] : 1e6f,
              kbz = validB ? p.Kp[3 * kB + 2] : 1e6f;
  const int qid = p.order ? p.order[n] : n;
  const float qx = p.q[3 * (size_t)qid], qy = p.q[3 * (size_t)qid + 1], qz = p.q[3 * (size_t)qid + 2];
  const int* row = p.idx + (size_t)qid * p.H + t;
  const float inv_scale = p.inv_scale;
  const unsigned Ns = (unsigned)Ns_;
  const unsigned Cin = (unsigned)p.Cin;
  int cnt = 0;

  constexpr int CCH = NT * 8;   // channels per pass; wide layers on few queries spread the passes over gridDim.y
  for (int c0 = blockIdx.y * CCH; c0 < p.Cin; c0 += gridDim.y * CCH) {
    float acc[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const float* fcol = p.feat + c0 + NT * g;
    asm volatile("" : "+l"(fcol));   // opaque: keep the pointer in registers instead of re-deriving it every step

    // the indices of step h0 + 8 are fetched while step h0 computes: one dependent load per step, not two
    unsigned ida_n = Ns, idb_n = Ns;
    if (t < p.H) ida_n = (unsigned)__ldg(row);
    if (t + 4 < p.H) idb_n = (unsigned)__ldg(row + 4);
    for (int h0 = 0; h0 < p.H; h0 += 8) {
      const unsigned ida = min(ida_n, Ns);       // -1 padding of the non-batch op (0xffffffff) behaves like the shadow
      const unsigned idb = min(idb_n, Ns);
      ida_n = Ns;
      idb_n = Ns;
      if (h0 + 8 + t < p.H) ida_n = (unsigned)__ldg(row + h0 + 8);
      if (h0 + 12 + t < p.H) idb_n = (unsigned)__ldg(row + h0 + 12);
      const float4 spa = __ldg(&p.s4[ida]), spb = __ldg(&p.s4[idb]);
      float fa[NT], fb[NT];
#pragma unroll
      for (int v = 0; v < NT; v += 4) {
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f), y = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ida < Ns) x = __ldg(reinterpret_cast<const float4*>(fcol + (size_t)(ida * Cin) + v));
        if (idb < Ns) y = __ldg(reinterpret_cast<const float4*>(fcol + (size_t)(idb * Cin) + v));
        fa[v] = x.x; fa[v + 1] = x.y; fa[v + 2] = x.z; fa[v + 3] = x.w;
        fb[v] = y.x; fb[v + 1] = y.y; fb[v + 2] = y.z; fb[v + 3] = y.w;
      }
      if (c0 == 0) cnt += (spa.w > 0.f ? 1 : 0) + (spb.w > 0.f ? 1 : 0);
      const float rax = spa.x - qx, ray = spa.y - qy, raz = spa.z - qz;
      const float rbx = spb.x - qx, rby = spb.y - qy, rbz = spb.z - qz;
      auto weight = [&](float rx, float ry, float rz, float kx, float ky, float kz) {
        const float dx = rx - kx, dy = ry - ky, dz = rz - kz;
        const float d2 = fmaf(dz, dz, fmaf(dy, dy, fmaf(dx, dx, 1e-10f)));     // d^2 + 1e-10 (:215)
        return fmaxf(fmaf(-sqrt_approx(d2), inv_scale, 1.f), 0.f);             // 1 - d / (2 extent), clipped
      };
      unsigned ah[4], al[4];
      split3(weight(rax, ray, raz, kax, kay, kaz), ah[0], al[0]);
      split3(weight(rax, ray, raz, kbx, kby, kbz), ah[1], al[1]);
      split3(weight(rbx, rby, rbz, kax, kay, kaz), ah[2], al[2]);
      split3(weight(rbx, rby, rbz, kbx, kby, kbz), ah[3], al[3]);
#pragma unroll
      for (int i = 0; i < NT; ++i) {
        unsigned bh0, bl0, bh1, bl1;
        split3(fa[i], bh0, bl0);
        split3(fb[i], bh1, bl1);
        mma_tf32(acc[i], ah, bh0, bh1);
        mma_tf32(acc[i], al, bh0, bh1);
        mma_tf32(acc[i], ah, bl0, bl1);
      }
    }

    // ---- write wf: rows kA (acc[.][0..1]) and kB (acc[.][2..3]), channels c0 + 2*NT*t + [0, 2*NT) -------------
    float* dst = p.wf + (size_t)(n - p.n0) * K * p.Cin + c0 + 2 * NT * t;
#pragma unroll
    for (int v = 0; v < NT; v += 4) {
      *reinterpret_cast<float4*>(dst + (size_t)kA * p.Cin + v) = make_float4(acc[v][0], acc[v + 1][0], acc[v + 2][0], acc[v + 3][0]);
      *reinterpret_cast<float4*>(dst + (size_t)kA * p.Cin + NT + v) = make_float4(acc[v][1], acc[v + 1][1], acc[v + 2][1], acc[v + 3][1]);
      if (validB) {
        *reinterpret_cast<float4*>(dst + (size_t)kB * p.Cin + v) = make_float4(acc[v][2], acc[v + 1][2], acc[v + 2][2], acc[v + 3][2]);
        *reinterpret_cast<float4*>(dst + (size_t)kB * p.Cin + NT + v) = make_float4(acc[v][3], acc[v + 1][3], acc[v + 2][3], acc[v + 3][3]);
      }
    }
  }
  if (p.inv_nn != nullptr && blockIdx.y == 0) {
    // lanes 0-3 (g == 0) hold the counts of the neighbour slots t, t+4 (mod 8) of every step: together all of them
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 1);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 2);
    if (lane == 0) p.inv_nn[n - p.n0] = 1.f / (float)max(cnt, 1);
  }
}

// ---------------------------------------------------------------------------------------------------
// The pared kernel with the gathers STAGED through shared memory. The kernel above can be bound by the L1 data pipe
// (LSU wavefronts) -- a 128-bit warp load is served a
// quarter-warp at a time, one wavefront per cache line the quarter touches, and in the mma fragment layout
// (lane = 4 g + t, neighbour <-> t) every quarter holds four neighbours: 16 wavefronts per row load instead of 4, and
// the same for the packed points. Here the rows of a step arrive by cp.async in the COALESCED assignment (the 8 lanes
// of a quarter-warp copy the 128 contiguous bytes of one row: 4 wavefronts per instruction; the shadow row is a
// zero-fill), and the fragment lanes read them back with conflict-free 128-bit shared loads (XOR-swizzled chunks);
// lanes 0..7 fetch the step's 8 neighbour ids with one access and copy the 8 packed points. Per 8-neighbour step and
// 32-channel pass: ~35 wavefronts instead of ~70. Double-buffered per warp; no CTA-level synchronisation.
__device__ __forceinline__ uint32_t s1_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void s1_cp_async16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;   // src-size 0: the 16 destination bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ float4 s1_lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// swizzle of the 16-byte chunk index inside a 128-byte segment, by row & 3, such that the 8 (row, chunk) pairs a
// quarter-warp reads in fragment layout fall into 8 different bank groups
template <int NT>
__device__ __forceinline__ int s1_swz(int r3) {
  return NT == 4 ? 2 * r3 : (NT == 8 ? ((r3 & 1) | ((r3 & 2) << 1)) : r3);
}

template <int NT>
__global__ void __launch_bounds__(kS1Warps * 32, NT == 4 ? 8 : (NT == 8 ? 5 : 3))
kpconv_stage1_staged_kernel(Stage1Params p) {
  constexpr int K = 15;
  constexpr int ROWB = NT * 32;            // bytes of one row of a channel pass (NT * 8 channels)
  constexpr int BUFB = 8 * ROWB + 128;     // 8 rows + 8 packed points
  __shared__ __align__(128) unsigned char stage_sm[kS1Warps][2][BUFB];
  const int Ns_ = dyn_rows(p.Ns, p.ns_dev), n1_ = min(p.n1, dyn_rows(p.Nq, p.nq_dev));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int n = p.n0 + blockIdx.x * kS1Warps + warp;
  if (n >= n1_) return;  // warp-uniform
  const int kA = g, kB = g + 8;
  const bool validB = kB < K;
  const float kax = p.Kp[3 * kA], kay = p.Kp[3 * kA + 1], kaz = p.Kp[3 * kA + 2];
  const float kbx = validB ? p.Kp[3 * kB] : 1e6f, kby = validB ? p.Kp[3 * kB + 1] : 1e6f,
              kbz = validB ? p.Kp[3 * kB + 2] : 1e6f;
  const int qid = p.order ? p.order[n] : n;
  const float qx = p.q[3 * (size_t)qid], qy = p.q[3 * (size_t)qid + 1], qz = p.q[3 * (size_t)qid + 2];
  const int* rowq = p.idx + (size_t)qid * p.H;
  const float inv_scale = p.inv_scale;
  const unsigned Ns = (unsigned)Ns_;
  const unsigned Cin = (unsigned)p.Cin;
  const uint32_t base = s1_smem_u32(&stage_sm[warp][0][0]);
  const int cr = lane >> 3, cc = lane & 7;             // copy role: rows cr and cr + 4, chunk cc of every 128-byte segment
  // per-lane shared-memory offsets, computed once and pinned (ptxas otherwise re-derives them from %tid every step)
  uint32_t wr_row = (uint32_t)(cr * ROWB + (cc ^ s1_swz<NT>(cr & 3)) * 16);   // rows cr and cr + 4 share row & 3
  uint32_t wr_s4 = (uint32_t)(8 * ROWB + lane * 16);
  uint32_t rd_s4 = (uint32_t)(8 * ROWB + t * 16);
  uint32_t rd_row[NT / 4];                             // fragment role: rows t and t + 4, channels NT g + v ..
#pragma unroll
  for (int v = 0; v < NT; v += 4) {
    const int chunk = g * (NT / 4) + v / 4;
    rd_row[v / 4] = (uint32_t)(t * ROWB + (chunk & ~7) * 16 + (((chunk & 7) ^ s1_swz<NT>(t)) * 16));
    asm volatile("" : "+r"(rd_row[v / 4]));
  }
  asm volatile("" : "+r"(wr_row), "+r"(wr_s4), "+r"(rd_s4));
  int cnt = 0;

  constexpr int CCH = NT * 8;
  for (int c0 = blockIdx.y * CCH; c0 < p.Cin; c0 += gridDim.y * CCH) {
    float acc[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const float* fsrc = p.feat + c0 + 4 * cc;
    asm volatile("" : "+l"(fsrc));
    auto load_ids = [&](int h0) -> unsigned {
      unsigned v = Ns;                                   // slots beyond H and the -1 padding: the shadow
      if (lane < 8 && h0 + lane < p.H) v = (unsigned)__ldg(rowq + h0 + lane);
      return min(v, Ns);
    };
    auto issue = [&](unsigned idv, uint32_t buf) {
      if (lane < 8) s1_cp_async16(buf + wr_s4, p.s4 + idv, true);
      const unsigned i0 = __shfl_sync(0xffffffffu, idv, cr), i1 = __shfl_sync(0xffffffffu, idv, cr + 4);
      const bool ok0 = i0 < Ns, ok1 = i1 < Ns;
      const float* s0 = fsrc + (size_t)((ok0 ? i0 : 0u) * Cin);
      const float* s1 = fsrc + (size_t)((ok1 ? i1 : 0u) * Cin);
#pragma unroll
      for (int seg = 0; seg < ROWB / 128; ++seg) {
        s1_cp_async16(buf + wr_row + seg * 128, s0 + seg * 32, ok0);
        s1_cp_async16(buf + wr_row + 4 * ROWB + seg * 128, s1 + seg * 32, ok1);
      }
    };
    uint32_t cur = base, nxt = base + BUFB;
    unsigned idv_n = load_ids(0);
    issue(idv_n, cur);
    asm volatile("cp.async.commit_group;" ::: "memory");
    idv_n = load_ids(8);
    for (int h0 = 0; h0 < p.H; h0 += 8) {
      if (h0 + 8 < p.H) issue(idv_n, nxt);               // the rows of step h0 + 8 fly while step h0 computes
      asm volatile("cp.async.commit_group;" ::: "memory");
      idv_n = load_ids(h0 + 16);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
      __syncwarp();
      const float4 spa = s1_lds128(cur + rd_s4), spb = s1_lds128(cur + rd_s4 + 64);
      float fa[NT], fb[NT];
#pragma unroll
      for (int v = 0; v < NT; v += 4) {
        const float4 x = s1_lds128(cur + rd_row[v / 4]), y = s1_lds128(cur + rd_row[v / 4] + 4 * ROWB);
        fa[v] = x.x; fa[v + 1] = x.y; fa[v + 2] = x.z; fa[v + 3] = x.w;
        fb[v] = y.x; fb[v + 1] = y.y; fb[v + 2] = y.z; fb[v + 3] = y.w;
      }
      if (c0 == 0) cnt += (spa.w > 0.f ? 1 : 0) + (spb.w > 0.f ? 1 : 0);
      const float rax = spa.x - qx, ray = spa.y - qy, raz = spa.z - qz;
      const float rbx = spb.x - qx, rby = spb.y - qy, rbz = spb.z - qz;
      auto weight = [&](float rx, float ry, float rz, float kx, float ky, float kz) {
        const float dx = rx - kx, dy = ry - ky, dz = rz - kz;
        const float d2 = fmaf(dz, dz, fmaf(dy, dy, fmaf(dx, dx, 1e-10f)));     // d^2 + 1e-10 (:215)
        return fmaxf(fmaf(-sqrt_approx(d2), inv_scale, 1.f), 0.f);             // 1 - d / (2 extent), clipped
      };
      unsigned ah[4], al[4];
      split3(weight(rax, ray, raz, kax, kay, kaz), ah[0], al[0]);
      split3(weight(rax, ray, raz, kbx, kby, kbz), ah[1], al[1]);
      split3(weight(rbx, rby, rbz, kax, kay, kaz), ah[2], al[2]);
      split3(weight(rbx, rby, rbz, kbx, kby, kbz), ah[3], al[3]);
#pragma unroll
      for (int i = 0; i < NT; ++i) {
        unsigned bh0, bl0, bh1, bl1;
        split3(fa[i], bh0, bl0);
        split3(fb[i], bh1, bl1);
        mma_tf32(acc[i], ah, bh0, bh1);
        mma_tf32(acc[i], al, bh0, bh1);
        mma_tf32(acc[i], ah, bl0, bl1);
      }
      __syncwarp();   // every lane is done with the buffer before the next iteration's copies overwrite it
      const uint32_t tmp = cur;
      cur = nxt;
      nxt = tmp;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");

    float* dst = p.wf + (size_t)(n - p.n0) * K * p.Cin + c0 + 2 * NT * t;
#pragma unroll
    for (int v = 0; v < NT; v += 4) {
      *reinterpret_cast<float4*>(dst + (size_t)kA * p.Cin + v) = make_float4(acc[v][0], acc[v + 1][0], acc[v + 2][0], acc[v + 3][0]);
      *reinterpret_cast<float4*>(dst + (size_t)kA * p.Cin + NT + v) = make_float4(acc[v][1], acc[v + 1][1], acc[v + 2][1], acc[v + 3][1]);
      if (validB) {
        *reinterpret_cast<float4*>(dst + (size_t)kB * p.Cin + v) = make_float4(acc[v][2], acc[v + 1][2], acc[v + 2][2], acc[v + 3][2]);
        *reinterpret_cast<float4*>(dst + (size_t)kB * p.Cin + NT + v) = make_float4(acc[v][3], acc[v + 1][3], acc[v + 2][3], acc[v + 3][3]);
      }
    }
  }
  if (p.inv_nn != nullptr && blockIdx.y == 0) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 1);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, 2);
    if (lane == 0) p.inv_nn[n - p.n0] = 1.f / (float)max(cnt, 1);
  }
}

// FAST = the D3Feat configuration (KP_influence = linear, aggregation = sum) resolved at compile time; the
// generic instantiation keeps the runtime switches for constant / gaussian / closest.
template <int NT, bool DEFORM, bool FAST>
__global__ void __launch_bounds__(kS1Warps * 32) kpconv_stage1_mma_kernel(Stage1Params p) {
  const int Ns_ = dyn_rows(p.Ns, p.ns_dev), n1_ = min(p.n1, dyn_rows(p.Nq, p.nq_dev));
  constexpr int K = 15;
  static_assert(NT % 4 == 0, "one float4 per four n-tiles");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int n = p.n0 + blockIdx.x * kS1Warps + warp;
  if (n >= n1_) return;  // warp-uniform
  const int qid = p.order ? p.order[n] : n;
  // this lane's two kernel points (rigid: shared by all queries; deformable: Kp + offsets[query])
  const int kA = g, kB = g + 8;
  const bool validB = kB < K;
  float kax = p.Kp[3 * kA], kay = p.Kp[3 * kA + 1], kaz = p.Kp[3 * kA + 2];
  float kbx = validB ? p.Kp[3 * kB] : 0.f, kby = validB ? p.Kp[3 * kB + 1] : 0.f, kbz = validB ? p.Kp[3 * kB + 2] : 0.f;
  if (DEFORM) {
    const float* off = p.offsets + (size_t)qid * K * 3;
    kax += off[3 * kA]; kay += off[3 * kA + 1]; kaz += off[3 * kA + 2];
    if (validB) { kbx += off[3 * kB]; kby += off[3 * kB + 1]; kbz += off[3 * kB + 2]; }
  }
  const float qx = p.q[3 * (size_t)qid], qy = p.q[3 * (size_t)qid + 1], qz = p.q[3 * (size_t)qid + 2];
  const int* row = p.idx + (size_t)qid * p.H;
  const float ext2 = p.extent * p.extent;
  const unsigned tmask = 0x11111111u << t;   // the 8 lanes that hold the same neighbours as this lane
  int nn_count = 0;

  auto weight = [&](float d2) -> float {
    if (FAST || p.influence == D3F_INFLUENCE_LINEAR) return fmaxf(1.f - sqrt_approx(d2 + 1e-10f) * p.inv_scale, 0.f);
    if (p.influence == D3F_INFLUENCE_GAUSSIAN) return __expf(-d2 * p.gauss_inv);
    return DEFORM ? (d2 < ext2 ? 1.f : 0.f) : 1.f;
  };

  constexpr int CCH = NT * 8;   // channels per pass
  for (int c0 = 0; c0 < p.Cin; c0 += CCH) {
    float acc[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    // row base as an opaque byte pointer and row offsets as one unsigned 32 x 32 -> 64 multiply-add: ptxas otherwise
    // re-derives the pointer from %tid and rebuilds the 64-bit address with five instructions per row load
    const char* fcol = reinterpret_cast<const char*>(p.feat + c0 + NT * g);
    asm volatile("" : "+l"(fcol));
    const unsigned cin_bytes = (unsigned)p.Cin * 4u;

    for (int h0 = 0; h0 < p.H; h0 += 8) {
      const int ha = h0 + t, hb = h0 + t + 4;
      unsigned ida = ha < p.H ? (unsigned)row[ha] : (unsigned)Ns_, idb = hb < p.H ? (unsigned)row[hb] : (unsigned)Ns_;
      ida = min(ida, (unsigned)Ns_);        // -1 padding (0xffffffff) and out-of-range ids: the shadow entry
      idb = min(idb, (unsigned)Ns_);
      const float4 spa = __ldg(&p.s4[ida]), spb = __ldg(&p.s4[idb]);
      const bool reala = ida < (unsigned)Ns_, realb = idb < (unsigned)Ns_;
      // feature rows in fragment layout (issued before the weight math: latency overlaps it). A register-
      // pipelined variant (rows one step ahead) was measured SLOWER: occupancy (63 vs 93 regs) matters more.
      float fa[NT], fb[NT];
#pragma unroll
      for (int v = 0; v < NT; v += 4) {
        float4 x = reala ? __ldg(reinterpret_cast<const float4*>(fcol + (size_t)ida * cin_bytes + 4 * v)) : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 y = realb ? __ldg(reinterpret_cast<const float4*>(fcol + (size_t)idb * cin_bytes + 4 * v)) : make_float4(0.f, 0.f, 0.f, 0.f);
        fa[v] = x.x; fa[v + 1] = x.y; fa[v + 2] = x.z; fa[v + 3] = x.w;
        fb[v] = y.x; fb[v + 1] = y.y; fb[v + 2] = y.z; fb[v + 3] = y.w;
      }
      // squared distances to this lane's two kernel points
      const float rax = spa.x - qx, ray = spa.y - qy, raz = spa.z - qz;
      const float rbx = spb.x - qx, rby = spb.y - qy, rbz = spb.z - qz;
      float d_aA = (rax - kax) * (rax - kax) + (ray - kay) * (ray - kay) + (raz - kaz) * (raz - kaz);
      float d_aB = (rax - kbx) * (rax - kbx) + (ray - kby) * (ray - kby) + (raz - kbz) * (raz - kbz);
      float d_bA = (rbx - kax) * (rbx - kax) + (rby - kay) * (rby - kay) + (rbz - kaz) * (rbz - kaz);
      float d_bB = (rbx - kbx) * (rbx - kbx) + (rby - kby) * (rby - kby) + (rbz - kbz) * (rbz - kbz);
      float w_aA = weight(d_aA), w_aB = validB ? weight(d_aB) : 0.f;
      float w_bA = weight(d_bA), w_bB = validB ? weight(d_bB) : 0.f;
      if (!FAST && p.closest) {
        // arg-min over all 15 kernel points of each neighbour = reduction over the 8 lanes sharing t
        float ma = d_aA, mb = d_bA;
        int ia = kA, ib = kA;
        if (validB && d_aB < ma) { ma = d_aB; ia = kB; }
        if (validB && d_bB < mb) { mb = d_bB; ib = kB; }
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          float oa = __shfl_xor_sync(0xffffffffu, ma, o), ob = __shfl_xor_sync(0xffffffffu, mb, o);
          int ja = __shfl_xor_sync(0xffffffffu, ia, o), jb = __shfl_xor_sync(0xffffffffu, ib, o);
          if (oa < ma || (oa == ma && ja < ia)) { ma = oa; ia = ja; }
          if (ob < mb || (ob == mb && jb < ib)) { mb = ob; ib = jb; }
        }
        w_aA = ia == kA ? w_aA : 0.f; w_aB = ia == kB ? w_aB : 0.f;
        w_bA = ib == kA ? w_bA : 0.f; w_bB = ib == kB ? w_bB : 0.f;
      }
      bool keepa = reala, keepb = realb;
      if (DEFORM) {
        // a neighbour is kept if ANY deformed kernel point has it in range (:435-451)
        const unsigned ra = __ballot_sync(0xffffffffu, d_aA < ext2 || (validB && d_aB < ext2));
        const unsigned rb = __ballot_sync(0xffffffffu, d_bA < ext2 || (validB && d_bB < ext2));
        keepa = keepa && (ra & tmask) != 0;
        keepb = keepb && (rb & tmask) != 0;
      }
      if (!keepa) { w_aA = 0.f; w_aB = 0.f; }
      if (!keepb) { w_bA = 0.f; w_bB = 0.f; }
      if (c0 == 0 && p.count_nn) {
        // lanes 0..3 (g == 0) cover the eight neighbours of this step once
        nn_count += __popc(__ballot_sync(0xffffffffu, spa.w > 0.f) & 0xFu) + __popc(__ballot_sync(0xffffffffu, spb.w > 0.f) & 0xFu);
      }
      // A fragment: a0 = (kA, nb a), a1 = (kB, nb a), a2 = (kA, nb b), a3 = (kB, nb b); 3xTF32 split
      unsigned ah[4], al[4];
      split3(w_aA, ah[0], al[0]);
      split3(w_aB, ah[1], al[1]);
      split3(w_bA, ah[2], al[2]);
      split3(w_bB, ah[3], al[3]);
#pragma unroll
      for (int i = 0; i < NT; ++i) {
        unsigned bh0, bl0, bh1, bl1;
        split3(fa[i], bh0, bl0);
        split3(fb[i], bh1, bl1);
        mma_tf32(acc[i], ah, bh0, bh1);
        mma_tf32(acc[i], al, bh0, bh1);
        mma_tf32(acc[i], ah, bl0, bl1);
      }
    }

    // ---- write wf: rows kA (acc[.][0..1]) and kB (acc[.][2..3]), channels c0 + 2*NT*t + [0, 2*NT) -------------
    float* dst = p.wf + (size_t)(n - p.n0) * K * p.Cin + c0 + 2 * NT * t;
    const float modA = (DEFORM && p.modulations) ? p.modulations[(size_t)qid * K + kA] : 1.f;
    const float modB = (DEFORM && p.modulations && validB) ? p.modulations[(size_t)qid * K + kB] : 1.f;
#pragma unroll
    for (int v = 0; v < NT; v += 4) {
      *reinterpret_cast<float4*>(dst + (size_t)kA * p.Cin + v) =
          make_float4(acc[v][0] * modA, acc[v + 1][0] * modA, acc[v + 2][0] * modA, acc[v + 3][0] * modA);
      *reinterpret_cast<float4*>(dst + (size_t)kA * p.Cin + NT + v) =
          make_float4(acc[v][1] * modA, acc[v + 1][1] * modA, acc[v + 2][1] * modA, acc[v + 3][1] * modA);
      if (validB) {
        *reinterpret_cast<float4*>(dst + (size_t)kB * p.Cin + v) =
            make_float4(acc[v][2] * modB, acc[v + 1][2] * modB, acc[v + 2][2] * modB, acc[v + 3][2] * modB);
        *reinterpret_cast<float4*>(dst + (size_t)kB * p.Cin + NT + v) =
            make_float4(acc[v][3] * modB, acc[v + 1][3] * modB, acc[v + 2][3] * modB, acc[v + 3][3] * modB);
      }
    }
  }
  if (p.inv_nn != nullptr && lane == 0) p.inv_nn[n - p.n0] = 1.f / (float)max(nn_count, 1);
}

// ---------------------------------------------------------------------------------------------------
// Stage 1 for any number of kernel points (config.num_kernel_points, utils/config.py; D3Feat ships K = 15, for which the
// specialised kernels above exist). One warp per query; the correlation weights of a 32-neighbour chunk live in shared
// memory [k][neighbour], wf[n,k,:] is accumulated chunk by chunk in global memory (the chunk's rows are re-read per
// kernel point out of L1). Correctness path, not a tuned one.
constexpr int kAnyKMax = 64;

template <bool DEFORM>
__global__ void __launch_bounds__(kS1Warps * 32) kpconv_stage1_anyk_kernel(Stage1Params p, int K) {
  const int Ns_ = dyn_rows(p.Ns, p.ns_dev), n1_ = min(p.n1, dyn_rows(p.Nq, p.nq_dev));
  extern __shared__ float anyk_smem[];   // per warp: wts[K][32], kp[K][3]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* wts = anyk_smem + (size_t)warp * (K * 32 + K * 3);
  float* kp_s = wts + K * 32;
  const int n = p.n0 + blockIdx.x * kS1Warps + warp;
  if (n >= n1_) return;  // warp-uniform
  const int qid = p.order ? p.order[n] : n;
  for (int t = lane; t < K * 3; t += 32) {
    float v = p.Kp[t];
    if (DEFORM) v += p.offsets[(size_t)qid * K * 3 + t];
    kp_s[t] = v;
  }
  const float qx = p.q[3 * (size_t)qid], qy = p.q[3 * (size_t)qid + 1], qz = p.q[3 * (size_t)qid + 2];
  const int* row = p.idx + (size_t)qid * p.H;
  const float ext2 = p.extent * p.extent;
  float* dst = p.wf + (size_t)(n - p.n0) * K * p.Cin;
  __syncwarp();
  int nn_count = 0;
  for (int h0 = 0; h0 < p.H || h0 == 0; h0 += 32) {
    const int h = h0 + lane;
    int id = (h < p.H) ? row[h] : Ns_;
    if (id < 0 || id > Ns_) id = Ns_;
    const bool real = id < Ns_;
    const float4 sp = __ldg(&p.s4[id]);
    const float rx = sp.x - qx, ry = sp.y - qy, rz = sp.z - qz;
    float dmin = 3.0e38f;
    int kmin = 0;
    bool in_range = false;
    for (int k = 0; k < K; ++k) {
      float dx = rx - kp_s[3 * k], dy = ry - kp_s[3 * k + 1], dz = rz - kp_s[3 * k + 2];
      float d2 = dx * dx + dy * dy + dz * dz;
      if (d2 < dmin) { dmin = d2; kmin = k; }
      in_range = in_range || (d2 < ext2);
      float wk;
      if (p.influence == D3F_INFLUENCE_LINEAR) wk = fmaxf(1.f - sqrtf(d2 + 1e-10f) * p.inv_scale, 0.f);
      else if (p.influence == D3F_INFLUENCE_GAUSSIAN) wk = expf(-d2 * p.gauss_inv);
      else wk = DEFORM ? (d2 < ext2 ? 1.f : 0.f) : 1.f;
      wts[k * 32 + lane] = wk;
    }
    const bool keep = real && (!DEFORM || in_range);
    for (int k = 0; k < K; ++k) {
      float wk = wts[k * 32 + lane];
      if (p.closest && k != kmin) wk = 0.f;
      if (!keep) wk = 0.f;
      if (DEFORM && p.modulations) wk *= p.modulations[(size_t)qid * K + k];   // wf_k * mod_k (:489-490)
      wts[k * 32 + lane] = wk;
    }
    if (p.count_nn) nn_count += __popc(__ballot_sync(0xffffffffu, sp.w > 0.f));
    const unsigned keep_mask = __ballot_sync(0xffffffffu, keep);
    __syncwarp();
    for (int c0 = 0; c0 < p.Cin; c0 += 32) {   // every lane runs every iteration (full-mask shuffles inside)
      const int c = c0 + lane;
      const bool c_ok = c < p.Cin;
      for (int k = 0; k < K; ++k) {
        float acc = (h0 == 0 || !c_ok) ? 0.f : dst[(size_t)k * p.Cin + c];
        unsigned m = keep_mask;
        while (m) {
          const int j = __ffs(m) - 1;
          m &= m - 1;
          const int idj = __shfl_sync(0xffffffffu, id, j);
          if (c_ok) acc = fmaf(wts[k * 32 + j], p.feat[(size_t)idj * p.Cin + c], acc);
        }
        if (c_ok) dst[(size_t)k * p.Cin + c] = acc;
      }
    }
    __syncwarp();
  }
  if (p.inv_nn != nullptr && lane == 0) p.inv_nn[n - p.n0] = 1.f / (float)max(nn_count, 1);
}

template <bool DEFORM>
static int launch_stage1(int K, const Stage1Params& p, cudaStream_t stream) {
  int nq = p.n1 - p.n0;
  bool al16 = (reinterpret_cast<uintptr_t>(p.feat) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.wf) & 15) == 0;
  if (K == 15 && al16 && (p.Cin == 32 || p.Cin == 64 || p.Cin % 128 == 0)) {
    const int blocks = ceil_div(nq, kS1Warps);
    const bool fast = p.influence == D3F_INFLUENCE_LINEAR && !p.closest;
    static const bool no_pared = [] { const char* v = getenv("D3F_S1_PARED"); return v != nullptr && v[0] == '0'; }();
    if (fast && !DEFORM && !no_pared && (long long)(p.Ns + 1) * p.Cin < (1ll << 31)) {
      // Wide layers (Cin >= 128: levels 2-4, 15k queries and fewer) run as 64-channel passes spread over gridDim.y:
      // one warp per (query, pass). Measured against 128-channel passes (NT = 16: 153 registers, 12 warps per SM,
      // 26 % issue utilisation): 128->128 @ 15k 0.155 -> 0.143 ms, 256->256 @ 4k 0.125 -> 0.120, 512->512 @ 1.2k
      // 0.117 -> 0.112 -- the re-evaluated correlation weights cost less than the occupancy gains.
      const char* sv = getenv("D3F_S1_STAGED");          // read per call: tests switch it
      const int staged = sv ? atoi(sv) : 0;
      const dim3 grid_wide(blocks, p.Cin >= 128 ? p.Cin / 64 : 1);
      if (staged) {
        if (p.Cin == 32) kpconv_stage1_staged_kernel<4><<<blocks, kS1Warps * 32, 0, stream>>>(p);
        else kpconv_stage1_staged_kernel<8><<<grid_wide, kS1Warps * 32, 0, stream>>>(p);
        D3F_LAUNCH_CHECK("kpconv_stage1_staged_kernel");
        return D3F_OK;
      }
      // (32-channel passes for Cin = 64 were measured too: 0.271 vs 0.260 ms at 60k queries -- worse)
      if (p.Cin == 32) kpconv_stage1_fast_kernel<4><<<blocks, kS1Warps * 32, 0, stream>>>(p);
      else kpconv_stage1_fast_kernel<8><<<grid_wide, kS1Warps * 32, 0, stream>>>(p);
      D3F_LAUNCH_CHECK("kpconv_stage1_fast_kernel");
      return D3F_OK;
    }
    if (fast) {
      if (p.Cin == 32) kpconv_stage1_mma_kernel<4, DEFORM, true><<<blocks, kS1Warps * 32, 0, stream>>>(p);
      else if (p.Cin == 64) kpconv_stage1_mma_kernel<8, DEFORM, true><<<blocks, kS1Warps * 32, 0, stream>>>(p);
      else kpconv_stage1_mma_kernel<16, DEFORM, true><<<blocks, kS1Warps * 32, 0, stream>>>(p);
    } else {
      if (p.Cin == 32) kpconv_stage1_mma_kernel<4, DEFORM, false><<<blocks, kS1Warps * 32, 0, stream>>>(p);
      else if (p.Cin == 64) kpconv_stage1_mma_kernel<8, DEFORM, false><<<blocks, kS1Warps * 32, 0, stream>>>(p);
      else kpconv_stage1_mma_kernel<16, DEFORM, false><<<blocks, kS1Warps * 32, 0, stream>>>(p);
    }
    D3F_LAUNCH_CHECK("kpconv_stage1_mma_kernel");
    return D3F_OK;
  }
  // (channels per lane, queries per warp): every broadcast weight read should feed as much math as possible.
  // Cin % 128 == 0 never gets here (taken by the tensor-core kernels above), so CPL = 2 is the widest instance.
  if (K == 15 && al16 && p.Cin % 64 == 0) {
    kpconv_stage1_v2_kernel<2, 1, DEFORM><<<ceil_div(nq, kS1Warps), kS1Warps * 32, 0, stream>>>(p);
  } else if (K == 15 && al16 && p.Cin % 32 == 0) {
    kpconv_stage1_v2_kernel<2, 2, DEFORM><<<ceil_div(nq, kS1Warps * 2), kS1Warps * 32, 0, stream>>>(p);
  } else if (K == 15) {
    // generic K = 15 path (odd widths)
    kpconv_stage1_kernel<15, 1, DEFORM><<<ceil_div(nq, kS1Warps), kS1Warps * 32, 0, stream>>>(p);
  } else {
    const size_t smem = (size_t)kS1Warps * (K * 32 + K * 3) * sizeof(float);
    kpconv_stage1_anyk_kernel<DEFORM><<<ceil_div(nq, kS1Warps), kS1Warps * 32, smem, stream>>>(p, K);
  }
  D3F_LAUNCH_CHECK("kpconv_stage1_kernel");
  return D3F_OK;
}

// ---------------------------------------------------------------------------------------------------
// First layer of the network: Cin = 1 (constant-one input feature, datasets/ThreeDMatch.py:316). The whole
// KPConv of a query fits in one warp: lanes <-> neighbours for the correlation weights, a warp reduction gives
// wf[k] = sum_h w[h,k] f[h], then lanes <-> output channels for out[c] = (sum_k wf[k] W[k,0,c]) / nn + epilogue.
// One kernel, nothing but the output row is written.
struct Cin1Params {
  const float* q; const float4* s4; const int* idx; const float* Kp; const float* W;
  int Nq, Ns, H, Cout;
  float inv_scale, gauss_inv;
  int influence, closest, normalize;
  float shadow;
  const float* bn_scale; const float* bn_shift; const float* bias;
  float leaky_alpha;
  const int* order;
  float* out;
  const int* nq_dev; const int* ns_dev;
};

// 8 lanes per query (4 queries per warp): a lane walks neighbours sl, sl+8, ... and keeps the 15 partial sums
// wf[k] in registers; a 3-step shuffle reduction inside the 8-lane group finishes wf, then the group's lanes split the
// output channels with W[15, Cout] staged once per CTA in shared memory.
// FAST = linear influence, sum aggregation (every D3Feat model): the 45 kernel-point coordinates live in registers
// instead of 45 shared-memory loads per neighbour, no closest-point bookkeeping, the weight is two FMAs around the MUFU.
template <bool FAST>
__global__ void __launch_bounds__(256, 3) kpconv_cin1_kernel(Cin1Params p) {
  const int Ns_ = dyn_rows(p.Ns, p.ns_dev), Nq_ = dyn_rows(p.Nq, p.nq_dev);
  constexpr int K = 15;
  extern __shared__ float c1_smem[];   // W[K*Cout] then Kp[K*3]
  float* Ws = c1_smem;
  float* kp_s = c1_smem + K * p.Cout;
  for (int t = threadIdx.x; t < K * p.Cout; t += blockDim.x) Ws[t] = p.W[t];
  for (int t = threadIdx.x; t < K * 3; t += blockDim.x) kp_s[t] = p.Kp[t];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int sub = lane >> 3, sl = lane & 7;
  const int slot0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4;
  if (slot0 >= Nq_) return;  // warp-uniform
  const int slot = slot0 + sub;
  const bool qvalid = slot < Nq_;
  const int n = p.order ? p.order[qvalid ? slot : slot0] : (qvalid ? slot : slot0);
  const float qx = p.q[3 * (size_t)n], qy = p.q[3 * (size_t)n + 1], qz = p.q[3 * (size_t)n + 2];
  const int* row = p.idx + (size_t)n * p.H;
  float wf[K];
#pragma unroll
  for (int k = 0; k < K; ++k) wf[k] = 0.f;
  int nn = 0;
  if (FAST) {
    float kp[K * 3];
#pragma unroll
    for (int i = 0; i < K * 3; ++i) kp[i] = kp_s[i];
    const float inv_scale = p.inv_scale;
    // two-deep software pipeline over the lane's neighbours: index of h + 16 and point of h + 8 are in flight while
    // neighbour h is evaluated (-1 padding -> the shadow entry Ns, as for slots beyond H)
    const unsigned Nsu = (unsigned)Ns_;
    unsigned id1 = Nsu, id2 = Nsu;
    if (sl < p.H) id1 = min((unsigned)__ldg(row + sl), Nsu);
    if (sl + 8 < p.H) id2 = min((unsigned)__ldg(row + sl + 8), Nsu);
    float4 sp_n = __ldg(&p.s4[id1]);
    for (int h = sl; h < p.H; h += 8) {
      const float4 sp = sp_n;               // (x, y, z, feature); entry Ns = shadow point with feature 0
      sp_n = __ldg(&p.s4[id2]);
      id2 = Nsu;
      if (h + 16 < p.H) id2 = min((unsigned)__ldg(row + h + 16), Nsu);
      const float f = sp.w, rx = sp.x - qx, ry = sp.y - qy, rz = sp.z - qz;
      nn += f > 0.f ? 1 : 0;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const float dx = rx - kp[3 * k], dy = ry - kp[3 * k + 1], dz = rz - kp[3 * k + 2];
        const float d2 = fmaf(dz, dz, fmaf(dy, dy, fmaf(dx, dx, 1e-10f)));
        const float wk = fmaxf(fmaf(-sqrt_approx(d2), inv_scale, 1.f), 0.f);
        wf[k] = fmaf(wk, f, wf[k]);           // f = 0 for shadow neighbours
      }
    }
  } else
  for (int h = sl; h < p.H; h += 8) {
    int id = row[h];
    if (id < 0 || id > Ns_) id = Ns_;
    const float4 sp = __ldg(&p.s4[id]);   // (x, y, z, feature); entry Ns = shadow point with feature 0
    const float f = sp.w, rx = sp.x - qx, ry = sp.y - qy, rz = sp.z - qz;
    nn += f > 0.f ? 1 : 0;
    float w[K];
    float dmin = 3.0e38f;
    int kmin = 0;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      float dx = rx - kp_s[3 * k], dy = ry - kp_s[3 * k + 1], dz = rz - kp_s[3 * k + 2];
      float d2 = dx * dx + dy * dy + dz * dz;
      if (d2 < dmin) { dmin = d2; kmin = k; }
      float wk;
      if (p.influence == D3F_INFLUENCE_LINEAR) wk = fmaxf(1.f - sqrt_approx(d2 + 1e-10f) * p.inv_scale, 0.f);
      else if (p.influence == D3F_INFLUENCE_GAUSSIAN) wk = __expf(-d2 * p.gauss_inv);
      else wk = 1.f;
      w[k] = wk;
    }
#pragma unroll
    for (int k = 0; k < K; ++k) wf[k] += (p.closest && k != kmin) ? 0.f : w[k] * f;   // f = 0 for shadow neighbours
  }
  // reduce over the 8 lanes of the query group
#pragma unroll
  for (int o = 1; o < 8; o <<= 1) {
#pragma unroll
    for (int k = 0; k < K; ++k) wf[k] += __shfl_xor_sync(0xffffffffu, wf[k], o);
    nn += __shfl_xor_sync(0xffffffffu, nn, o);
  }
  if (!qvalid) return;
  const float inv_nn = p.normalize ? 1.f / (float)max(nn, 1) : 1.f;
  for (int c = sl; c < p.Cout; c += 8) {
    float y = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) y = fmaf(wf[k], Ws[k * p.Cout + c], y);
    y *= inv_nn;
    if (p.bn_scale) y = fmaf(y, p.bn_scale[c], p.bn_shift[c]);
    if (p.bias) y += p.bias[c];
    if (p.leaky_alpha >= 0.f) y = y > 0.f ? y : y * p.leaky_alpha;
    p.out[(size_t)n * p.Cout + c] = y;
  }
}

// Auxiliary stream + events for the chunk pipeline: one set per (host thread, device), created lazily and destroyed
// with the host thread. Nothing is shared between host threads, so the library stays re-entrant.
struct AuxStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t s1_done[2] = {nullptr, nullptr};
  cudaEvent_t gemm_done[2] = {nullptr, nullptr};
};
constexpr int kMaxDevices = 32;
struct AuxStreams {
  AuxStream dev[kMaxDevices];
  ~AuxStreams() {   // errors ignored: at process exit the context may already be gone
    for (int d = 0; d < kMaxDevices; ++d) {
      if (dev[d].stream == nullptr) continue;
      int cur = 0;
      if (cudaGetDevice(&cur) != cudaSuccess || cudaSetDevice(d) != cudaSuccess) continue;
      for (int i = 0; i < 2; ++i) {
        cudaEventDestroy(dev[d].s1_done[i]);
        cudaEventDestroy(dev[d].gemm_done[i]);
      }
      cudaStreamDestroy(dev[d].stream);
      cudaSetDevice(cur);
    }
  }
};
static AuxStream* aux_stream() {
  static thread_local AuxStreams all;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  AuxStream& a = all.dev[dev];
  if (a.stream != nullptr) return &a;
  // The first multi-chunk call of a thread may come while that thread captures a CUDA graph (global capture mode,
  // as torch.cuda.graph uses). Creating the stream and events is not part of the work being captured, so it runs in
  // relaxed mode, which a capture in progress neither refuses nor is invalidated by.
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  cudaThreadExchangeStreamCaptureMode(&mode);
  AuxStream n;
  bool ok = cudaStreamCreateWithFlags(&n.stream, cudaStreamNonBlocking) == cudaSuccess;
  for (int i = 0; ok && i < 2; ++i)
    ok = cudaEventCreateWithFlags(&n.s1_done[i], cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&n.gemm_done[i], cudaEventDisableTiming) == cudaSuccess;
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (!ok) return nullptr;      // the call then runs its chunks on the caller's stream alone
  a = n;
  return &a;
}

// Queries per chunk of the two-kernel path (stage 1 writes wf[chunk, K*Cin], the contraction of chunk i overlaps
// stage 1 of chunk i+1). Every chunk costs a stage-1 tail, a GEMM launch with its fixed latency and a partial wave,
// and both kernels fill the machine on their own so the overlap buys little, while HBM takes the wf round trip of the
// largest layer in well under the stage-1 time. So: one chunk per layer up to 512 MB of wf per buffer (1 GB of scratch
// per encoder stream out of the 80 GB of an H100); larger layers are cut into
// equal chunks of that size.
static int chunk_queries(int K, int Cin) {
  static const int forced = [] { const char* v = getenv("D3F_KPCONV_CHUNK"); return v ? atoi(v) : 0; }();
  if (forced >= 128) return forced / 128 * 128;      // tuning experiments
  const long long per = (long long)K * Cin * 4;
  long long n = (512ll << 20) / per;
  if (n < 1024) n = 1024;
  return (int)(n / 128 * 128);
}

int kpconv_chunk_queries(int K, int Cin) { return chunk_queries(K, Cin); }

// The support pack of a layer (s4[Ns+1]: x, y, z and the normalisation flag, or the feature itself for the first
// layer). The backward pass packs with this same function, so its neighbour count uses the forward's predicate.
int kpconv_prep_supports(bool deform, const float* s, const float* feat, int Ns, const int* ns_dev, int K, int Cin,
                         int normalize, float4* s4, cudaStream_t stream) {
  const bool norm = normalize != 0 && !deform;
  const bool first_layer = Cin == 1 && !deform && K == 15;
  int pmode = first_layer ? 2 : (norm ? 1 : 0);
  const float shadow = deform ? 1000.f : 1e6f;
  const bool vec = pmode == 1 && Cin % 4 == 0 && Cin >= 32 && (reinterpret_cast<uintptr_t>(feat) & 15) == 0;
  if (vec && Cin < 64)
    prep_supports_vec_kernel<8><<<ceil_div((Ns + 1) * 8, 256), 256, 0, stream>>>(s, feat, Ns, ns_dev, Cin, shadow, s4);
  else if (vec && Cin < 128)
    prep_supports_vec_kernel<16><<<ceil_div((Ns + 1) * 16, 256), 256, 0, stream>>>(s, feat, Ns, ns_dev, Cin, shadow, s4);
  else if (vec)
    prep_supports_vec_kernel<32><<<ceil_div((Ns + 1) * 32, 256), 256, 0, stream>>>(s, feat, Ns, ns_dev, Cin, shadow, s4);
  else
    prep_supports_kernel<<<ceil_div((Ns + 1) * 32, 256), 256, 0, stream>>>(s, feat, Ns, ns_dev, Cin, pmode, shadow, s4);
  D3F_LAUNCH_CHECK("prep_supports_kernel");
  return D3F_OK;
}

// Stage 1 of a rigid layer on its own: wf[n1 - n0, K*Cin] for the query slots [n0, n1), in the forward's query order
// (none here: slot = query), no neighbour count. The weight gradient re-derives wf with it.
int kpconv_stage1_wf(const float* q, const float4* s4, const int* idx, const float* feat, const float* Kp, int Nq, int Ns,
                     int H, int K, int Cin, float extent, int influence, int mode, int n0, int n1, float* wf,
                     cudaStream_t stream, const int* nq_dev, const int* ns_dev) {
  Stage1Params p;
  p.q = q; p.s4 = s4; p.idx = idx; p.feat = feat; p.count_nn = 0;
  p.Kp = Kp; p.offsets = nullptr; p.modulations = nullptr;
  p.Nq = Nq; p.Ns = Ns; p.H = H; p.Cin = Cin;
  p.n0 = n0; p.n1 = n1;
  p.order = nullptr;
  p.extent = extent;
  p.inv_scale = 1.f / (2.f * extent);
  float sigma = extent * 0.3f;
  p.gauss_inv = 1.f / (2.f * sigma * sigma + 1e-9f);
  p.influence = influence;
  p.closest = mode == D3F_MODE_CLOSEST;
  p.shadow = 1e6f;
  p.wf = wf;
  p.inv_nn = nullptr;
  p.nq_dev = nq_dev; p.ns_dev = ns_dev;
  return launch_stage1<false>(K, p, stream);
}

struct KpconvWs {
  float* wf[2];   // stage 1 output, double-buffered (stage 1 of chunk i + 1 overlaps the GEMM of chunk i)
  float* nn[2];   // 1 / neighbour count of each row of wf
  float4* s4;     // packed supports + the shadow point
  float* split;   // split-K partials of the tensor-core GEMM (null when it needs none)
  float* w_img;   // weight image of the fused kernel
};

static size_t kpconv_layout(int Nq, int Ns, int K, int Cin, int Cout, void* base, KpconvWs* w_out) {
  int chunk = chunk_queries(K, Cin);
  if (chunk > Nq) chunk = Nq > 0 ? Nq : 1;
  Carver cv(base);
  KpconvWs w;
  for (int b = 0; b < 2; ++b) w.wf[b] = cv.take<float>((size_t)chunk * K * Cin);
  for (int b = 0; b < 2; ++b) w.nn[b] = cv.take<float>(chunk);
  w.s4 = cv.take<float4>((size_t)Ns + 1);
  const size_t split_floats = tc_gemm_split_ws_floats(chunk, Cout, K * Cin);
  w.split = split_floats ? cv.take<float>(split_floats) : nullptr;
  w.w_img = cv.take<float>(kpconv_fused_image_floats());
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

int kpconv_forward_impl(bool deform, const float* q, const float* s, const int* idx, const float* feat,
                        const float* Kp, const float* offsets, const float* modulations, const float* W,
                        const float* W_packed, const int* query_order, int Nq, int Ns, int H, int K, int Cin, int Cout,
                        float extent,
                        int influence, int mode, int normalize,
                        const float* bn_scale, const float* bn_shift, const float* bias, float leaky_alpha,
                        float* out, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                        const int* nq_dev, const int* ns_dev) {
  D3F_REQUIRE(Nq >= 0 && Ns >= 0 && H >= 0 && Cin >= 1 && Cout >= 1, D3F_ERR_INVALID,
              "kpconv: bad shape Nq=%d Ns=%d H=%d Cin=%d Cout=%d", Nq, Ns, H, Cin, Cout);
  D3F_REQUIRE(K >= 1 && K <= kAnyKMax, D3F_ERR_INVALID, "kpconv: num_kernel_points=%d outside [1, %d]", K, kAnyKMax);
  D3F_REQUIRE(influence >= 0 && influence <= 2, D3F_ERR_INVALID,
              "Unknown influence function type (config.KP_influence)");
  D3F_REQUIRE(mode == D3F_MODE_SUM || mode == D3F_MODE_CLOSEST, D3F_ERR_INVALID,
              "Unknown convolution mode. Should be 'closest' or 'sum'");
  D3F_REQUIRE(extent > 0.f, D3F_ERR_INVALID, "kpconv: KP_extent=%g", (double)extent);
  D3F_REQUIRE((bn_scale == nullptr) == (bn_shift == nullptr), D3F_ERR_INVALID, "kpconv: bn_scale/bn_shift mismatch");
  D3F_REQUIRE(!deform || offsets != nullptr || Nq == 0, D3F_ERR_INVALID, "kpconv_deform: offsets missing");
  KpconvWs w;
  const size_t need = kpconv_layout(Nq, Ns, K, Cin, Cout, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "kpconv: workspace too small");
  if (Nq == 0) return D3F_OK;
  int chunk = chunk_queries(K, Cin);
  if (chunk > Nq) chunk = Nq;
  float4* s4 = w.s4;
  const bool norm = normalize != 0 && !deform;
  {
    const int rc = kpconv_prep_supports(deform, s, feat, Ns, ns_dev, K, Cin, normalize, s4, stream);
    if (rc) return rc;
  }
  // The first-layer kernel stages W[K, Cout] and Kp in 48 KB of shared memory: Cout <= 816. A wider Cin = 1 layer (or
  // the feature gradient of a Cout = 1 layer, whose transposed problem has Cin = 1) runs the two-stage path below;
  // its support pack then holds the feature itself, and the `> 0` test of stage 1's count is the same predicate.
  const size_t c1_smem = (size_t)(K * Cout + K * 3) * sizeof(float);
  if (Cin == 1 && !deform && K == 15 && c1_smem <= 48 * 1024) {
    Cin1Params c1;
    c1.q = q; c1.s4 = s4; c1.idx = idx; c1.Kp = Kp; c1.W = W;
    c1.Nq = Nq; c1.Ns = Ns; c1.H = H; c1.Cout = Cout;
    c1.inv_scale = 1.f / (2.f * extent);
    float sg = extent * 0.3f;
    c1.gauss_inv = 1.f / (2.f * sg * sg + 1e-9f);
    c1.influence = influence; c1.closest = mode == D3F_MODE_CLOSEST; c1.normalize = normalize != 0;
    c1.shadow = 1e6f;
    c1.bn_scale = bn_scale; c1.bn_shift = bn_shift; c1.bias = bias; c1.leaky_alpha = leaky_alpha;
    c1.order = query_order;
    c1.out = out;
    c1.nq_dev = nq_dev; c1.ns_dev = ns_dev;
    if (influence == D3F_INFLUENCE_LINEAR && mode == D3F_MODE_SUM)
      kpconv_cin1_kernel<true><<<ceil_div(ceil_div(Nq, 4) * 32, 256), 256, c1_smem, stream>>>(c1);
    else
      kpconv_cin1_kernel<false><<<ceil_div(ceil_div(Nq, 4) * 32, 256), 256, c1_smem, stream>>>(c1);
    D3F_LAUNCH_CHECK("kpconv_cin1_kernel");
    return D3F_OK;
  }
  if (!deform && W_packed != nullptr &&
      kpconv_fused_supported(Nq, H, K, Cin, Cout, influence, mode, feat, W, out, query_order)) {
    return kpconv_fused_forward(q, s4, idx, feat, Kp, W, w.w_img, Nq, Ns, H, Cout, extent, norm ? 1 : 0, bn_scale, bn_shift,
                                bias, leaky_alpha, out, stream, nq_dev, ns_dev);
  }
  Stage1Params p;
  p.q = q; p.s4 = s4; p.idx = idx; p.feat = feat; p.count_nn = norm ? 1 : 0;
  p.Kp = Kp; p.offsets = offsets; p.modulations = modulations;
  p.Nq = Nq; p.Ns = Ns; p.H = H; p.Cin = Cin;
  p.extent = extent;
  p.inv_scale = deform ? 1.f / extent : 1.f / (2.f * extent);
  float sigma = extent * 0.3f;
  p.gauss_inv = 1.f / (2.f * sigma * sigma + 1e-9f);
  p.influence = influence;
  p.closest = mode == D3F_MODE_CLOSEST;
  p.shadow = deform ? 1000.f : 1e6f;
  p.order = query_order;
  p.nq_dev = nq_dev; p.ns_dev = ns_dev;
  // Chunk pipeline: stage 1 of chunk i+1 (issue-bound on the SM pipes) runs on the caller's stream while the
  // contraction of chunk i (latency-bound, tensor pipe mostly idle, ~9 us of fixed cost per launch) runs on an
  // auxiliary stream; wf / inv_nn are double-buffered and the two streams are joined with events, so from the
  // caller's point of view everything is still ordered on `stream`.
  const int n_chunks = ceil_div(Nq, chunk);
  AuxStream* aux = n_chunks > 1 ? aux_stream() : nullptr;
  for (int ci = 0, n0 = 0; n0 < Nq; n0 += chunk, ++ci) {
    const int b = ci & 1;
    float* wf = w.wf[b];
    float* inv_nn = w.nn[b];
    p.wf = wf;
    p.inv_nn = norm ? inv_nn : nullptr;
    p.n0 = n0;
    p.n1 = min(Nq, n0 + chunk);
    if (aux && ci >= 2) D3F_CUDA(cudaStreamWaitEvent(stream, aux->gemm_done[b], 0));   // buffer b free again
    int rc = deform ? launch_stage1<true>(K, p, stream) : launch_stage1<false>(K, p, stream);
    if (rc) return rc;
    cudaStream_t gs = stream;
    if (aux) {
      D3F_CUDA(cudaEventRecord(aux->s1_done[b], stream));
      D3F_CUDA(cudaStreamWaitEvent(aux->stream, aux->s1_done[b], 0));
      gs = aux->stream;
    }
    Epilogue ep;
    ep.rowscale = norm ? inv_nn : nullptr;
    ep.bn_scale = bn_scale; ep.bn_shift = bn_shift; ep.bias = bias; ep.residual = nullptr;
    ep.leaky_alpha = leaky_alpha;
    // chunk rows are query SLOTS; with a visiting order the epilogue scatters row m to query order[n0 + m]
    ep.row_map = query_order ? query_order + n0 : nullptr;
    ep.m_dev = nq_dev; ep.m_off = n0;                 // rows of this chunk that exist: clamp(*nq_dev - n0, 0, chunk)
    float* cbase = query_order ? out : out + (size_t)n0 * Cout;
    if (W_packed != nullptr && tc_gemm_supported(wf, K * Cin))
      rc = tc_gemm(wf, W_packed, cbase, p.n1 - n0, Cout, K * Cin, ep, gs, w.split);   // chunk GEMMs are serial on gs
    else
      rc = gemm_f32(wf, W, cbase, p.n1 - n0, Cout, K * Cin, ep, gs);
    if (rc) return rc;
    if (aux) D3F_CUDA(cudaEventRecord(aux->gemm_done[b], aux->stream));
  }
  if (aux) {   // join: everything enqueued after this call on `stream` sees the complete output
    D3F_CUDA(cudaStreamWaitEvent(stream, aux->gemm_done[0], 0));
    if (n_chunks > 1) D3F_CUDA(cudaStreamWaitEvent(stream, aux->gemm_done[1], 0));
  }
  return D3F_OK;
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_kpconv_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout) {
  (void)H;
  return kpconv_layout(Nq, Ns, K, Cin, Cout, nullptr, nullptr);
}

extern "C" int d3f_kpconv_forward(const float* q, const float* s, const int* idx, const float* feat, const float* Kp,
                                  const float* W, const float* W_packed, const int* query_order, int Nq, int Ns, int H,
                                  int K, int Cin, int Cout, float extent, int influence, int mode, int normalize,
                                  const float* bn_scale, const float* bn_shift, const float* bias, float leaky_alpha,
                                  float* out, void* workspace, size_t workspace_bytes, d3f_stream_t stream,
                                  const int* nq_dev, const int* ns_dev) {
  // an empty support set (Ns == 0: every index is the shadow point) has no coordinates or features to point at
  D3F_REQUIRE(Nq == 0 || (q && idx && Kp && W && out && workspace && (Ns == 0 || (s && feat))), D3F_ERR_INVALID,
              "d3f_kpconv_forward: null pointer");
  return kpconv_forward_impl(false, q, s, idx, feat, Kp, nullptr, nullptr, W, W_packed, query_order, Nq, Ns, H, K, Cin,
                             Cout, extent, influence, mode, normalize, bn_scale, bn_shift, bias, leaky_alpha, out,
                             workspace, workspace_bytes, (cudaStream_t)stream, nq_dev, ns_dev);
}

extern "C" int d3f_kpconv_deform_forward(const float* q, const float* s, const int* idx, const float* feat,
                                         const float* Kp, const float* offsets, const float* modulations,
                                         const float* W, const float* W_packed, const int* query_order, int Nq, int Ns,
                                         int H, int K, int Cin, int Cout, float extent, int influence, int mode,
                                         const float* bn_scale, const float* bn_shift, const float* bias,
                                         float leaky_alpha, float* out, void* workspace, size_t workspace_bytes,
                                         d3f_stream_t stream, const int* nq_dev, const int* ns_dev) {
  D3F_REQUIRE(Nq == 0 || (q && idx && Kp && W && out && workspace && offsets && (Ns == 0 || (s && feat))),
              D3F_ERR_INVALID, "d3f_kpconv_deform_forward: null pointer");
  return kpconv_forward_impl(true, q, s, idx, feat, Kp, offsets, modulations, W, W_packed, query_order, Nq, Ns, H, K,
                             Cin, Cout, extent, influence, mode, 0, bn_scale, bn_shift, bias, leaky_alpha, out,
                             workspace, workspace_bytes, (cudaStream_t)stream, nq_dev, ns_dev);
}

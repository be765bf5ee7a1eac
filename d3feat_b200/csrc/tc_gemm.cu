// Tensor-core GEMM for sm_90a: wgmma.mma_async (tf32) with the accumulator in registers, fp32-accurate through
// a 3xTF32 split:   A = Ah + Al,  B = Bh + Bl  (Ah/Bh = operand rounded to TF32, Al/Bl = exact remainder)
//                   D += Ah*Bh + Al*Bh + Ah*Bl          (dropped Al*Bl term ~ 2^-22 relative)
//
//   C[M,N] = epilogue( rowscale[m] * (A[M,K] @ W[K,N]) )
//
// * A is the activation matrix (row-major fp32 in global memory). One producer thread loads each 128 x 32 k-chunk of
//   it by TMA through a 2D tensor map (SWIZZLE_128B, out-of-bounds rows and columns zero-filled) into an mbarrier ring.
// * W is static: it is packed once (pack_weight_kernel) into K-major [Npad, Kpad] hi/lo images that arrive by TMA bulk
//   copies on the same barrier as the A chunk.
// * Two consumer warpgroups (M = 64 rows each, N = BN, K = 8 per instruction) read their A fragments from the swizzled
//   stage with conflict-free 32-bit shared loads, split them into (hi, lo) in registers and issue the register-A (RS)
//   form of wgmma against the B images in shared memory.
// * Epilogue: each consumer warp turns its 16 x BN accumulator block through a 1 KB corner of shared memory, 8 rows x
//   32 columns at a time, so that 8 lanes hold one row's 128 contiguous bytes. Rowscale / BN / bias / residual /
//   LeakyReLU are applied in that layout (BN and bias vectors staged in shared memory once per column tile), and C and
//   the residual move as whole 128-byte row pieces: 16-byte accesses when N % 4 == 0, single floats otherwise.
// * Footprint: 9 warps; for BN <= 64 a CTA stays within half an SM's registers and shared memory, so two GEMM CTAs,
//   or one GEMM CTA and the kernels of another stream, share an SM and cover each other's k-chunk drains and epilogues.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <stdlib.h>

#include "ops.cuh"
#include "tc_common.cuh"

namespace d3f {

constexpr int kTcBM = 128;       // rows per tile (two wgmma warpgroups of M = 64)
constexpr int kTcBK = 32;        // fp32 per k-chunk = one 128 B swizzle row
constexpr int kTcConsumerWarps = 8;
constexpr int kTcThreads = 32 * kTcConsumerWarps + 32;   // 2 consumer warpgroups (warps 0-7) + 1 producer warp

// ---------------------------------------------------------------------------------------------------
// W[K,N] row-major -> packed[Kpad/32][2][Npad][32]: for every 32-wide k-chunk a (hi, lo) pair of ready-made shared
// memory images: row n holds the 32 k-values of output column n as 128 bytes whose 16-byte chunks are XOR-swizzled
// with (n & 7) -- exactly the K-major SWIZZLE_128B layout the wgmma descriptor reads. A BN-row tile of a k-chunk is
// therefore ONE contiguous block per image and is fetched by a single TMA bulk copy (cp.async.bulk).
__global__ void __launch_bounds__(256) pack_weight_kernel(const float* __restrict__ W, int K, int N, int Kpad,
                                                          int Npad, float* __restrict__ packed) {
  long long total = (long long)Npad * Kpad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int k = (int)(i / Npad), n = (int)(i % Npad);      // consecutive threads: consecutive n (coalesced reads of W)
    float x = (n < N && k < K) ? W[(size_t)k * N + n] : 0.f;
    float hi, lo;
    split_tf32(x, hi, lo);
    int kc = k >> 5, kl = k & 31;
    size_t slab = (size_t)kc * 2 * Npad * 32;
    size_t off = (size_t)n * 32 + (size_t)((((kl >> 2) ^ (n & 7)) << 2) | (kl & 3));
    packed[slab + off] = hi;
    packed[slab + (size_t)Npad * 32 + off] = lo;
  }
}

static int tc_padded_k(int K) { return (K + kTcBK - 1) / kTcBK * kTcBK; }
static int tc_block_n(int N) { return N > 64 ? 128 : (N > 32 ? 64 : 32); }
static int tc_padded_n(int N) { int bn = tc_block_n(N); return (N + bn - 1) / bn * bn; }

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_packed_weight_floats(int K, int N) { return 2 * (size_t)tc_padded_k(K) * tc_padded_n(N); }

extern "C" int d3f_pack_weight(const float* W, int K, int N, float* packed, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(K >= 1 && N >= 1 && W && packed, D3F_ERR_INVALID, "pack_weight: bad arguments");
  int Kpad = tc_padded_k(K), Npad = tc_padded_n(N);
  long long total = (long long)Npad * Kpad;
  int blocks = (int)min((total + 255) / 256, (long long)kNumSMs * 8);
  pack_weight_kernel<<<blocks, 256, 0, stream>>>(W, K, N, Kpad, Npad, packed);
  D3F_LAUNCH_CHECK("pack_weight_kernel");
  return D3F_OK;
}

namespace d3f {

// ---------------------------------------------------------------------------------------------------
// Accumulation. Each k-chunk (12 wgmmas) is summed into a fresh register fragment that the consumer adds to the running
// sum with round-to-nearest once the chunk has retired: the tensor pipe's own fp32 accumulate is biased towards zero,
// and restarting it every chunk keeps that chain 12 MMAs long whatever K is. Measured on an H100 SXM (400 W power
// limit) against one running accumulator, M x K x N = 4096 x 7680 x 512, max-norm error vs float64: 1.2e-6 vs 8.5e-5
// on all-positive data (mean signed error -2.7e-7 vs -7.9e-5), 8.4e-7 vs 6.0e-5 on normal data.
//
// Inside a chunk each K = 8 step is one commit group and two steps are in flight (wait_group 1), so only two steps'
// split A fragments are live. A consumer does wait for the chunk's last step before the next chunk: overlapping two
// chunks would keep two accumulators live, which rules out two CTAs per SM; the other warpgroup and the second CTA keep
// the tensor pipe busy across that drain instead.
//
// Ring: a stage is one raw A chunk (16 KB) + the B hi/lo images. BN <= 64: two CTAs per SM, so <= 96 registers per
// thread (9 warps per CTA: one of the SM's four register-file quarters holds 5 of the 18 warps) and <= 113 KB of shared
// memory each; BN = 128 (64-register accumulators) keeps one CTA per SM and 3 stages. The epilogue area (per consumer
// warp one 1 KB pass and 3 x BN floats of column vectors) comes on top of the ring: 108 / 111 / 165 KB in all for
// BN = 32 / 64 / 128.
template <int BN>
struct TcSmem {
  static constexpr int kCtasPerSm = BN >= 128 ? 1 : 2;
  static constexpr int kStages = BN >= 64 ? 3 : 4;
  static constexpr int kABytes = kTcBM * 128;  // the raw fp32 A tile of one k-chunk
  static constexpr int kBBytes = BN * 128;     // one image (hi or lo) of the B tile
  static constexpr int kStageBytes = kABytes + 2 * kBBytes;
  static constexpr int kEpiWarpBytes = 1024 + 3 * BN * 4;  // per consumer warp: one epilogue pass + the column vectors
  static constexpr int kTotal = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/ + kTcConsumerWarps * kEpiWarpBytes;
  static_assert(kCtasPerSm * (kTotal + 1024) <= 233472, "shared memory of an H100 SM (228 KB, 1 KB reserved per CTA)");
};

// One kernel for both launch shapes: grid.x = every output tile (one tile per CTA; split-K over grid.z) or fewer CTAs
// than tiles (persistent: CTA b takes tiles b, b + gridDim.x, ...; the producer's ring runs across tile boundaries, so
// the next tile's operands load while the consumers run the epilogue of the current one). n-tiles of one row block are
// neighbours in the tile order: the A rows stay in L2.
//
// tmA / tmA2: tensor maps of the A operand, [A | A2] along K when K1 < Kpad (K1 = columns of A, a multiple of the
// k-chunk, so a whole k-chunk comes from one of the two matrices). Rows past the device row count ep.m_dev but below the
// capacity are loaded but never stored.
template <int BN>
__global__ void __launch_bounds__(kTcThreads, TcSmem<BN>::kCtasPerSm)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2, int K1,
               const float* __restrict__ Bp, float* __restrict__ C, int Mcap, int N, int Kpad, int Npad,
               int chunks_per_split, Epilogue ep) {
  // the split-K slabs are laid out with the launch capacity; the rows that exist come from device memory if given
  const int M = ep.m_dev ? min(Mcap, max(__ldg(ep.m_dev) - ep.m_off, 0)) : Mcap;
  const int ntn = Npad / BN;
  const int tiles = ceil_div(M, kTcBM) * ntn;
  if ((int)blockIdx.x >= tiles) return;   // CTA-uniform, before any barrier
  extern __shared__ uint8_t smem_raw[];
  using S = TcSmem<BN>;
  constexpr int kStages = S::kStages;
  // 1024 B alignment: SWIZZLE_128B atoms are 8 rows x 128 B and the swizzle uses absolute address bits
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + kStages * S::kStageBytes);   // [kStages] A chunk + B images landed
  uint64_t* empty = full + kStages;                                // [kStages] the consumers are done with the stage

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // split-K: CTA z owns the k-chunks [kt0, kt0 + nk) and writes raw partial sums to its own [M,N] slab of C
  const int kt0 = blockIdx.z * chunks_per_split;
  const int nk = min(Kpad / kTcBK - kt0, chunks_per_split);
  float* Cz = C + (size_t)blockIdx.z * Mcap * N;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(&full[s]), 1);                        // the producer's arrive.expect_tx
      mbar_init(smem_u32(&empty[s]), kTcConsumerWarps);        // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kTcConsumerWarps) {
    // ===================== producer: one thread issues every copy of the ring ==============================
    if (lane == 0) {
      const int total = (tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x * nk;   // chunks of my tiles
      int tile = (int)blockIdx.x, kt = 0;
      for (int g = 0; g < total; ++g) {
        const int s = g % kStages;
        mbar_wait(smem_u32(&empty[s]), ((uint32_t)(g / kStages) & 1u) ^ 1u);   // stage free
        const uint32_t st = smem_u32(smem + s * S::kStageBytes);
        const uint32_t fb = smem_u32(&full[s]);
        const int m0 = (tile / ntn) * kTcBM, n0 = (tile % ntn) * BN;
        const int k0 = (kt0 + kt) * kTcBK;
        mbar_arrive_expect_tx(fb, (uint32_t)S::kStageBytes);
        if (k0 < K1)
          tma_load_2d(st, &tmA, k0, m0, fb);
        else
          tma_load_2d(st, &tmA2, k0 - K1, m0, fb);
        // B operand of this k-chunk: two contiguous pre-swizzled images (hi, lo) of BN rows x 128 B
        const float* slab = Bp + (size_t)(kt0 + kt) * 2 * Npad * 32 + (size_t)n0 * 32;
        tma_bulk_g2s(st + S::kABytes, slab, S::kBBytes, fb);
        tma_bulk_g2s(st + S::kABytes + S::kBBytes, slab + (size_t)Npad * 32, S::kBBytes, fb);
        if (++kt == nk) {
          kt = 0;
          tile += (int)gridDim.x;
        }
      }
    }
  } else {
    // ===================== consumers: two warpgroups, 64 rows of the tile each ==============================
    // Per k-chunk and K = 8 step three wgmmas (3xTF32): Ah.Bh + Al.Bh + Ah.Bl (the Al.Bl term, ~2^-22 relative, is
    // dropped). Then the stage is released and the chunk's fragment joins the running sum.
    constexpr int R = BN / 2;                 // accumulator registers per thread (m64 x BN per warpgroup)
    const int cw = warp >> 2;                 // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
    const int wq = warp & 3;                  // warp inside the warpgroup: rows 16 wq .. 16 wq + 15 of its 64
    // this thread's A fragment: rows r0 and r0 + 8, columns 8 j + t and 8 j + t + 4 of every K = 8 step j. In the
    // SWIZZLE_128B stage row r holds its 16-byte pieces XOR-ed with r % 8 (the same for r0 and r0 + 8): the eight
    // rows of a warp's load hit eight different pieces, the four threads of a row four banks of one piece.
    const int r0 = 64 * cw + 16 * wq + (lane >> 2);
    const uint32_t a_row = (uint32_t)r0 * 128u + (uint32_t)(lane & 3) * 4u, a_swz = (uint32_t)(r0 & 7);
    // x[q] = A[r0 + 8 (q & 1)][8 j + t + 4 (q >> 1)] of the stage at sa: the tf32 fragment order of wgmma_tf32_rs
    auto load_a = [&](float* x, uint32_t sa, int j) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        x[q] = lds32(sa + a_row + (uint32_t)(q & 1) * 1024u + ((((uint32_t)(2 * j + (q >> 1))) ^ a_swz) << 4));
    };
    float acc[R], sum[R];
    int g = 0;
    for (int t = (int)blockIdx.x; t < tiles; t += (int)gridDim.x) {
      const int m0 = (t / ntn) * kTcBM, n0 = (t % ntn) * BN;
#pragma unroll
      for (int j = 0; j < R; ++j) sum[j] = 0.f;
      for (int kt = 0; kt < nk; ++kt, ++g) {
        const int s = g % kStages;
        mbar_wait(smem_u32(&full[s]), (uint32_t)(g / kStages) & 1u);
        const uint32_t sa = smem_u32(smem + s * S::kStageBytes);
        const uint64_t b_hi = make_smem_desc(sa + S::kABytes), b_lo = make_smem_desc(sa + S::kABytes + S::kBBytes);
        // one commit group per K = 8 step; the split fragment of step j lives in buffer j % 2 until wait_group 1
        // after step j + 1 has retired it, so at most two steps' fragments (16 registers) are live
        float x[4];
        uint32_t ah[2][4], al[2][4];
        load_a(x, sa, 0);
#pragma unroll
        for (int j = 0; j < R; ++j) acc[j] = 0.f;
#pragma unroll
        for (int j = 0; j < kTcBK / 8; ++j) {
          uint32_t* h = ah[j & 1];
          uint32_t* l = al[j & 1];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float hi, lo;
            split_tf32(x[q], hi, lo);
            h[q] = __float_as_uint(hi);
            l[q] = __float_as_uint(lo);
          }
          const uint64_t adv = (uint64_t)((j * 32) >> 4);   // +32 B per K = 8 step inside the swizzle atom
          wgmma_fence();
          wgmma_tf32_rs<BN>(acc, h, b_hi + adv);
          wgmma_tf32_rs<BN>(acc, l, b_hi + adv);
          wgmma_tf32_rs<BN>(acc, h, b_lo + adv);
          wgmma_commit();
          if (j + 1 < kTcBK / 8) load_a(x, sa, j + 1);
          wgmma_wait<1>();
        }
        wgmma_wait<0>();
        wgmma_reg_fence<R>(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&empty[s]));       // this warp is done with the stage
#pragma unroll
        for (int j = 0; j < R; ++j) sum[j] += acc[j];
      }
      // ===================== epilogue: fragment -> shared memory -> whole 128-byte row pieces ======================
      const bool has_bn = ep.bn_scale != nullptr, has_bias = ep.bias != nullptr, has_res = ep.residual != nullptr;
      const bool has_leaky = ep.leaky_alpha >= 0.f;
      // a lane's four adjacent columns of a row are one aligned 16-byte access (a split-K slab starts a multiple of
      // N floats into C)
      const bool vec = (N & 3) == 0 &&
                       ((reinterpret_cast<uintptr_t>(C) | reinterpret_cast<uintptr_t>(ep.residual)) & 15) == 0;
      // this warp's corner of the epilogue area: one 8 row x 128 B pass, then [bn_scale | bn_shift | bias] of BN columns
      const uint32_t st_tile = smem_u32(smem + kStages * S::kStageBytes + 256) + (uint32_t)warp * S::kEpiWarpBytes;
      const uint32_t st_par = st_tile + 1024u;
      // The BN / bias vectors of this column tile, once per warp and again only when the tile's columns change.
      if (t == (int)blockIdx.x || ntn > 1) {
        for (int c = lane; c < BN; c += 32) {
          const int n = n0 + c;
          if (has_bn) {
            sts32(st_par + 4u * c, n < N ? ep.bn_scale[n] : 0.f);
            sts32(st_par + 4u * (BN + c), n < N ? ep.bn_shift[n] : 0.f);
          }
          if (has_bias) sts32(st_par + 4u * (2 * BN + c), n < N ? ep.bias[n] : 0.f);
        }
      }   // visible to the warp after the __syncwarp of the first pass below
      // A pass moves 8 rows x 32 columns of the warp's 16 x BN block: the fragment layout (row l / 4, column pairs
      // 8 j + 2 (l % 4)) goes in with 8-byte stores, and comes back as rows: 8 lanes hold the eight 16-byte pieces of
      // one row, so a warp-wide access to C or the residual covers 4 rows x 128 contiguous bytes. Piece p of row r
      // sits at p ^ (2 (r % 4)) ^ (r / 4): both the stores (half a warp = rows r..r + 3 x 2 pieces) and the loads (a
      // quarter warp = one row) touch every bank once.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int cg = 0; cg < BN / 32; ++cg) {
          {
            const uint32_t r = (uint32_t)(lane >> 2), tq = (uint32_t)(lane & 3);
            const uint32_t swz = ((r & 3u) << 1) ^ (r >> 2);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * cg + jj;
              sts64(st_tile + r * 128u + (((uint32_t)(2 * jj) + (tq >> 1)) ^ swz) * 16u + (tq & 1u) * 8u,
                    sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
            }
          }
          __syncwarp();
          const int pc = lane & 7;                       // this lane's 16-byte piece: columns 4 pc .. 4 pc + 3
          const int gn = n0 + 32 * cg + 4 * pc;
          const uint32_t par = st_par + 4u * (32 * cg + 4 * pc);   // this lane's four columns of the vectors
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const uint32_t r = (uint32_t)(lane >> 3) + 4u * i;
            const float4 v = lds128(st_tile + r * 128u + (((uint32_t)pc ^ ((r & 3u) << 1) ^ (r >> 2)) << 4));
            const int gm = m0 + 64 * cw + 16 * wq + 8 * h + (int)r;
            if (gm >= M || gn >= N) continue;
            const float rs = ep.rowscale != nullptr ? ep.rowscale[gm] : 1.f;
            // output row: identity, or the caller's row map (KPConv walks its queries in the hash grid's cell order
            // and scatters the rows back)
            const size_t orow = ep.row_map ? (size_t)ep.row_map[gm] : (size_t)gm;
            float* cp = Cz + orow * N + gn;
            const float* rp = has_res ? ep.residual + orow * N + gn : nullptr;
            float y[4] = {v.x * rs, v.y * rs, v.z * rs, v.w * rs};
            float res[4] = {0.f, 0.f, 0.f, 0.f};
            if (has_res) {
              if (vec) {
                const float4 rv = *reinterpret_cast<const float4*>(rp);
                res[0] = rv.x; res[1] = rv.y; res[2] = rv.z; res[3] = rv.w;
              } else {
#pragma unroll
                for (int e = 0; e < 4; ++e)
                  if (gn + e < N) res[e] = rp[e];
              }
            }
            if (has_bn) {
              const float4 sc = lds128(par), sh = lds128(par + 4u * BN);
              y[0] = fmaf(y[0], sc.x, sh.x); y[1] = fmaf(y[1], sc.y, sh.y);
              y[2] = fmaf(y[2], sc.z, sh.z); y[3] = fmaf(y[3], sc.w, sh.w);
            }
            if (has_bias) {
              const float4 bi = lds128(par + 8u * BN);
              y[0] += bi.x; y[1] += bi.y; y[2] += bi.z; y[3] += bi.w;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              y[e] += res[e];
              if (has_leaky) y[e] = y[e] > 0.f ? y[e] : y[e] * ep.leaky_alpha;
            }
            if (vec) {
              *reinterpret_cast<float4*>(cp) = make_float4(y[0], y[1], y[2], y[3]);
            } else {
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (gn + e < N) cp[e] = y[e];
            }
          }
          __syncwarp();   // the pass has been read before the next one overwrites it
        }
      }
    }
  }
}

// fixed-order reduction of the split-K partials + the block epilogue
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, int splits, int Mcap, int N,
                                                            Epilogue ep, float* __restrict__ C) {
  const int M = ep.m_dev ? min(Mcap, max(__ldg(ep.m_dev) - ep.m_off, 0)) : Mcap;
  const long long slab = (long long)Mcap * N;
  long long total = (long long)M * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int m = (int)(i / N), n = (int)(i % N);
    float y = 0.f;
    for (int z = 0; z < splits; ++z) y += part[(size_t)z * slab + i];
    if (ep.rowscale) y *= ep.rowscale[m];
    if (ep.bn_scale) y = fmaf(y, ep.bn_scale[n], ep.bn_shift[n]);
    if (ep.bias) y += ep.bias[n];
    const size_t orow = ep.row_map ? (size_t)ep.row_map[m] : (size_t)m;
    if (ep.residual) y += ep.residual[orow * N + n];
    if (ep.leaky_alpha >= 0.f) y = y > 0.f ? y : y * ep.leaky_alpha;
    C[orow * N + n] = y;
  }
}

// 2D tensor map of a row-major fp32 matrix [rows, cols] (cols % 4 == 0, 16-byte aligned): boxes of 128 rows x one
// k-chunk, SWIZZLE_128B (the K-major layout the consumers' fragment loads expect), zero fill out of bounds. The driver's
// encoder is looked up through the runtime, so the library does not need libcuda to load (the CPU-only build imports it).
static int encode_a_map(CUtensorMap* map, const float* A, int rows, int cols) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    D3F_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    D3F_REQUIRE(q == cudaDriverEntryPointSuccess && fn != nullptr, D3F_ERR_CUDA,
                "tc_gemm: the driver has no cuTensorMapEncodeTiled");
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)kTcBK, (cuuint32_t)kTcBM};
  const cuuint32_t elem[2] = {1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(A), dims, strides, box, elem,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  D3F_REQUIRE(r == CUDA_SUCCESS, D3F_ERR_CUDA, "tc_gemm: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return D3F_OK;
}

// persistent = true: at most kCtasPerSm CTAs per SM, each walking several tiles (see tc_gemm_kernel)
template <int BN>
static int launch_tc(const float* A, const float* A2, int K1, const float* Bp, float* C, int M, int N, int K,
                     const Epilogue& ep, cudaStream_t stream, int splits, float* split_ws, bool persistent) {
  using S = TcSmem<BN>;
  static bool configured = false;   // idempotent attribute set; benign if two host threads race
  if (!configured) {
    D3F_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal));
    configured = true;
  }
  const int Kpad = tc_padded_k(K), Npad = tc_padded_n(N);
  const int nk = Kpad / kTcBK;
  const int tiles = ceil_div(M, kTcBM) * (Npad / BN);
  // the maps are kernel parameters: a CUDA graph capture records them by value
  CUtensorMap tmA, tmA2;
  if (A2 != nullptr) {
    int rc = encode_a_map(&tmA, A, M, K1);
    if (rc == D3F_OK) rc = encode_a_map(&tmA2, A2, M, K - K1);
    if (rc != D3F_OK) return rc;
  } else {
    const int rc = encode_a_map(&tmA, A, M, K);
    if (rc != D3F_OK) return rc;
    tmA2 = tmA;
    K1 = Kpad;
  }
  if (splits <= 1) {
    const int cap = kNumSMs * S::kCtasPerSm;
    const int grid = persistent && tiles > cap ? cap : tiles;
    tc_gemm_kernel<BN><<<grid, kTcThreads, S::kTotal, stream>>>(tmA, tmA2, K1, Bp, C, M, N, Kpad, Npad, nk, ep);
    D3F_LAUNCH_CHECK("tc_gemm_kernel");
    return D3F_OK;
  }
  const int cps = ceil_div(nk, splits);
  splits = ceil_div(nk, cps);
  Epilogue raw;
  raw.rowscale = nullptr; raw.bn_scale = nullptr; raw.bn_shift = nullptr; raw.bias = nullptr; raw.residual = nullptr;
  raw.leaky_alpha = -1.f; raw.row_map = nullptr; raw.m_dev = ep.m_dev; raw.m_off = ep.m_off;
  dim3 grid(tiles, 1, splits);
  tc_gemm_kernel<BN><<<grid, kTcThreads, S::kTotal, stream>>>(tmA, tmA2, K1, Bp, split_ws, M, N, Kpad, Npad, cps, raw);
  D3F_LAUNCH_CHECK("tc_gemm_kernel");
  long long total = (long long)M * N;
  int blocks = (int)min((total + 255) / 256, (long long)kNumSMs * 8);
  splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(split_ws, splits, M, N, ep, C);
  D3F_LAUNCH_CHECK("splitk_reduce_kernel");
  return D3F_OK;
}

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

bool tc_gemm_supported(const float* A, int K) {
  return (K % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
}

// A[M,K] fp32 row-major, Bp = packed weight (d3f_pack_weight), C[M,N]
// split-K plan for GEMMs that cannot fill the GPU with output tiles: returns the number of K splits (1 = none)
// Deterministic split-K plan for GEMMs whose output tiles cannot fill the GPU. The k-loop of a CTA is latency bound
// (about a microsecond per k-chunk), so the cost of a plan is (waves of CTAs) x (k-chunks per CTA) plus the extra
// pass of the reduction; the cheapest of s = 1..8 wins. Returns the number of K splits (1 = none).
static int tc_gemm_splits(int M, int N, int K) {
  const int bn = tc_block_n(N);
  const long long ctas = (long long)ceil_div(M, kTcBM) * (tc_padded_n(N) / bn);
  const int nk = tc_padded_k(K) / kTcBK;
  if (ctas >= 96 || nk < 16) return 1;
  int best = 1;
  long long best_cost = (long long)ceil_div((int)ctas, kNumSMs) * nk * 8;   // in eighths of a k-chunk
  for (int s = 2; s <= 8 && s <= nk / 4; ++s) {
    const int cps = ceil_div(nk, s);
    const int eff = ceil_div(nk, cps);   // splits actually launched
    if (eff != s) continue;
    long long cost = (long long)ceil_div((int)(ctas * s), kNumSMs) * cps * 8 + 40 + 6 * s;   // + reduce launch, traffic
    if (cost < best_cost) {
      best_cost = cost;
      best = s;
    }
  }
  return best;
}
// Workspace bound that holds for every M' <= M of the same GEMM family (the chunks of one KPConv share a buffer): the
// planner only splits below 96 output tiles and never more than 8 ways, and a partial slab is at most one 128 x bn
// tile per CTA, so 8 x min(tiles, 95) tiles always suffice.
size_t tc_gemm_split_ws_floats(int M, int N, int K) {
  const int bn = tc_block_n(N);
  const long long ctas = (long long)ceil_div(M, kTcBM) * (tc_padded_n(N) / bn);
  const int nk = tc_padded_k(K) / kTcBK;
  if (nk < 16) return 0;
  // rows/cols covered by one CTA tile: 128 x bn. Worst case over all M' <= M: min(ctas, 95) tiles x 8 splits.
  const long long tiles = ctas < 95 ? ctas : 95;
  return (size_t)(8 * tiles * kTcBM * bn);
}

int tc_gemm(const float* A, const float* Bp, float* C, int M, int N, int K, const Epilogue& ep, cudaStream_t stream,
            float* split_ws, const float* A2, int K1) {
  if (M <= 0 || N <= 0) return D3F_OK;
  D3F_REQUIRE(tc_gemm_supported(A, K), D3F_ERR_INVALID, "tc_gemm: needs K %% 4 == 0 and 16-byte aligned A");
  if (A2 != nullptr)
    D3F_REQUIRE(K1 > 0 && K1 < K && K1 % kTcBK == 0 && tc_gemm_supported(A2, K - K1), D3F_ERR_INVALID,
                "tc_gemm: split A operand needs K1 %% %d == 0 and a 16-byte aligned second matrix", kTcBK);
  int bn = tc_block_n(N);
  // skinny-K, huge-M GEMMs (the level-0/1 unary convolutions) are bound by per-tile fixed costs and the C write:
  // 64-wide column tiles halve the accumulator registers of a consumer thread. The packed image is the same (Npad is a
  // multiple of 128, hence of 64).
  if (bn == 128 && K <= 256 && M >= 8192) bn = 64;
  const int splits = split_ws != nullptr ? tc_gemm_splits(M, N, K) : 1;
  // Persistent CTAs (one per SM, the ring running across tiles) for the skinny-K GEMMs: a tile of <= 4 k-chunks is
  // over before a freshly launched CTA would have filled its ring. D3F_TC_STREAM=1 (read per call: tests switch it on
  // and off) extends this to every GEMM without split-K.
  const bool persistent = splits <= 1 && (tc_padded_k(K) / kTcBK <= 4 || env_int("D3F_TC_STREAM", 0) != 0);
  switch (bn) {
    case 128: return launch_tc<128>(A, A2, K1, Bp, C, M, N, K, ep, stream, splits, split_ws, persistent);
    case 64: return launch_tc<64>(A, A2, K1, Bp, C, M, N, K, ep, stream, splits, split_ws, persistent);
    default: return launch_tc<32>(A, A2, K1, Bp, C, M, N, K, ep, stream, splits, split_ws, persistent);
  }
}

}  // namespace d3f

extern "C" int d3f_unary_pair_forward(const float* x1, int Cin1, const float* x2, int Cin2, const float* W_packed,
                                      int N, int Cout, const float* shift, float leaky_alpha, float* out,
                                      d3f_stream_t stream, const int* n_dev) {
  D3F_REQUIRE(N >= 0 && Cin1 >= 1 && Cin2 >= 1 && Cout >= 1, D3F_ERR_INVALID,
              "d3f_unary_pair_forward: bad shape N=%d Cin=%d+%d Cout=%d", N, Cin1, Cin2, Cout);
  D3F_REQUIRE(N == 0 || (x1 && x2 && W_packed && out), D3F_ERR_INVALID, "d3f_unary_pair_forward: null pointer");
  D3F_REQUIRE(Cin1 % 32 == 0 && Cin2 % 4 == 0, D3F_ERR_INVALID,
              "d3f_unary_pair_forward: Cin1 must be a multiple of 32 and Cin2 of 4 (got %d, %d)", Cin1, Cin2);
  Epilogue ep;
  ep.rowscale = nullptr;
  ep.bn_scale = nullptr;
  ep.bn_shift = nullptr;
  ep.bias = shift;
  ep.residual = nullptr;
  ep.leaky_alpha = leaky_alpha;
  ep.row_map = nullptr;
  ep.m_dev = n_dev;
  return tc_gemm(x1, W_packed, out, N, Cout, Cin1 + Cin2, ep, (cudaStream_t)stream, nullptr, x2, Cin1);
}

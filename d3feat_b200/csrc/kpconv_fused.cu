// Rigid KPConv (kernels/convolution_ops.py:161-255) as ONE persistent kernel for the Cin = 32 layers (the two largest
// KPConvs of the D3Feat encoder: level-0 resnetb conv2 and the level-0 -> 1 strided conv2, models/network_blocks.py:
// 321-368, 561-612). No intermediate leaves the SM:
//
//   gather warps (15 per CTA)   one query per warp at a time, rows handed out from a shared counter: neighbour ids ->
//                               packed support points -> feature rows (coalesced 128 B row reads, loads issued one
//                               8-neighbour step ahead of the math, ids two steps ahead, two alternating register sets),
//                               kernel-point correlation weights in registers in mma A-fragment layout,
//                               wf[16 kp x 32 ch] += w^T . f on the tensor pipe (mma.sync m16n8k8, 3xTF32), x 1/nn, then
//                               the query's wf row is split (hi, lo) and written STRAIGHT into the shared-memory operand
//                               of the contraction: per kernel point [48 hi rows | 48 lo rows] x 128 B, K-major
//                               SWIZZLE_128B, the layout the wgmma descriptors read.
//   control warp 15 (lane 0)    W ring producer: TMA bulk copies of pre-swizzled 8 KB images, 4 stages.
//   MMA warpgroup 16..19        out^T[64 x 96] += Wimg[kp] (64 rows = TF32-hi and remainder of the 32 output channels) .
//                               [wf_hi | wf_lo][:, kp, :]^T on wgmma (tf32, M = 64, N = 96, ONE wgmma per K = 8 step,
//                               60 per tile), accumulator in registers; then hi + lo rows, hi + lo columns ->
//                               batch-norm affine -> bias -> LeakyReLU -> out.
//
// Tile shape: the wf operand of a tile is 15 kernel points x [48 hi rows | 48 lo rows] x 128 B = 180 KB and shares the
// 227 KB of an SM with a 4-stage ring of 8 KB W images. One tile in flight: the gather warps are already inside their
// next queries while its 60 MMAs run; only the WRITE of the next tile's rows waits for them (`consumed` counter).
#include <stdlib.h>

#include "ops.cuh"
#include "tc_common.cuh"

namespace d3f {

namespace {

constexpr int kFRows = 48;                       // queries per tile (see "Tile shape" above)
constexpr int kFGatherWarps = 15;                // rows are handed out dynamically
constexpr int kFCtrlWarp = 15;                   // lane 0: W ring producer, nothing else
constexpr int kFEpiWarp0 = 16;                   // warps 16..19: the MMA warpgroup (wgmma + epilogue)
constexpr int kFThreads = 20 * 32;
// (20 warps = 5 per SM sub-partition: 5 x 32 x 96 registers fit its 16 K registers; a 21st warp would cap everyone at 80)
constexpr int kFKp = 15;
constexpr int kFImageBytes = kFRows * 128;       // hi (or lo) rows of one kernel point: 6 KB
constexpr int kFChunkBytes = 2 * kFImageBytes;   // one kernel point of the wf tile: [48 hi rows | 48 lo rows] x 128 B
static_assert(kFImageBytes % 1024 == 0, "SWIZZLE_128B atoms are 1024 B");
constexpr int kFABytes = kFKp * kFChunkBytes;    // 180 KB
constexpr int kFWStages = 4;
constexpr int kFWStage = 64 * 128;                // one kernel point of W: [64 rows (hi / lo of 32 channels)] x 128 B

struct FusedSmem {
  static constexpr int kWBytes = kFWStages * kFWStage;
  static constexpr int kBarOff = kFABytes + kWBytes;                  // mbarriers
  static constexpr int kNumBars = 8 + 2 * kFWStages;
  static constexpr int kCtrOff = kBarOff + kNumBars * 8;             // the row counter and the consumed counter
  static constexpr int kTotal = kCtrOff + 16 + 1024 /*alignment slack*/;
  static_assert(kTotal <= 232448, "shared memory budget of an SM (227 KB)");
};

struct FusedParams {
  const float* q;            // [Nq,3]
  const float4* s4;          // [Ns+1] (x, y, z, flag), entry Ns = shadow point
  const int* idx;            // [Nq,H]
  const float* feat;         // [Ns,32]
  const float* Kp;           // [15,3]
  const float* Wp;           // 15 images of [64][32] floats (pack_weight_fused32_kernel)
  int Nq, Ns, H, Cout, Npad;
  float inv_scale;           // 1 / (2 extent)  (:215)
  int count_nn;
  const float* bn_scale; const float* bn_shift; const float* bias;
  float leaky_alpha;
  float* out;                // [Nq,Cout]
  const int* nq_dev;         // optional: actual query / support counts in device memory (Nq / Ns are capacities)
  const int* ns_dev;
  int dbg;                   // D3F_FUSED_DBG (experiments): bit 0 = static row assignment
};

__device__ __forceinline__ void mma_tf32_1688(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// hi = x rounded to nearest TF32 (low 13 mantissa bits zero), lo = x - hi exactly
__device__ __forceinline__ void split_hl(float x, unsigned& hi, unsigned& lo) {
  hi = (__float_as_uint(x) + 0x1000u) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}
__device__ __forceinline__ float sqrt_apx(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));   // .ftz: no denormal rescue around the MUFU
  return r;
}

// mbarrier wait that backs off: a spinning warp would otherwise steal issue slots from the warps doing the work
__device__ __forceinline__ void mbar_wait_sleep(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  for (;;) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    __nanosleep(128);
  }
}

// position of a gather warp in its stream of (tile, query slot, 8-neighbour step)
// (rows are handed out dynamically: rowg = k * 48 + row counts the rows of this CTA's tile sequence)
struct Pos {
  int rowg, s;
};

struct StepIds {
  int ida, idb;
};
struct StepData {
  float4 spa, spb, fa, fb;
  bool reala, realb;
};

}  // namespace

__global__ void __launch_bounds__(kFThreads, 1) kpconv_fused32_kernel(FusedParams pin) {
  FusedParams p = pin;
  p.Nq = dyn_rows(pin.Nq, pin.nq_dev);
  p.Ns = dyn_rows(pin.Ns, pin.ns_dev);
  using S_ = FusedSmem;
  constexpr int kWS = kFWStages;
  extern __shared__ uint8_t fused_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)fused_smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  uint64_t* bars = (uint64_t*)(smem + S_::kBarOff);
  // bars: 0 a_full (all lanes of the warps that wrote the tile's rows), 8.. w_full[kWS], then w_empty[kWS]
  const uint32_t bar_a_full = smem_u32(&bars[0]);
  constexpr int kWB = 8;   // first W barrier
  int* row_ctr = (int*)(smem + S_::kCtrOff);       // next row of this CTA's tile sequence (gather warps)
  // number of this CTA's tiles whose MMAs have retired. A plain counter, not an mbarrier: a gather warp may skip several
  // tiles (its rows are taken by the others), and a parity wait on a barrier that is two or more phases ahead waits for
  // a FUTURE phase -- with the warp's own row part of that future tile, a deadlock.
  int* consumed = (int*)(smem + S_::kCtrOff + 4);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles = ceil_div(p.Nq, kFRows);
  const int tstride = gridDim.x;

  int my_tiles = 0;
  for (int tl = blockIdx.x; tl < tiles; tl += tstride) ++my_tiles;
  if (tid == 0) {
    *row_ctr = 0;
    *consumed = 0;
    mbar_init(bar_a_full, kFRows * 32);              // every lane of the warp that produced a row arrives for it
    for (int s = 0; s < kWS; ++s) {
      mbar_init(smem_u32(&bars[kWB + s]), 1);
      mbar_init(smem_u32(&bars[kWB + kWS + s]), 4);  // one arrive per warp of the MMA warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < kFGatherWarps) {
    // =========================== gather / stage-1 warps ==================================================
    const int g = lane >> 2, t = lane & 3;
    const int S = (p.H + 7) >> 3;
    const int kA = g, kB = g + 8;
    const bool validB = kB < kFKp;
    const float kax = p.Kp[3 * kA], kay = p.Kp[3 * kA + 1], kaz = p.Kp[3 * kA + 2];
    const float kbx = validB ? p.Kp[3 * kB] : 0.f, kby = validB ? p.Kp[3 * kB + 1] : 0.f,
                kbz = validB ? p.Kp[3 * kB + 2] : 0.f;
    const float* fcol = p.feat + 4 * g;      // lane (g, t): channels [4g, 4g+4) of its neighbours' rows

    // Rows are handed out one at a time from a shared counter: a warp takes its next row two steps before it finishes
    // the current one: with a static split (3 rows per warp and tile) every warp would wait for the slowest one at
    // every tile.
    const int total_rows = my_tiles * kFRows;
    int static_next = warp;
    auto grab = [&]() {
      if (p.dbg & 1) {                       // experiment: warp w takes rows w, w + 16, ...
        const int r = static_next;
        static_next += kFGatherWarps;
        return r;
      }
      int r = 0;
      if (lane == 0) r = atomicAdd(row_ctr, 1);
      return __shfl_sync(0xffffffffu, r, 0);
    };
    auto advance = [&](Pos& ps) {
      if (++ps.s == S) {
        ps.s = 0;
        ps.rowg = grab();
      }
    };
    auto valid = [&](const Pos& ps) { return ps.rowg < total_rows; };
    auto query_of = [&](const Pos& ps) {
      const int k = ps.rowg / kFRows;
      return ((int)blockIdx.x + k * tstride) * kFRows + (ps.rowg - k * kFRows);
    };
    auto load_ids = [&](const Pos& ps, StepIds& o) {
      const int n = query_of(ps);
      o.ida = p.Ns;
      o.idb = p.Ns;
      if (valid(ps) && n < p.Nq) {
        const int* row = p.idx + (size_t)n * p.H;
        const int ha = 8 * ps.s + t, hb = ha + 4;
        if (ha < p.H) o.ida = __ldg(row + ha);
        if (hb < p.H) o.idb = __ldg(row + hb);
      }
    };
    auto load_data = [&](StepIds ids, StepData& o) {
      int ida = ids.ida, idb = ids.idb;
      if (ida < 0 || ida > p.Ns) ida = p.Ns;      // -1 padding of the non-batch op behaves like the shadow
      if (idb < 0 || idb > p.Ns) idb = p.Ns;
      o.reala = ida < p.Ns;
      o.realb = idb < p.Ns;
      o.spa = __ldg(&p.s4[ida]);
      o.spb = __ldg(&p.s4[idb]);
      o.fa = o.reala ? __ldg(reinterpret_cast<const float4*>(fcol + (size_t)ida * 32)) : make_float4(0.f, 0.f, 0.f, 0.f);
      o.fb = o.realb ? __ldg(reinterpret_cast<const float4*>(fcol + (size_t)idb * 32)) : make_float4(0.f, 0.f, 0.f, 0.f);
    };

    Pos cur{grab(), 0}, p1 = cur, p2 = cur;
    advance(p1);
    p2 = p1;
    advance(p2);
    // Two register sets, used alternately (no copies between iterations: a register move of a loaded value would
    // wait for the load and expose the full L2 latency every step): dA / dB hold the data of the current / next
    // step, iA / iB the neighbour ids of the step after that.
    StepIds iA, iB;
    StepData dA, dB;
    {
      StepIds ids0;
      load_ids(cur, ids0);
      load_ids(p1, iB);
      load_data(ids0, dA);
    }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    int nn_count = 0;
    int waited_k = 0;                  // tiles [0, waited_k) of this CTA are known to have been consumed by the MMAs
    float qx = 0.f, qy = 0.f, qz = 0.f;
    {
      const int n = query_of(cur);
      if (valid(cur) && n < p.Nq) { qx = p.q[3 * (size_t)n]; qy = p.q[3 * (size_t)n + 1]; qz = p.q[3 * (size_t)n + 2]; }
    }

    // one 8-neighbour step: `d0` = this step's data, `d1` receives the next step's data (ids `i1`, loaded an iteration
    // ago), `i2` receives the ids of the step after that
    auto step = [&](const StepData& d0, StepData& d1, const StepIds& i1, StepIds& i2) {
      load_data(i1, d1);
      load_ids(p2, i2);
      // last step of a query: fetch the next query's coordinates now, under this step's math
      float nqx = 0.f, nqy = 0.f, nqz = 0.f;
      if (cur.s == S - 1) {
        const int nn = query_of(p1);
        if (valid(p1) && nn < p.Nq) { nqx = p.q[3 * (size_t)nn]; nqy = p.q[3 * (size_t)nn + 1]; nqz = p.q[3 * (size_t)nn + 2]; }
      }

      // ---- correlation weights of 2 neighbours x 2 kernel points per lane, wf += w^T . f ----------------------
      {
        const float rax = d0.spa.x - qx, ray = d0.spa.y - qy, raz = d0.spa.z - qz;
        const float rbx = d0.spb.x - qx, rby = d0.spb.y - qy, rbz = d0.spb.z - qz;
        const float d_aA = (rax - kax) * (rax - kax) + (ray - kay) * (ray - kay) + (raz - kaz) * (raz - kaz);
        const float d_aB = (rax - kbx) * (rax - kbx) + (ray - kby) * (ray - kby) + (raz - kbz) * (raz - kbz);
        const float d_bA = (rbx - kax) * (rbx - kax) + (rby - kay) * (rby - kay) + (rbz - kaz) * (rbz - kaz);
        const float d_bB = (rbx - kbx) * (rbx - kbx) + (rby - kby) * (rby - kby) + (rbz - kbz) * (rbz - kbz);
        // linear influence, 1 - d / (2 extent) clipped at 0 (:213-216); shadow / dropped neighbours weigh 0
        float w_aA = fmaxf(1.f - sqrt_apx(d_aA + 1e-10f) * p.inv_scale, 0.f);
        float w_aB = validB ? fmaxf(1.f - sqrt_apx(d_aB + 1e-10f) * p.inv_scale, 0.f) : 0.f;
        float w_bA = fmaxf(1.f - sqrt_apx(d_bA + 1e-10f) * p.inv_scale, 0.f);
        float w_bB = validB ? fmaxf(1.f - sqrt_apx(d_bB + 1e-10f) * p.inv_scale, 0.f) : 0.f;
        if (!d0.reala) { w_aA = 0.f; w_aB = 0.f; }
        if (!d0.realb) { w_bA = 0.f; w_bB = 0.f; }
        if (p.count_nn)   // lanes 0..3 (g == 0) cover the eight neighbours of this step once (:249-253)
          nn_count += __popc(__ballot_sync(0xffffffffu, d0.spa.w > 0.f) & 0xFu) +
                      __popc(__ballot_sync(0xffffffffu, d0.spb.w > 0.f) & 0xFu);
        unsigned ah[4], al[4];
        split_hl(w_aA, ah[0], al[0]);
        split_hl(w_aB, ah[1], al[1]);
        split_hl(w_bA, ah[2], al[2]);
        split_hl(w_bB, ah[3], al[3]);
        const float fa[4] = {d0.fa.x, d0.fa.y, d0.fa.z, d0.fa.w};
        const float fb[4] = {d0.fb.x, d0.fb.y, d0.fb.z, d0.fb.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          unsigned bh0, bl0, bh1, bl1;
          split_hl(fa[i], bh0, bl0);
          split_hl(fb[i], bh1, bl1);
          mma_tf32_1688(acc[i], ah, bh0, bh1);
          mma_tf32_1688(acc[i], al, bh0, bh1);
          mma_tf32_1688(acc[i], ah, bl0, bl1);
        }
      }

      // ---- end of a query: its wf row goes into the A operand --------------------------------------------------
      if (cur.s == S - 1) {
        const int k = cur.rowg / kFRows, row = cur.rowg - k * kFRows;
        while (waited_k < k) {             // the wf tile was last read by the MMAs of tile k - 1
          int c;
          asm volatile("ld.acquire.cta.shared.b32 %0, [%1];" : "=r"(c) : "r"(smem_u32(consumed)) : "memory");
          waited_k = c;
          if (waited_k < k) __nanosleep(128);
        }
        // lane (g, t) holds kernel points {g, g+8} x channels [8t, 8t+8): column j of n-tile i is channel 4j + i, so
        // (acc[0..3][0]) = channels 8t..8t+3 = 16-byte chunk 2t of the row, (acc[0..3][1]) = chunk 2t+1
        const uint32_t roff = (uint32_t)row * 128u;
        const uint32_t c0 = (uint32_t)(((2 * t) ^ (row & 7)) << 4), c1 = (uint32_t)(((2 * t + 1) ^ (row & 7)) << 4);
        // even g writes chunk 2t first, odd g chunk 2t+1: the 32 lanes of one store then cover 8 distinct bank groups
        const bool swap = (g & 1) != 0;
        // D3Feat's density normalisation (:249-253) is applied to the wf row itself: (sum_k wf_k W_k) / nn ==
        // sum_k (wf_k / nn) W_k, so nothing but the A operand travels from the gather warps to the contraction
        const float inv_nn = p.count_nn ? 1.f / (float)max(nn_count, 1) : 1.f;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int kp = half == 0 ? kA : kB;
          if (half == 1 && !validB) break;
          const uint32_t hi_addr = sbase + (uint32_t)kp * kFChunkBytes + roff;
          const uint32_t lo_addr = hi_addr + kFImageBytes;   // lo rows follow the 48 hi rows of the same kernel point
          const int e0 = half * 2, e1 = half * 2 + 1;
          float4 h0, l0, h1, l1;
          {
            unsigned a, b;
            split_hl(acc[0][e0] * inv_nn, a, b); h0.x = __uint_as_float(a); l0.x = __uint_as_float(b);
            split_hl(acc[1][e0] * inv_nn, a, b); h0.y = __uint_as_float(a); l0.y = __uint_as_float(b);
            split_hl(acc[2][e0] * inv_nn, a, b); h0.z = __uint_as_float(a); l0.z = __uint_as_float(b);
            split_hl(acc[3][e0] * inv_nn, a, b); h0.w = __uint_as_float(a); l0.w = __uint_as_float(b);
            split_hl(acc[0][e1] * inv_nn, a, b); h1.x = __uint_as_float(a); l1.x = __uint_as_float(b);
            split_hl(acc[1][e1] * inv_nn, a, b); h1.y = __uint_as_float(a); l1.y = __uint_as_float(b);
            split_hl(acc[2][e1] * inv_nn, a, b); h1.z = __uint_as_float(a); l1.z = __uint_as_float(b);
            split_hl(acc[3][e1] * inv_nn, a, b); h1.w = __uint_as_float(a); l1.w = __uint_as_float(b);
          }
          sts128(hi_addr + (swap ? c1 : c0), swap ? h1 : h0);
          sts128(hi_addr + (swap ? c0 : c1), swap ? h0 : h1);
          sts128(lo_addr + (swap ? c1 : c0), swap ? l1 : l0);
          sts128(lo_addr + (swap ? c0 : c1), swap ? l0 : l1);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
        nn_count = 0;
        fence_proxy_async();                // generic-proxy writes -> visible to the tensor core (async proxy)
        mbar_arrive(bar_a_full);            // 32 arrivals per row, kFRows rows per phase
        qx = nqx; qy = nqy; qz = nqz;     // coordinates of the next query
      }
      cur = p1;
      p1 = p2;
      advance(p2);
    };

    while (valid(cur)) {
      step(dA, dB, iB, iA);
      if (!valid(cur)) break;
      step(dB, dA, iA, iB);
    }
  } else if (warp == kFCtrlWarp) {
    // =========================== control thread: W ring producer ===================================================
    // The W image of every kernel point of every tile, in the order the MMA warpgroup consumes them.
    if (lane == 0) {
      const int total_chunks = my_tiles * kFKp;
      for (int pc = 0; pc < total_chunks; ++pc) {
        const int st = pc % kWS;
        if (pc >= kWS) mbar_wait_sleep(smem_u32(&bars[kWB + kWS + st]), (uint32_t)((pc / kWS - 1) & 1));
        const uint32_t full = smem_u32(&bars[kWB + st]);
        mbar_arrive_expect_tx(full, (uint32_t)kFWStage);
        tma_bulk_g2s(sbase + kFABytes + (uint32_t)st * kFWStage, p.Wp + (size_t)(pc % kFKp) * (kFWStage / 4),
                     (uint32_t)kFWStage, full);
      }
    }
  } else {
    // =========================== MMA warpgroup (warps 16..19): contraction + epilogue ==============================
    // Swapped orientation: D^T[64 x 96] = Wimg[64 x 32ch] . [wf_hi(48 rows) | wf_lo(48 rows)]^T per kernel point and
    // K = 8 step. The 64 rows of a W image are the 32 output channels twice (TF32-hi and the exact remainder, 8 + 8 per
    // 16-row slab of a warp), the 96 operand rows are the tile's queries twice (hi and lo of their wf), so ONE wgmma
    // yields Wh.wf_hi, Wl.wf_hi, Wh.wf_lo (and the negligible Wl.wf_lo): 60 wgmmas per 48 queries. The gather warps are
    // already writing the next tile's rows while this warpgroup runs the epilogue.
    const int qd = warp - kFEpiWarp0;
    // accumulator fragment (tc_common.cuh): rows 16 qd + lane / 4 (Wh of channel co) and + 8 (Wl of channel co),
    // columns 8 j + 2 (lane % 4) + e: query 8 j + 2 (lane % 4) + e against wf_hi for j < 6, against wf_lo for j >= 6
    const int co = 8 * qd + (lane >> 2);
    const float e_sc = p.bn_scale ? p.bn_scale[co] : 1.f, e_sh = p.bn_scale ? p.bn_shift[co] : 0.f;
    const float e_bi = p.bias ? p.bias[co] : 0.f;
    float acc[48];
    int it = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += tstride, ++it) {
      mbar_wait_sleep(bar_a_full, (uint32_t)(it & 1));          // all 48 rows of the tile are in shared memory
#pragma unroll
      for (int j = 0; j < 48; ++j) acc[j] = 0.f;
      for (int kp = 0; kp < kFKp; ++kp) {
        const int c = it * kFKp + kp;
        const int st = c % kWS;
        mbar_wait(smem_u32(&bars[kWB + st]), (uint32_t)((c / kWS) & 1));
        wgmma_fence();
        const uint64_t dw = make_smem_desc(sbase + kFABytes + (uint32_t)st * kFWStage);
        const uint64_t df = make_smem_desc(sbase + (uint32_t)kp * kFChunkBytes);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint64_t adv = (uint64_t)((j * 32) >> 4);   // +32 B per K = 8 step inside the swizzle atom
          wgmma_tf32<96>(acc, dw + adv, df + adv);
        }
        wgmma_commit();
        if (kp > 0) {                                          // the previous kernel point's W stage is free
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(smem_u32(&bars[kWB + kWS + (c - 1) % kWS]));
        }
      }
      wgmma_wait<0>();
      wgmma_reg_fence<48>(acc);
      if (lane == 0) mbar_arrive(smem_u32(&bars[kWB + kWS + (it * kFKp + kFKp - 1) % kWS]));
      asm volatile("bar.sync 1, 128;" ::: "memory");          // every warp's wgmmas of this tile have retired
      if (qd == 0 && lane == 0)   // the wf tile may be overwritten
        asm volatile("st.release.cta.shared.b32 [%0], %1;" ::"r"(smem_u32(consumed)), "r"(it + 1) : "memory");
#pragma unroll
      for (int j = 0; j < 6; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float x = (acc[4 * j + e] + acc[4 * j + 2 + e]) + (acc[4 * (j + 6) + e] + acc[4 * (j + 6) + 2 + e]);
          const int n = tile * kFRows + 8 * j + 2 * (lane & 3) + e;
          if (n < p.Nq) {
            x = fmaf(x, e_sc, e_sh) + e_bi;
            if (p.leaky_alpha >= 0.f) x = x > 0.f ? x : x * p.leaky_alpha;
            p.out[(size_t)n * 32 + co] = x;
          }
        }
      }
    }
  }
}

// W[15][32][32] (K_values of a 32 -> 32 KPConv) -> 15 shared-memory images of [64 rows][32 channels]: row r of quadrant
// qd = r / 16 holds output channel 8 qd + (r % 8), rows with (r % 16) < 8 its TF32-rounded value, the others the exact
// remainder; K-major SWIZZLE_128B (16-byte chunks XOR-ed with r % 8), i.e. ready to be dropped into an SM by one TMA
// bulk copy and read by the wgmma descriptor.
__global__ void __launch_bounds__(256) pack_weight_fused32_kernel(const float* __restrict__ W, float* __restrict__ img) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kFKp * 64 * 32) return;
  const int kp = i / (64 * 32), r = (i / 32) % 64, c = i % 32;
  const int qd = r >> 4, part = (r >> 3) & 1, co = 8 * qd + (r & 7);
  const float x = W[((size_t)kp * 32 + c) * 32 + co];
  unsigned hi, lo;
  split_hl(x, hi, lo);
  const size_t off = (size_t)kp * 64 * 32 + (size_t)r * 32 + (size_t)((((c >> 2) ^ (r & 7)) << 2) | (c & 3));
  img[off] = __uint_as_float(part == 0 ? hi : lo);
}

// The fused kernel covers the D3Feat configuration of the Cin = 32 layers: K = 15 kernel points, linear influence, sum
// aggregation, Cout = 32, 16-byte aligned features, and enough queries to fill the GPU.
bool kpconv_fused_supported(int Nq, int H, int K, int Cin, int Cout, int influence, int mode, const float* feat,
                            const float* W, const float* out, const int* query_order) {
  // D3F_FUSED_KPCONV=1 selects this kernel. Default off: a persistent 227 KB-per-SM CTA leaves no room for the
  // pyramid kernels of the next batch that the two-stream pipeline overlaps with the encoder.
  const char* v = getenv("D3F_FUSED_KPCONV");
  if (v == nullptr || v[0] != '1') return false;
  return H >= 1 && K == kFKp && Cin == 32 && Cout == 32 && influence == D3F_INFLUENCE_LINEAR &&
         mode == D3F_MODE_SUM && W != nullptr && query_order == nullptr && Nq >= kFRows * kNumSMs / 2 &&
         (reinterpret_cast<uintptr_t>(feat) & 15) == 0 && out != nullptr;
}

size_t kpconv_fused_image_floats() { return (size_t)kFKp * kFWStage / sizeof(float); }

int kpconv_fused_forward(const float* q, const float4* s4, const int* idx, const float* feat, const float* Kp,
                         const float* W, float* w_img, int Nq, int Ns, int H, int Cout, float extent, int normalize,
                         const float* bn_scale, const float* bn_shift, const float* bias, float leaky_alpha, float* out,
                         cudaStream_t stream, const int* nq_dev, const int* ns_dev) {
  D3F_REQUIRE(Cout == 32 && w_img != nullptr, D3F_ERR_INVALID, "kpconv_fused: Cout=%d / missing image buffer", Cout);
  pack_weight_fused32_kernel<<<ceil_div(kFKp * 64 * 32, 256), 256, 0, stream>>>(W, w_img);
  D3F_LAUNCH_CHECK("pack_weight_fused32_kernel");
  FusedParams p;
  p.q = q; p.s4 = s4; p.idx = idx; p.feat = feat; p.Kp = Kp; p.Wp = w_img;
  p.Nq = Nq; p.Ns = Ns; p.H = H; p.Cout = Cout; p.Npad = 32;
  p.inv_scale = 1.f / (2.f * extent);
  p.count_nn = normalize ? 1 : 0;
  p.bn_scale = bn_scale; p.bn_shift = bn_shift; p.bias = bias; p.leaky_alpha = leaky_alpha;
  p.out = out;
  p.nq_dev = nq_dev; p.ns_dev = ns_dev;
  const char* dbg = getenv("D3F_FUSED_DBG");
  p.dbg = dbg ? atoi(dbg) : 0;
  static bool configured = false;
  if (!configured) {
    D3F_CUDA(cudaFuncSetAttribute(kpconv_fused32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FusedSmem::kTotal));
    configured = true;
  }
  const int tiles = ceil_div(Nq, kFRows);
  const int grid = tiles < kNumSMs ? tiles : kNumSMs;
  kpconv_fused32_kernel<<<grid, kFThreads, FusedSmem::kTotal, stream>>>(p);
  D3F_LAUNCH_CHECK("kpconv_fused32_kernel");
  return D3F_OK;
}

}  // namespace d3f

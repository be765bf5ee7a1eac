// Radius neighbours on a sort-based hash grid over the supports (cell edge = radius * 1.001, 27-cell scan,
// the three x-adjacent cells of a row are one contiguous run in the sorted order => 9 runs per query).
//
// Reference semantics (tf_custom_ops/tf_neighbors/neighbors/neighbors.cpp:211-332, nanoflann.hpp:249-253,
// 432-440, 1280-1289): every support of the same cloud with d2 < r2, d2 = ((dx*dx)+dy*dy)+dz*dz evaluated in
// fp32 with separately rounded mul/add (__fmul_rn/__fadd_rn: nvcc would otherwise contract to FMA),
// r2 = radius*radius in fp32, rows ascending in (d2, index), padded with pad_value.
//
// The 27-cell scan is provably complete only while every grid axis has at most kMaxScanAxisCells = 4096 cells (the
// derivation is beside make_grid, nbgrid.cuh): about 307 m at the 3DMatch level-0 radius 0.075, 3 km at KITTI's 0.75.
// Longer grids are refused on the host with D3F_ERR_INVALID before any launch, like the fp64 lookup of icp.cu.
#include <stdlib.h>

#include "nbgrid.cuh"
#include "ops.cuh"
#include "sort.cuh"

namespace d3f {

// Grid build = counting sort by cell: (1) count points per cell, (2) exclusive scan -> cell_start (cell c owns
// [cell_start[c], cell_start[c+1])), (3) scatter. The order of the points INSIDE a cell is whatever the atomics give;
// no result depends on it (rows are emitted in (d2, index) order). Supports at or past start[B] belong to no cloud and
// enter no cell.
__global__ void __launch_bounds__(256)
cell_count_kernel(const float* __restrict__ s, int Ns_cap, const int* __restrict__ ns_dev,
                  const int* __restrict__ start, int B, NbGrid g, uint32_t* __restrict__ cell_id,
                  int* __restrict__ cell_cnt) {
  const int Ns = cloud_rows(Ns_cap, ns_dev, start, B);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Ns) return;
  int b = batch_of(start, B, i);
  int cx = cell_coord(s[3 * (size_t)i], g.minx, g.inv_cell, g.nx);
  int cy = cell_coord(s[3 * (size_t)i + 1], g.miny, g.inv_cell, g.ny);
  int cz = cell_coord(s[3 * (size_t)i + 2], g.minz, g.inv_cell, g.nz);
  uint32_t c = (uint32_t)((long long)b * g.ncells + ((long long)cz * g.ny + cy) * g.nx + cx);
  cell_id[i] = c;
  atomicAdd(&cell_cnt[c], 1);
}

// sorted_pts[pos] = (x, y, z, bits(index)); cell_cnt is counted back down to zero. A support of no cloud keeps its own
// position, past every cell's run, so that the cell order stays a permutation of the rows.
__global__ void __launch_bounds__(256)
cell_scatter_kernel(const float* __restrict__ s, int Ns_cap, const int* __restrict__ ns_dev,
                    const int* __restrict__ start, int B, const uint32_t* __restrict__ cell_id,
                    const int* __restrict__ cell_start, int* __restrict__ cell_cnt, float4* __restrict__ sorted_pts) {
  const int Ns = dyn_rows(Ns_cap, ns_dev);
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Ns) return;
  const int pos = i < start[B] ? cell_start[cell_id[i]] + atomicSub(&cell_cnt[cell_id[i]], 1) - 1 : i;
  sorted_pts[pos] = make_float4(s[3 * (size_t)i], s[3 * (size_t)i + 1], s[3 * (size_t)i + 2], __uint_as_float((uint32_t)i));
}

__global__ void __launch_bounds__(256)
cell_order_kernel(const float4* __restrict__ sorted_pts, int Ns, int* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Ns) out[i] = (int)__float_as_uint(sorted_pts[i].w);
}

struct NbWs {
  uint32_t* cell_id;  // [Ns] cell of every support
  int* s_start;       // [B+1]
  int* q_start;       // [B+1] (count / fill)
  float4* sorted_pts;
  int* cell_start;    // [cells + 1]; the run of cell c is [cell_start[c], cell_start[c + 1])
  int* cell_cnt;      // [cells + 1] build-time counters
  int* scan_scratch;
};

// The workspace of a grid over Ns supports at `radius`, or 0 for a grid the search refuses.
static size_t nb_layout(int Ns, int B, float radius, const float* host_bbox, void* base, NbWs* w_out) {
  if (host_bbox == nullptr || !(radius > 0.f) || B < 1) return 0;
  const NbGrid g = make_grid(host_bbox, radius);
  const long long total_cells = g.ncells * B;
  if (total_cells > kMaxGridCells || !radius_scan_complete(g)) return 0;
  int n = Ns > 0 ? Ns : 1;
  Carver cv(base);
  NbWs w;
  w.cell_id = cv.take<uint32_t>(n);
  w.s_start = cv.take<int>(B + 1);
  w.q_start = cv.take<int>(B + 1);
  w.sorted_pts = cv.take<float4>(n);
  w.cell_start = cv.take<int>((size_t)total_cells + 1);
  w.cell_cnt = cv.take<int>((size_t)total_cells + 1);
  w.scan_scratch = cv.take<int>((size_t)scan_num_blocks((int)total_cells) + 1);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

int radius_neighbors_build(const float* supports, const int* s_batch_len, int B, int Ns, float radius,
                           const float* host_bbox, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                           const int* ns_dev, const int* s_start_pre) {
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "radius_neighbors: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(radius > 0.f && Ns >= 0 && host_bbox != nullptr, D3F_ERR_INVALID,
              "radius_neighbors: radius=%g Ns=%d invalid or host_bbox missing", (double)radius, Ns);
  NbGrid g = make_grid(host_bbox, radius);
  long long total = g.ncells * B;
  D3F_REQUIRE(total <= kMaxGridCells, D3F_ERR_CAPACITY,
              "radius_neighbors: grid %d x %d x %d x %d clouds exceeds %lld cells", g.nx, g.ny, g.nz, B,
              kMaxGridCells);
  D3F_REQUIRE(radius_scan_complete(g), D3F_ERR_INVALID,
              "radius_neighbors: grid %d x %d x %d has an axis longer than %d cells (of radius * 1.001)", g.nx, g.ny,
              g.nz, kMaxScanAxisCells);
  NbWs w;
  const size_t need = nb_layout(Ns, B, radius, host_bbox, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "radius_neighbors: workspace too small");
  if (s_start_pre != nullptr) w.s_start = const_cast<int*>(s_start_pre);   // the caller already scanned these lengths
  else if (launch_batch_start(s_batch_len, B, w.s_start, stream)) return D3F_ERR_CUDA;
  D3F_CUDA(cudaMemsetAsync(w.cell_cnt, 0, sizeof(int) * ((size_t)total + 1), stream));
  if (Ns == 0) {
    D3F_CUDA(cudaMemsetAsync(w.cell_start, 0, sizeof(int) * ((size_t)total + 1), stream));
    return D3F_OK;
  }
  cell_count_kernel<<<ceil_div(Ns, 256), 256, 0, stream>>>(supports, Ns, ns_dev, w.s_start, B, g, w.cell_id, w.cell_cnt);
  D3F_LAUNCH_CHECK("cell_count_kernel");
  if (exclusive_scan_i32(w.cell_cnt, w.cell_start, (int)total, w.cell_start + total, w.scan_scratch, stream))
    return D3F_ERR_CUDA;
  cell_scatter_kernel<<<ceil_div(Ns, 256), 256, 0, stream>>>(supports, Ns, ns_dev, w.s_start, B, w.cell_id, w.cell_start,
                                                             w.cell_cnt, w.sorted_pts);
  D3F_LAUNCH_CHECK("cell_scatter_kernel");
  return D3F_OK;
}

// The built grid of a workspace, for queries outside this file (nearest_in_cloud in nbgrid.cuh).
int radius_neighbors_view(const void* workspace, int Ns, int B, float radius, const float* host_bbox, NbView* out) {
  D3F_REQUIRE(B >= 1 && radius > 0.f && host_bbox != nullptr && out != nullptr, D3F_ERR_INVALID,
              "radius_neighbors_view: bad arguments");
  NbGrid g = make_grid(host_bbox, radius);
  long long total = g.ncells * B;
  D3F_REQUIRE(total <= kMaxGridCells, D3F_ERR_CAPACITY, "radius_neighbors: grid too large");
  // as in d3f_radius_neighbors_order: no grid of these arguments can have been built
  NbWs w;
  D3F_REQUIRE(nb_layout(Ns, B, radius, host_bbox, const_cast<void*>(workspace), &w) > 0, D3F_ERR_INVALID,
              "radius_neighbors_view: no grid of these arguments can be built");
  out->g = g;
  out->sorted_pts = w.sorted_pts;
  out->cell_start = w.cell_start;
  return D3F_OK;
}

// ---------------------------------------------------------------------------------------------------
constexpr int kNbWarps = 8;      // warps (= queries in flight) per CTA
constexpr int kNbListCap = 512;  // hits kept in shared memory per query before the generic path

struct Hit {
  float d2;
  int idx;
};

__device__ __forceinline__ bool hit_less(float da, int ia, float db, int ib) {
  return da < db || (da == db && ia < ib);
}

__device__ __forceinline__ float sq_dist_rn(float qx, float qy, float qz, float4 s) {
  float dx = __fsub_rn(qx, s.x), dy = __fsub_rn(qy, s.y), dz = __fsub_rn(qz, s.z);
  float r = __fmul_rn(dx, dx);
  r = __fadd_rn(r, __fmul_rn(dy, dy));
  r = __fadd_rn(r, __fmul_rn(dz, dz));
  return r;
}

// One block size K of a 64-element bitonic sort of unique 32-bit keys, elements 2*lane and 2*lane+1 in one lane:
// the exchanges at distance j >= 2 pair lane with lane ^ (j/2), the one at distance 1 stays inside the lane.
template <int K>
__device__ __forceinline__ void bitonic_block2(unsigned& ka, unsigned& kb, int lane) {
  const bool asc = K == 64 || (lane & (K >> 1)) == 0;      // direction of the block elements 2*lane, 2*lane+1 sit in
#pragma unroll
  for (int j = K >> 1; j >= 2; j >>= 1) {
    const unsigned oa = __shfl_xor_sync(0xffffffffu, ka, j >> 1), ob = __shfl_xor_sync(0xffffffffu, kb, j >> 1);
    const bool keep_min = ((lane & (j >> 1)) == 0) == asc;
    ka = keep_min ? min(ka, oa) : max(ka, oa);
    kb = keep_min ? min(kb, ob) : max(kb, ob);
  }
  const unsigned lo = min(ka, kb), hi = max(ka, kb);
  ka = asc ? lo : hi;
  kb = asc ? hi : lo;
}

// FILL = false: counts only. FILL = true: sorted rows.
template <bool FILL>
__global__ void __launch_bounds__(kNbWarps * 32)
radius_query_kernel(const float* __restrict__ q, int Nq_cap, const int* __restrict__ nq_dev,
                    const int* __restrict__ q_start, int B, NbGrid g, const float4* __restrict__ sorted_pts,
                    const int* __restrict__ cell_start, float r2, int cols, int pad_value_in,
                    const int* __restrict__ pad_dev, int* __restrict__ counts, int* __restrict__ out_max,
                    int* __restrict__ out_idx) {
  const int Nq = dyn_rows(Nq_cap, nq_dev);
  const int pad_value = pad_dev ? __ldg(pad_dev) : pad_value_in;   // the shadow index = number of supports (device)
  // per query: the 9 runs as (end of the run in the concatenated candidate numbering, sorted_pts offset of the run
  // minus its start in that numbering): candidate t of run r is sorted_pts[t + adj[r]]
  __shared__ int2 run_tab[kNbWarps][10];
  __shared__ Hit list[FILL ? kNbWarps : 1][FILL ? kNbListCap : 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int qi = blockIdx.x * kNbWarps + warp;
  if (qi >= Nq) return;  // warp-uniform
  const float qx = q[3 * (size_t)qi], qy = q[3 * (size_t)qi + 1], qz = q[3 * (size_t)qi + 2];
  int b;
  if (B <= 32) {   // largest b with q_start[b] <= qi: one load per lane and a vote instead of a dependent search
    const bool le = lane < B && __ldg(q_start + lane) <= qi;
    b = max(__popc(__ballot_sync(0xffffffffu, le)) - 1, 0);
  } else {
    b = batch_of(q_start, B, qi);
  }
  const int cx = cell_coord(qx, g.minx, g.inv_cell, g.nx);
  const int cy = cell_coord(qy, g.miny, g.inv_cell, g.ny);
  const int cz = cell_coord(qz, g.minz, g.inv_cell, g.nz);

  // lanes 0..8: one (dy,dz) row each -> contiguous run over cells cx-1..cx+1. The whole table holds at most
  // kMaxGridCells = 2^27 cells (checked on the host), so 32-bit cell numbers are exact.
  int rs = 0, rl = 0;
  if (lane < 9) {
    const int dz = (lane * 11) >> 5;            // lane / 3 for lane < 9
    const int yy = cy + (lane - 3 * dz) - 1, zz = cz + dz - 1;
    if (yy >= 0 && yy < g.ny && zz >= 0 && zz < g.nz) {
      const int row = b * (int)g.ncells + (zz * g.ny + yy) * g.nx;
      const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.nx - 1);
      // cells x0..x1 of one (y, z) row are adjacent in the table: one contiguous run of sorted_pts
      const int s = __ldg(cell_start + row + x0), e = __ldg(cell_start + row + x1 + 1);
      if (e > s) {
        rs = s;
        rl = e - s;
      }
    }
  }
  int inc = rl;
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane < 9) run_tab[warp][lane] = make_int2(inc, rs - (inc - rl));
  int T = __shfl_sync(0xffffffffu, inc, 8);
  if (qi >= __ldg(q_start + B)) T = 0;   // a query of no cloud: no neighbours, a row of padding
  if (lane == 9) run_tab[warp][9] = make_int2(0x7fffffff, 0);   // sentinel: the walk below never runs off the table
  __syncwarp();

  int n = 0;
  // each lane walks the concatenated runs with stride 32, so its run only moves forward (empty runs are skipped)
  const int2* tp = &run_tab[warp][0];
  int2 cur = *tp;
  const unsigned below = (1u << lane) - 1u;
  for (int t0 = 0; t0 < T; t0 += 32) {
    const int t = t0 + lane;
    bool hit = false;
    float d2 = 0.f;
    int sidx = 0;
    if (t < T) {
      while (t >= cur.x) cur = *++tp;
      const float4 sp = __ldg(sorted_pts + (t + cur.y));
      d2 = sq_dist_rn(qx, qy, qz, sp);
      sidx = (int)__float_as_uint(sp.w);
      hit = d2 < r2;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (FILL) {
      const int pos = n + __popc(m & below);
      if (hit && pos < kNbListCap) {
        list[warp][pos].d2 = d2;
        list[warp][pos].idx = sidx;
      }
    }
    n += __popc(m);
  }

  if (!FILL) {
    if (lane == 0) {
      counts[qi] = n;
      atomicMax(out_max, n);
    }
    return;
  }
  if (counts != nullptr && lane == 0) counts[qi] = n;
  if (out_max != nullptr && lane == 0) atomicMax(out_max, n);
  __syncwarp();
  int* row = out_idx + (size_t)qi * cols;
  // Fast path for n <= 64 (every row of a calibrated pyramid): bitonic sort of 32-bit keys = the d2 bit pattern with
  // its low 6 bits replaced by the hit's slot in `list`. Such keys are unique, one SHFL + one predicated min/max per
  // compare-exchange (the exact 64-bit (d2, idx) keys below cost ~7 instructions), and the sorted slot gives the
  // index back. The order is the exact (d2, idx) order iff no two hits agree in the upper 26 bits of d2 -- checked on
  // the sorted keys (neighbours only); a row that fails (ties, or d2 values within 64 ulp: ~0.3 % of rows) falls
  // through to the exact sort. Elements 2*lane and 2*lane+1 live in one lane, so the j = 1 exchanges need no shuffle.
  bool sorted_fast = false;
  if (n <= 64) {
    const int ia = 2 * lane, ib = ia + 1;
    unsigned ka = 0xffffffffu, kb = 0xffffffffu;   // d2 < r2 is finite: real keys are below the padding
    if (ia < n) ka = (__float_as_uint(list[warp][ia].d2) & ~63u) | (unsigned)ia;
    if (ib < n) kb = (__float_as_uint(list[warp][ib].d2) & ~63u) | (unsigned)ib;
    const int kmax = n <= 2 ? 2 : 2 << (31 - __clz(n - 1));   // next power of two >= n (warp-uniform)
    if (kmax >= 2) bitonic_block2<2>(ka, kb, lane);            // kmax is warp-uniform
    if (kmax >= 4) bitonic_block2<4>(ka, kb, lane);
    if (kmax >= 8) bitonic_block2<8>(ka, kb, lane);
    if (kmax >= 16) bitonic_block2<16>(ka, kb, lane);
    if (kmax >= 32) bitonic_block2<32>(ka, kb, lane);
    if (kmax >= 64) bitonic_block2<64>(ka, kb, lane);
    // padding sorts last, so elements [0, n) are the hits; neighbours in one 64-ulp bucket -> exact path
    const unsigned next_a = __shfl_down_sync(0xffffffffu, ka, 1);
    const bool clash = (ib < n && ((ka ^ kb) < 64u)) || (ib + 1 < n && lane < 31 && ((kb ^ next_a) < 64u));
    if (!__any_sync(0xffffffffu, clash)) {
      if (ia < n && ia < cols) row[ia] = list[warp][ka & 63u].idx;
      if (ib < n && ib < cols) row[ib] = list[warp][kb & 63u].idx;
      sorted_fast = true;
    }
  }
  if (sorted_fast) {
  } else if (n <= 64) {
    // the common case: bitonic sort of <= 64 packed (d2, idx) keys in registers, two per lane (elements lane and
    // lane + 32). d2 >= +0, so the float's bit pattern orders like its value and the 64-bit key orders like
    // (d2, idx) -- the same total order as hit_less.
    const unsigned long long kInf = ~0ull;
    unsigned long long a = kInf, b = kInf;
    if (lane < n) a = ((unsigned long long)__float_as_uint(list[warp][lane].d2) << 32) | (unsigned)list[warp][lane].idx;
    if (n <= 32) {
#pragma unroll
      for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
          unsigned long long o = __shfl_xor_sync(0xffffffffu, a, j);
          bool keep_min = ((lane & j) == 0) == ((lane & k) == 0);
          a = (keep_min == (o < a)) ? o : a;
        }
      }
      if (lane < n && lane < cols) row[lane] = (int)(unsigned)a;
    } else {
      if (lane + 32 < n)
        b = ((unsigned long long)__float_as_uint(list[warp][lane + 32].d2) << 32) | (unsigned)list[warp][lane + 32].idx;
#pragma unroll
      for (int k = 2; k <= 64; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
          if (j == 32) {   // partner of element lane is element lane + 32: same lane, ascending (k == 64)
            unsigned long long lo = a < b ? a : b, hi = a < b ? b : a;
            a = lo;
            b = hi;
          } else {
            unsigned long long oa = __shfl_xor_sync(0xffffffffu, a, j), ob = __shfl_xor_sync(0xffffffffu, b, j);
            bool lower = (lane & j) == 0;
            bool asc_a = (lane & k) == 0;                 // element index lane
            bool asc_b = ((lane + 32) & k) == 0;          // element index lane + 32
            a = ((lower == asc_a) == (oa < a)) ? oa : a;
            b = ((lower == asc_b) == (ob < b)) ? ob : b;
          }
        }
      }
      if (lane < cols) row[lane] = (int)(unsigned)a;                      // n > 32: elements 0..31 are all hits
      if (lane + 32 < n && lane + 32 < cols) row[lane + 32] = (int)(unsigned)b;
    }
  } else if (n <= kNbListCap) {
    // rank sort: rank = number of hits that precede in (d2, idx)
    for (int j = lane; j < n; j += 32) {
      float dj = list[warp][j].d2;
      int ij = list[warp][j].idx;
      int rank = 0;
      for (int k = 0; k < n; ++k) rank += hit_less(list[warp][k].d2, list[warp][k].idx, dj, ij) ? 1 : 0;
      if (rank < cols) row[rank] = ij;
    }
  } else {
    // generic path for very dense rows: emit the nearest `cols` one at a time by re-scanning the runs
    float last_d = -1.f;
    int last_i = -1;
    int emit = min(n, cols);
    for (int c = 0; c < emit; ++c) {
      float best_d = 3.0e38f;
      int best_i = 0x7fffffff;
      for (int t = lane; t < T; t += 32) {
        int r = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) r += (t >= run_tab[warp][k].x) ? 1 : 0;
        float4 sp = sorted_pts[t + run_tab[warp][r].y];
        float d2 = sq_dist_rn(qx, qy, qz, sp);
        int si = (int)__float_as_uint(sp.w);
        if (d2 < r2 && hit_less(last_d, last_i, d2, si) && hit_less(d2, si, best_d, best_i)) {
          best_d = d2;
          best_i = si;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        float od = __shfl_xor_sync(0xffffffffu, best_d, o);
        int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
        if (hit_less(od, oi, best_d, best_i)) {
          best_d = od;
          best_i = oi;
        }
      }
      if (lane == 0) row[c] = best_i;
      last_d = best_d;
      last_i = best_i;
    }
  }
  for (int c = n + lane; c < cols; c += 32) row[c] = pad_value;
}

// ---------------------------------------------------------------------------------------------------
// The same query with TWO queries per warp (16 lanes each). The kernel above is instruction bound: a large share of a
// query's warp instructions is the prologue (nine lanes busy) and the 64-key sort (two keys per lane, 15 of 21 exchange levels through shuffles). With 16 lanes per query the prologue
// serves two queries per warp instruction and a lane holds FOUR keys (elements 4 l .. 4 l + 3): only the exchanges at
// distance >= 4 need a shuffle (10 of 21 levels). The candidate loop is unchanged in lane efficiency (~110 candidates
// in steps of 16; the warp runs to the longer of its two lists).
// Rows whose sorted 32-bit keys clash (ties, d2 within 64 ulp) and rows with more than 64 hits take an exact rank sort
// over the shared-memory list (up to kNbListCap2 hits), denser rows the re-scan path -- per half-warp, under a
// half-warp mask, so the other query of the warp is not held up by warp-wide shuffles.
constexpr int kNbListCap2 = 256;   // hits kept in shared memory per query (16 queries per CTA: 32 KB)

__device__ __forceinline__ void cex_dir(unsigned& a, unsigned& b, bool asc) {   // in-lane compare-exchange
  const unsigned lo = min(a, b), hi = max(a, b);
  a = asc ? lo : hi;
  b = asc ? hi : lo;
}
// block size K of the 64-element bitonic sort, four elements per lane (i = 4 hl + e), 16 lanes
template <int K>
__device__ __forceinline__ void bitonic_block4(unsigned (&k)[4], int hl) {
  if (K == 2) {
    cex_dir(k[0], k[1], true);
    cex_dir(k[2], k[3], false);
    return;
  }
  const bool asc = K == 64 || (hl & (K >> 2)) == 0;      // all four elements of a lane sit in the same block for K >= 4
#pragma unroll
  for (int j = K >> 1; j >= 4; j >>= 1) {
    const bool keep_min = ((hl & (j >> 2)) == 0) == asc;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const unsigned o = __shfl_xor_sync(0xffffffffu, k[e], j >> 2);
      k[e] = keep_min ? min(k[e], o) : max(k[e], o);
    }
  }
  cex_dir(k[0], k[2], asc);
  cex_dir(k[1], k[3], asc);
  cex_dir(k[0], k[1], asc);
  cex_dir(k[2], k[3], asc);
}

__global__ void __launch_bounds__(kNbWarps * 32, 6)
radius_query2_kernel(const float* __restrict__ q, int Nq_cap, const int* __restrict__ nq_dev,
                     const int* __restrict__ q_start, int B, NbGrid g, const float4* __restrict__ sorted_pts,
                     const int* __restrict__ cell_start, float r2, int cols, int pad_value_in,
                     const int* __restrict__ pad_dev, int* __restrict__ counts, int* __restrict__ out_max,
                     int* __restrict__ out_idx) {
  const int Nq = dyn_rows(Nq_cap, nq_dev);
  const int pad_value = pad_dev ? __ldg(pad_dev) : pad_value_in;
  __shared__ int2 run_tab[kNbWarps * 2][10];
  __shared__ Hit list[kNbWarps * 2][kNbListCap2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int hw = lane >> 4, hl = lane & 15;
  const int slot = warp * 2 + hw;
  const int qi_raw = (blockIdx.x * kNbWarps + warp) * 2 + hw;
  if ((blockIdx.x * kNbWarps + warp) * 2 >= Nq) return;   // warp-uniform: both queries beyond the end
  const bool qvalid = qi_raw < Nq;
  const int qi = qvalid ? qi_raw : Nq - 1;                 // an odd tail half idles on a copy of the last query
  const unsigned hmask = 0xffffu << (16 * hw);
  const float qx = q[3 * (size_t)qi], qy = q[3 * (size_t)qi + 1], qz = q[3 * (size_t)qi + 2];
  int b;
  if (B <= 16) {
    const bool le = hl < B && __ldg(q_start + hl) <= qi;
    b = max(__popc((__ballot_sync(0xffffffffu, le) >> (16 * hw)) & 0xffffu) - 1, 0);
  } else {
    b = batch_of(q_start, B, qi);
  }
  const int cx = cell_coord(qx, g.minx, g.inv_cell, g.nx);
  const int cy = cell_coord(qy, g.miny, g.inv_cell, g.ny);
  const int cz = cell_coord(qz, g.minz, g.inv_cell, g.nz);
  int rs = 0, rl = 0;
  if (hl < 9) {
    const int dz = (hl * 11) >> 5;            // hl / 3 for hl < 9
    const int yy = cy + (hl - 3 * dz) - 1, zz = cz + dz - 1;
    if (yy >= 0 && yy < g.ny && zz >= 0 && zz < g.nz) {
      const int row = b * (int)g.ncells + (zz * g.ny + yy) * g.nx;
      const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.nx - 1);
      const int s = __ldg(cell_start + row + x0), e = __ldg(cell_start + row + x1 + 1);
      if (e > s) {
        rs = s;
        rl = e - s;
      }
    }
  }
  int inc = rl;
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o, 16);
    if (hl >= o) inc += t;
  }
  if (hl < 9) run_tab[slot][hl] = make_int2(inc, rs - (inc - rl));
  int T = __shfl_sync(0xffffffffu, inc, 8, 16);
  if (!qvalid || qi >= __ldg(q_start + B)) T = 0;   // a query of no cloud: no neighbours, a row of padding
  if (hl == 9) run_tab[slot][9] = make_int2(0x7fffffff, 0);
  __syncwarp();
  const int Tmax = max(T, __shfl_xor_sync(0xffffffffu, T, 16));

  int n = 0;
  const int2* tp = &run_tab[slot][0];
  int2 cur = *tp;
  const unsigned below = (1u << hl) - 1u;
  for (int t0 = 0; t0 < Tmax; t0 += 16) {
    const int t = t0 + hl;
    bool hit = false;
    float d2 = 0.f;
    int sidx = 0;
    if (t < T) {
      while (t >= cur.x) cur = *++tp;
      const float4 sp = __ldg(sorted_pts + (t + cur.y));
      d2 = sq_dist_rn(qx, qy, qz, sp);
      sidx = (int)__float_as_uint(sp.w);
      hit = d2 < r2;
    }
    const unsigned m = (__ballot_sync(0xffffffffu, hit) >> (16 * hw)) & 0xffffu;
    const int pos = n + __popc(m & below);
    if (hit && pos < kNbListCap2) {
      list[slot][pos].d2 = d2;
      list[slot][pos].idx = sidx;
    }
    n += __popc(m);
  }
  if (qvalid && hl == 0) {
    if (counts != nullptr) counts[qi] = n;
    if (out_max != nullptr) atomicMax(out_max, n);
  }
  __syncwarp();
  int* row = out_idx + (size_t)qi * cols;

  // ---- fast path: 64-key bitonic sort of unique 32-bit keys, both queries of the warp together ---------------
  bool done = !qvalid;
  {
    const int nmax = max(n, __shfl_xor_sync(0xffffffffu, n, 16));
    const bool mine = qvalid && n <= 64;
    unsigned k[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int i = 4 * hl + e;
      k[e] = (mine && i < n) ? ((__float_as_uint(list[slot][i].d2) & ~63u) | (unsigned)i) : 0xffffffffu;
    }
    const int nsort = min(nmax, 64);
    const int kmax = nsort <= 2 ? 2 : 2 << (31 - __clz(nsort - 1));   // warp-uniform
    if (kmax >= 2) bitonic_block4<2>(k, hl);
    if (kmax >= 4) bitonic_block4<4>(k, hl);
    if (kmax >= 8) bitonic_block4<8>(k, hl);
    if (kmax >= 16) bitonic_block4<16>(k, hl);
    if (kmax >= 32) bitonic_block4<32>(k, hl);
    if (kmax >= 64) bitonic_block4<64>(k, hl);
    const unsigned next0 = __shfl_down_sync(0xffffffffu, k[0], 1, 16);
    const int i0 = 4 * hl;
    bool clash = (i0 + 1 < n && ((k[0] ^ k[1]) < 64u)) || (i0 + 2 < n && ((k[1] ^ k[2]) < 64u)) ||
                 (i0 + 3 < n && ((k[2] ^ k[3]) < 64u)) || (i0 + 4 < n && hl < 15 && ((k[3] ^ next0) < 64u));
    const bool any_clash = ((__ballot_sync(0xffffffffu, mine && clash) >> (16 * hw)) & 0xffffu) != 0u;
    if (mine && !any_clash) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = i0 + e;
        if (i < n && i < cols) row[i] = list[slot][k[e] & 63u].idx;
      }
      done = true;
    }
  }
  // ---- exact paths, per half-warp ------------------------------------------------------------------------------
  if (!done) {
    if (n <= kNbListCap2) {
      // rank sort: rank = number of hits that precede in (d2, idx)
      for (int j = hl; j < n; j += 16) {
        const float dj = list[slot][j].d2;
        const int ij = list[slot][j].idx;
        int rank = 0;
        for (int kk = 0; kk < n; ++kk) rank += hit_less(list[slot][kk].d2, list[slot][kk].idx, dj, ij) ? 1 : 0;
        if (rank < cols) row[rank] = ij;
      }
    } else {
      // very dense rows: emit the nearest `cols` one at a time by re-scanning the runs
      float last_d = -1.f;
      int last_i = -1;
      const int emit = min(n, cols);
      for (int c = 0; c < emit; ++c) {
        float best_d = 3.0e38f;
        int best_i = 0x7fffffff;
        for (int t = hl; t < T; t += 16) {
          int r = 0;
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) r += (t >= run_tab[slot][kk].x) ? 1 : 0;
          const float4 sp = sorted_pts[t + run_tab[slot][r].y];
          const float d2 = sq_dist_rn(qx, qy, qz, sp);
          const int si = (int)__float_as_uint(sp.w);
          if (d2 < r2 && hit_less(last_d, last_i, d2, si) && hit_less(d2, si, best_d, best_i)) {
            best_d = d2;
            best_i = si;
          }
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
          const float od = __shfl_xor_sync(hmask, best_d, o);
          const int oi = __shfl_xor_sync(hmask, best_i, o);
          if (hit_less(od, oi, best_d, best_i)) {
            best_d = od;
            best_i = oi;
          }
        }
        if (hl == 0) row[c] = best_i;
        last_d = best_d;
        last_i = best_i;
      }
    }
  }
  if (qvalid)
    for (int c = n + hl; c < cols; c += 16) row[c] = pad_value;
}

static int query_common(bool fill, const float* queries, const int* q_batch_len, int Nq, int B, int Ns, float radius,
                        const float* host_bbox, const void* workspace, int cols, int pad_value, int* counts,
                        int* out_max, int* out_idx, cudaStream_t stream, const int* nq_dev = nullptr,
                        const int* pad_dev = nullptr, const int* q_start_pre = nullptr) {
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch && Nq >= 0 && radius > 0.f && host_bbox != nullptr, D3F_ERR_INVALID,
              "radius_neighbors: invalid arguments (B=%d Nq=%d radius=%g)", B, Nq, (double)radius);
  NbGrid g = make_grid(host_bbox, radius);
  long long total = g.ncells * B;
  D3F_REQUIRE(total <= kMaxGridCells, D3F_ERR_CAPACITY, "radius_neighbors: grid too large");
  D3F_REQUIRE(radius_scan_complete(g), D3F_ERR_INVALID,
              "radius_neighbors: grid %d x %d x %d has an axis longer than %d cells (of radius * 1.001)", g.nx, g.ny,
              g.nz, kMaxScanAxisCells);
  NbWs w;
  nb_layout(Ns, B, radius, host_bbox, const_cast<void*>(workspace), &w);
  if (q_start_pre != nullptr) w.q_start = const_cast<int*>(q_start_pre);
  else if (launch_batch_start(q_batch_len, B, w.q_start, stream)) return D3F_ERR_CUDA;
  if (out_max != nullptr && !fill) D3F_CUDA(cudaMemsetAsync(out_max, 0, sizeof(int), stream));
  if (Nq == 0) return D3F_OK;
  float r2 = radius * radius;  // neighbors.cpp:226 (fp32 product)
  int blocks = ceil_div(Nq, kNbWarps);
  // two queries per warp by default (step 3.09 -> 3.02 ms, 1 M-point search 0.85 -> 0.76 ms); D3F_NB_HALFWARP=0
  // selects the one-query-per-warp kernel (read per call: tests run both)
  const char* hv = getenv("D3F_NB_HALFWARP");
  if (fill && !(hv != nullptr && hv[0] == '0')) {
    radius_query2_kernel<<<ceil_div(Nq, kNbWarps * 2), kNbWarps * 32, 0, stream>>>(
        queries, Nq, nq_dev, w.q_start, B, g, w.sorted_pts, w.cell_start, r2, cols, pad_value, pad_dev, counts, out_max,
        out_idx);
    D3F_LAUNCH_CHECK("radius_query2_kernel");
    return D3F_OK;
  }
  if (fill) {
    radius_query_kernel<true><<<blocks, kNbWarps * 32, 0, stream>>>(queries, Nq, nq_dev, w.q_start, B, g, w.sorted_pts,
                                                                    w.cell_start, r2, cols, pad_value, pad_dev,
                                                                    counts, out_max, out_idx);
  } else {
    radius_query_kernel<false><<<blocks, kNbWarps * 32, 0, stream>>>(queries, Nq, nq_dev, w.q_start, B, g, w.sorted_pts,
                                                                     w.cell_start, r2, 0, 0, nullptr, counts,
                                                                     out_max, nullptr);
  }
  D3F_LAUNCH_CHECK("radius_query_kernel");
  return D3F_OK;
}

int radius_neighbors_fill(const float* queries, const int* q_batch_len, int Nq, int B, int Ns, float radius,
                          const float* host_bbox, const void* workspace, int cols, int pad_value, int* out_idx,
                          cudaStream_t stream, const int* nq_dev, const int* pad_dev, const int* q_start_pre) {
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "radius_neighbors: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(cols >= 0 && (out_idx != nullptr || cols == 0 || Nq == 0), D3F_ERR_INVALID,
              "radius_neighbors_fill: cols=%d / null output", cols);
  if (cols == 0) return D3F_OK;
  return query_common(true, queries, q_batch_len, Nq, B, Ns, radius, host_bbox, workspace, cols, pad_value, nullptr,
                      nullptr, out_idx, stream, nq_dev, pad_dev, q_start_pre);
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_radius_neighbors_workspace_bytes(int Ns, int B, float radius, const float* host_bbox) {
  return nb_layout(Ns, B, radius, host_bbox, nullptr, nullptr);
}

extern "C" int d3f_radius_neighbors_build(const float* supports, const int* s_batch_len, int B, int Ns, float radius,
                                          const float* host_bbox, void* workspace, size_t workspace_bytes,
                                          d3f_stream_t stream) {
  D3F_REQUIRE((supports != nullptr || Ns == 0) && s_batch_len != nullptr && workspace != nullptr, D3F_ERR_INVALID,
              "d3f_radius_neighbors_build: null pointer");
  return radius_neighbors_build(supports, s_batch_len, B, Ns, radius, host_bbox, workspace, workspace_bytes,
                                (cudaStream_t)stream);
}

extern "C" int d3f_radius_neighbors_count(const float* queries, const int* q_batch_len, int Nq, const float* supports,
                                          const int* s_batch_len, int B, int Ns, float radius, const float* host_bbox,
                                          const void* workspace, int* counts, int* out_max, d3f_stream_t stream) {
  (void)supports;
  (void)s_batch_len;
  D3F_REQUIRE((queries != nullptr || Nq == 0) && q_batch_len != nullptr && workspace != nullptr, D3F_ERR_INVALID,
              "d3f_radius_neighbors_count: null pointer");
  D3F_REQUIRE(counts != nullptr && out_max != nullptr, D3F_ERR_INVALID, "radius_neighbors_count: null output");
  return query_common(false, queries, q_batch_len, Nq, B, Ns, radius, host_bbox, workspace, 0, 0, counts, out_max,
                      nullptr, (cudaStream_t)stream);
}

extern "C" int d3f_radius_neighbors_fill(const float* queries, const int* q_batch_len, int Nq, const float* supports,
                                         const int* s_batch_len, int B, int Ns, float radius, const float* host_bbox,
                                         const void* workspace, int cols, int pad_value, int* out_idx,
                                         d3f_stream_t stream) {
  (void)supports;
  (void)s_batch_len;
  D3F_REQUIRE((queries != nullptr || Nq == 0) && q_batch_len != nullptr && workspace != nullptr, D3F_ERR_INVALID,
              "d3f_radius_neighbors_fill: null pointer");
  return radius_neighbors_fill(queries, q_batch_len, Nq, B, Ns, radius, host_bbox, workspace, cols, pad_value, out_idx,
                               (cudaStream_t)stream);
}

// Support indices in cell order (the payload of the sorted keys): a spatially coherent visiting order that
// gather kernels can use for their queries when queries == supports.
extern "C" int d3f_radius_neighbors_order(const void* workspace, int Ns, int B, float radius, const float* host_bbox,
                                          int* out_order, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(workspace != nullptr && (out_order != nullptr || Ns == 0), D3F_ERR_INVALID,
              "d3f_radius_neighbors_order: null pointer");
  D3F_REQUIRE(B >= 1 && radius > 0.f && host_bbox != nullptr, D3F_ERR_INVALID, "radius_neighbors_order: bad arguments");
  if (Ns <= 0) return D3F_OK;
  NbGrid g = make_grid(host_bbox, radius);
  long long total = g.ncells * B;
  D3F_REQUIRE(total <= kMaxGridCells, D3F_ERR_CAPACITY, "radius_neighbors: grid too large");
  // arguments whose grid d3f_radius_neighbors_build refuses have no workspace to order (the layout is 0)
  NbWs w;
  D3F_REQUIRE(nb_layout(Ns, B, radius, host_bbox, const_cast<void*>(workspace), &w) > 0, D3F_ERR_INVALID,
              "radius_neighbors_order: no grid of these arguments can be built");
  cell_order_kernel<<<ceil_div(Ns, 256), 256, 0, stream>>>(w.sorted_pts, Ns, out_order);
  D3F_LAUNCH_CHECK("cell_order_kernel");
  return D3F_OK;
}

// Training pairs of D3Feat on the GPU: the ground-truth correspondences of anchor / positive cloud pairs, the sampled
// keypoint correspondences and the generators' augmentation -- what datasets/KITTI.py (get_matching_indices, :35-48,
// 319-327; the keypoint draw :184-189; the augmentation :191-206), datasets/cal_overlap.py (:78-126) and
// datasets/ThreeDMatch.py (:218-229, rotate :24-45, the augmentation :266-273) compute on the host.
//
// The contract is oracle/pairs_np.py, exactly.
//
// Correspondences (two phases, as the radius neighbours). Anchor row s of pair p becomes q = R s + t (fp64, residual2's
// order, no FMA); d^2 against the positive cloud's rows as nearest_in_cloud computes it (nbgrid.cuh).
//   corr_prepare_kernel  one CTA: each pair's clouds, and the most blocks of kRows anchor rows of any pair.
//   corr_count_kernel    one CTA per (pair, block of kRows anchor rows), grid-stride over (block, pair): one thread per
//                        row counts its matches; the block's total (int64) goes to bcnt[p * max_blocks + block].
//   corr_offsets_kernel  one CTA: the exclusive scan of bcnt in (pair, block) order, offset, count and overlap.
//   corr_fill_kernel     the count kernel's work items again: each row recounts, takes its place from a CTA scan and
//                        writes its matches, insertion-sorted by positive row (the grid's in-cell order comes from
//                        atomics; the output order must not).
// Sampling: without replacement, a 32-bit key per candidate from its own counter and the stable radix sort of
// (pair << 32 | key); with replacement, draw_index of the draw's counter. One thread per (pair, draw) picks.
// Augmentation: one CTA draws every pair's parameters and scans the output offsets; one thread per output row then
// applies noise, rotation, scale and shift in fp64 and writes the point and its backup point.
//
// Counters (rng.cuh: z = splitmix64(seed + c * golden)), c = (pair << 36) | (index << 4) | slot, one slot per purpose
// and side; u = (z >> 11) * 2^-53.
#include <algorithm>
#include <cmath>

#include "nbgrid.cuh"
#include "ops.cuh"
#include "rng.cuh"
#include "solver.cuh"
#include "sort.cuh"

namespace d3f {

namespace {

constexpr int kRows = 256;               // anchor rows per work item
constexpr int kItemCtasPerSM = 4;        // count / fill: persistent CTAs per SM
constexpr int kOneCta = 1024;            // prepare / offsets / augmentation parameters
constexpr int kMaxPairs = 1 << 24;       // the pair field of a counter (c < 2^64)

// counter slots (oracle/pairs_np.py SLOT_*)
constexpr int kSlotNoise = 0;            // + 3 * side + axis, index = cloud-local row
constexpr int kSlotAngle = 6;            // + side, index = rotation (0 .. num_axis - 1)
constexpr int kSlotAxis = 8;             // + side, index 0 (num_axis = 1)
constexpr int kSlotScale = 10;           // index 0
constexpr int kSlotShift = 11;           // + side, index = axis
constexpr int kSlotDraw = 13;            // index = draw m (with replacement)
constexpr int kSlotKey = 14;             // index = candidate c (without replacement)

__device__ __forceinline__ unsigned long long draw(unsigned long long seed, int p, unsigned i, int slot) {
  const unsigned long long c = ((unsigned long long)(unsigned)p << 36) | ((unsigned long long)i << 4) | (unsigned)slot;
  return splitmix64(seed + c * kGolden);
}

__device__ __forceinline__ double uniform(unsigned long long seed, int p, unsigned i, int slot) {
  return (double)(draw(seed, p, i, slot) >> 11) * 0x1p-53;
}

struct PairInfo {
  int a_lo, n_a;     // anchor rows
  int p_lo, n_p;     // positive rows
  int pos;           // positive cloud, -1 when the pair names a cloud outside [0, B)
  int nblk;          // blocks of kRows anchor rows
};

// rows [lo, lo + n) of cloud b: the lengths' exclusive scan cut at the row count
__device__ __forceinline__ void cloud_range(const int* start, int b, int n_rows, int& lo, int& n) {
  lo = min(max(start[b], 0), n_rows);
  n = max(min(max(start[b + 1], 0), n_rows) - lo, 0);
}

__device__ __forceinline__ PairInfo pair_info(const int* start, int B, int n_rows, const int* pairs, int p) {
  const int a = pairs[2 * p], b = pairs[2 * p + 1];
  PairInfo pi{0, 0, 0, 0, -1, 0};
  if (a >= 0 && a < B && b >= 0 && b < B) {
    cloud_range(start, a, n_rows, pi.a_lo, pi.n_a);
    cloud_range(start, b, n_rows, pi.p_lo, pi.n_p);
    pi.pos = b;
    pi.nblk = ceil_div(pi.n_a, kRows);
  }
  return pi;
}

// q = R s + t in residual2's order, m = the pair's row-major 4x4
__device__ __forceinline__ void transform(const double* __restrict__ m, const float s[3], double q[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a)
    q[a] = dadd(dadd(dadd(dmul(__ldg(m + 4 * a), s[0]), dmul(__ldg(m + 4 * a + 1), s[1])),
                     dmul(__ldg(m + 4 * a + 2), s[2])),
                __ldg(m + 4 * a + 3));
}

__device__ __forceinline__ void load3(const float* __restrict__ points, int row, float s[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) s[a] = __ldg(points + 3 * (size_t)row + a);
}

// exclusive scan of one value per thread over a CTA of blockDim.x (a multiple of 32, at most 1024) threads; *total gets
// the CTA's sum. Every thread must call it.
__device__ __forceinline__ long long cta_exclusive_scan(long long v, long long* total) {
  __shared__ long long warp_sums[32];
  __shared__ long long cta_total;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  long long inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    long long w = lane < nw ? warp_sums[lane] : 0;
    long long winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    if (lane < nw) warp_sums[lane] = winc - w;
    if (lane == 31) cta_total = winc;           // nw <= 32: lane 31 holds the CTA total
  }
  __syncthreads();
  const long long excl = warp_sums[warp] + inc - v;
  *total = cta_total;
  __syncthreads();                               // warp_sums is reused by the next call
  return excl;
}

// ---- correspondences ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kOneCta)
corr_prepare_kernel(int N, const int* __restrict__ start, int B, const int* __restrict__ pairs, int P,
                    PairInfo* __restrict__ info, int* __restrict__ max_blocks) {
  __shared__ int mb;
  if (threadIdx.x == 0) mb = 0;
  __syncthreads();
  const int n_rows = cloud_rows(N, nullptr, start, B);
  for (int p = threadIdx.x; p < P; p += kOneCta) {
    const PairInfo pi = pair_info(start, B, n_rows, pairs, p);
    info[p] = pi;
    if (pi.pos >= 0 && pi.n_p > 0) atomicMax(&mb, pi.nblk);
  }
  __syncthreads();
  if (threadIdx.x == 0) *max_blocks = mb;
}

struct Search {
  const float* points;
  NbView view;
  const double* trans;
  double tau2;
  int nearest;
};

// the matches of anchor row r of pair p: their number, and (nearest) the positive row
__device__ __forceinline__ int row_matches(const Search& S, const PairInfo& pi, int p, int r, double q[3], int& j) {
  float s[3];
  load3(S.points, pi.a_lo + r, s);
  transform(S.trans + (size_t)p * 16, s, q);
  if (S.nearest) {
    j = nearest_in_cloud(S.view, pi.pos, q[0], q[1], q[2], S.tau2).row;
    return j >= 0;
  }
  int c = 0;
  const double tau2 = S.tau2;
  visit_cloud_rows(S.view, pi.pos, q[0], q[1], q[2], [&](int, double d2) { c += d2 < tau2; });
  return c;
}

// work item e = k * P + p: block k of pair p's anchor rows, for k < the most blocks of any pair
__global__ void __launch_bounds__(kRows)
corr_count_kernel(Search S, const PairInfo* __restrict__ info, int P, const int* __restrict__ max_blocks,
                  long long* __restrict__ bcnt) {
  const int mb = __ldg(max_blocks);
  const int items = P * mb;                          // P * ceil(N / 256) * 256 is within int32 (host check)
  for (int e = blockIdx.x; e < items; e += gridDim.x) {
    const int k = e / P, p = e - k * P;
    const PairInfo pi = info[p];
    if (pi.pos < 0 || pi.n_p == 0 || k >= pi.nblk) continue;   // uniform across the CTA; bcnt is zeroed
    const int r = k * kRows + threadIdx.x;
    int c = 0;
    if (r < pi.n_a) {
      double q[3];
      int j;
      c = row_matches(S, pi, p, r, q, j);
    }
    long long total;
    cta_exclusive_scan(c, &total);
    if (threadIdx.x == 0) bcnt[(size_t)p * mb + k] = total;
  }
}

// bcnt becomes its exclusive scan; offset[p] = the first of pair p, count and overlap
__global__ void __launch_bounds__(kOneCta)
corr_offsets_kernel(const PairInfo* __restrict__ info, int P, const int* __restrict__ max_blocks,
                    long long* __restrict__ bcnt, long long* __restrict__ offset, int* __restrict__ count,
                    double* __restrict__ overlap) {
  const int mb = *max_blocks;
  const long long n = (long long)P * mb;
  long long carry = 0;
  for (long long base = 0; base < n; base += kOneCta) {
    const long long i = base + threadIdx.x;
    const long long v = i < n ? bcnt[i] : 0;
    long long total;
    const long long excl = cta_exclusive_scan(v, &total);
    if (i < n) bcnt[i] = carry + excl;
    carry += total;
  }
  __syncthreads();
  for (int p = threadIdx.x; p <= P; p += kOneCta) offset[p] = p == P ? carry : (mb == 0 ? 0 : bcnt[(size_t)p * mb]);
  __syncthreads();
  for (int p = threadIdx.x; p < P; p += kOneCta) {
    const long long c = offset[p + 1] - offset[p];
    count[p] = (int)min(c, (long long)INT32_MAX);
    const int n_a = info[p].n_a;
    overlap[p] = n_a > 0 ? ddiv((double)c, (double)n_a) : 0.0;
  }
}

// appends row (r, j - lo) to [base, end) when d^2 < tau2, keeping the run sorted by positive row
struct InsertRow {
  int* rows;
  long long base, end;
  double tau2;
  int r, lo;
  __device__ __forceinline__ void operator()(int j, double d2) {
    if (!(d2 < tau2)) return;
    const int v = j - lo;
    long long o = end++;
    rows[2 * o] = r;
    while (o > base && rows[2 * (o - 1) + 1] > v) {
      rows[2 * o + 1] = rows[2 * (o - 1) + 1];
      --o;
    }
    rows[2 * o + 1] = v;
  }
};

// min blocks 1: with ptxas' default register target the insertion scan spills 4 bytes
__global__ void __launch_bounds__(kRows, 1)
corr_fill_kernel(Search S, const PairInfo* __restrict__ info, int P, const int* __restrict__ max_blocks,
                 const long long* __restrict__ boff, long long M, int* __restrict__ rows) {
  const int mb = __ldg(max_blocks);
  const int items = P * mb;
  for (int e = blockIdx.x; e < items; e += gridDim.x) {
    const int k = e / P, p = e - k * P;
    const PairInfo pi = info[p];
    if (pi.pos < 0 || pi.n_p == 0 || k >= pi.nblk) continue;   // uniform across the CTA
    const int r = k * kRows + threadIdx.x;
    int c = 0, j = -1;
    double q[3];
    if (r < pi.n_a) c = row_matches(S, pi, p, r, q, j);
    long long total;
    const long long base = boff[(size_t)p * mb + k] + cta_exclusive_scan(c, &total);
    if (c == 0 || base + c > M) continue;
    if (S.nearest) {
      rows[2 * base] = r;
      rows[2 * base + 1] = j - pi.p_lo;
      continue;
    }
    // every row with d^2 < tau2, insertion-sorted by positive row into [base, base + c)
    visit_cloud_rows(S.view, pi.pos, q[0], q[1], q[2], InsertRow{rows, base, base, S.tau2, r, pi.p_lo});
  }
}

struct CorrWork {
  int* start;
  int* max_blocks;
  PairInfo* info;
  long long* bcnt;
  void* nb;
  size_t nb_bytes;
};

// fp32 grid radius: tau rounded up, so that the grid's cells cover tau (nbgrid.cuh)
float grid_radius(double distance) {
  float r = (float)distance;
  if ((double)r < distance) r = nextafterf(r, INFINITY);
  return r;
}

long long corr_items(int N, int P) { return (long long)P * ((N + kRows - 1) / kRows); }

bool corr_args_ok(int N, int B, int P, double distance, const float* host_bbox) {
  if (N < 0 || B < 1 || B > kMaxBatch || P < 1 || P > kMaxPairs || host_bbox == nullptr ||
      !std::isfinite(distance) || !(distance > 0))
    return false;
  if (corr_items(N, P) * kRows > INT32_MAX) return false;
  const NbGrid g = make_grid(host_bbox, grid_radius(distance));
  return g.ncells * B <= kMaxGridCells && nearest_lookup_exact(g, host_bbox);
}

// every size the workspace depends on, or 0
size_t corr_layout(int N, int B, int P, double distance, const float* host_bbox, CorrWork* w, void* base) {
  if (!corr_args_ok(N, B, P, distance, host_bbox)) return 0;
  const size_t nb = d3f_radius_neighbors_workspace_bytes(N, B, grid_radius(distance), host_bbox);
  if (nb == 0) return 0;
  Carver cv(base);
  CorrWork x;
  x.start = cv.take<int>(B + 1);
  x.max_blocks = cv.take<int>(1);
  x.info = cv.take<PairInfo>(P);
  x.bcnt = cv.take<long long>((size_t)corr_items(N, P));
  x.nb = cv.take<char>(nb);
  x.nb_bytes = nb;
  if (w != nullptr) *w = x;
  return cv.off;
}

int corr_check(const char* who, const float* points, int B, int N, const float* host_bbox, const int* pairs, int P,
               const double* trans, double distance, int mode, void* workspace, size_t workspace_bytes, CorrWork* w) {
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "%s: B=%d must be in [1,%d]", who, B, kMaxBatch);
  D3F_REQUIRE(N >= 0 && P >= 1 && P <= kMaxPairs, D3F_ERR_INVALID, "%s: bad shape N=%d P=%d", who, N, P);
  D3F_REQUIRE(mode == D3F_CORR_RADIUS || mode == D3F_CORR_NEAREST, D3F_ERR_INVALID, "%s: mode=%d", who, mode);
  D3F_REQUIRE(std::isfinite(distance) && distance > 0.0, D3F_ERR_INVALID, "%s: distance=%g must be finite and > 0",
              who, distance);
  D3F_REQUIRE((points || N == 0) && host_bbox && pairs && trans && workspace, D3F_ERR_INVALID, "%s: null pointer",
              who);
  D3F_REQUIRE(corr_items(N, P) * kRows <= INT32_MAX, D3F_ERR_INVALID,
              "%s: P*ceil(N/256)*256 exceeds int32 (N=%d P=%d)", who, N, P);
  const NbGrid g = make_grid(host_bbox, grid_radius(distance));
  D3F_REQUIRE(g.ncells * B <= kMaxGridCells && radius_scan_complete(g), D3F_ERR_INVALID,
              "%s: grid %d x %d x %d x %d clouds at distance %g exceeds %lld cells or 4096 per axis", who, g.nx, g.ny,
              g.nz, B, distance, kMaxGridCells);
  D3F_REQUIRE(nearest_lookup_exact(g, host_bbox), D3F_ERR_INVALID,
              "%s: host_bbox coordinates beyond 1024 cells (of distance * 1.001) from the origin", who);
  const size_t need = corr_layout(N, B, P, distance, host_bbox, w, workspace);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu bytes)", who,
              workspace_bytes, need);
  return D3F_OK;
}

Search make_search(const float* points, const NbView& view, const double* trans, double distance, int mode) {
  return Search{points, view, trans, distance * distance, mode == D3F_CORR_NEAREST};
}

// ---- sampling ----------------------------------------------------------------------------------------------------

// [lo, hi) of pair p's candidates, clamped into [0, M)
__device__ __forceinline__ void candidates(const long long* __restrict__ offset, int p, long long M, long long& lo,
                                           long long& hi) {
  lo = min(max(offset[p], 0ll), M);
  hi = min(max(offset[p + 1], lo), M);
}

// key of entry i: (pair << 32 | 32-bit draw of its candidate index); entries of no pair get pair P and sort last
__global__ void __launch_bounds__(256)
sample_keys_kernel(const long long* __restrict__ offset, int P, int M, unsigned long long seed,
                   uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= M) return;
  int lo_p = 0, hi_p = P - 1;                        // the last pair whose first candidate is at or before i
  while (lo_p < hi_p) {
    const int mid = (lo_p + hi_p + 1) >> 1;
    if (min(max(offset[mid], 0ll), (long long)M) <= i) lo_p = mid; else hi_p = mid - 1;
  }
  long long lo, hi;
  candidates(offset, lo_p, M, lo, hi);
  uint64_t key = ((uint64_t)P << 32) | 0xffffffffu;
  uint32_t c = 0;
  if (i >= lo && i < hi) {
    c = (uint32_t)(i - lo);
    key = ((uint64_t)lo_p << 32) | (draw(seed, lo_p, c, kSlotKey) >> 32);
  }
  keys[i] = key;
  vals[i] = c;
}

__global__ void __launch_bounds__(256)
sample_pick_kernel(const long long* __restrict__ offset, const int* __restrict__ rows, int M, int P,
                   const int* __restrict__ anchor_len, int k, int replace, int min_count, unsigned long long seed,
                   const uint32_t* __restrict__ sorted, int* __restrict__ anc, int* __restrict__ pos,
                   int* __restrict__ valid) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (t >= (long long)P * k) return;
  const int p = (int)(t / k), m = (int)(t - (long long)p * k);
  long long lo, hi;
  candidates(offset, p, M, lo, hi);
  const int n = (int)(hi - lo);
  const bool ok = n >= max(min_count, 1) && (replace || n >= k);
  if (m == 0) valid[p] = ok;
  int a = -1, b = -1;
  if (ok) {
    // rows before offset[0] belong to no pair and sort last, so pair p's candidates sit at lo - offset[0] in `sorted`
    const long long lo0 = min(max(offset[0], 0ll), (long long)M);
    const unsigned c = replace ? (unsigned)draw_index(draw(seed, p, (unsigned)m, kSlotDraw), n)
                               : sorted[(lo - lo0) + m];
    if (c < (unsigned)n) {
      a = rows[2 * (lo + c)];
      b = rows[2 * (lo + c) + 1] + __ldg(anchor_len + p);
    }
  }
  anc[t] = a;
  pos[t] = b;
}

int sort_bits(int P) {
  int b = 0;
  while ((1ll << b) <= (long long)P) ++b;          // pair ids 0 .. P (P: entries of no pair)
  return 32 + b;
}

size_t sample_layout(int M, int P, SortBuffers* sb, void* base) {
  if (M < 0 || P < 1 || P > kMaxPairs) return 0;
  Carver cv(base);
  SortBuffers s;
  for (int i = 0; i < 2; ++i) {
    s.keys[i] = cv.take<uint64_t>((size_t)std::max(M, 1));
    s.vals[i] = cv.take<uint32_t>((size_t)std::max(M, 1));
  }
  s.block_hist = cv.take<int>(256 * (size_t)sort_num_blocks(M));
  if (sb != nullptr) *sb = s;
  return cv.off;
}

// ---- augmentation ------------------------------------------------------------------------------------------------

struct Augment {
  unsigned long long seed;
  double noise;
  int num_axis;
  int scale_shift;
  double scale_min, scale_max, shift_range;
};

// the reference's rotate(): float32 R from fp64 cos / sin of theta = u * 2 * pi, row and column `axis` of the identity
__device__ __forceinline__ void rotation(const Augment& A, int p, int side, int a, float R[9]) {
  const double theta = dmul(dmul(uniform(A.seed, p, (unsigned)a, kSlotAngle + side), 2.0), 3.141592653589793);
  const int axis = A.num_axis == 1 ? (int)dmul(uniform(A.seed, p, 0u, kSlotAxis + side), 3.0) : a;
  const float c = (float)cos(theta), s = (float)sin(theta);
  const float m[9] = {c, -s, -s, s, c, -s, s, s, c};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) R[3 * i + j] = (i == axis || j == axis) ? (i == j ? 1.0f : 0.0f) : m[3 * i + j];
}

__global__ void __launch_bounds__(kOneCta)
aug_prepare_kernel(int N, const int* __restrict__ start, int B, const int* __restrict__ pairs, int P, Augment A,
                   int4* __restrict__ info, int* __restrict__ out_lengths, long long* __restrict__ row_offset,
                   float* __restrict__ R, double* __restrict__ scale, double* __restrict__ shift) {
  const int n_rows = cloud_rows(N, nullptr, start, B);
  long long carry = 0;
  for (int base = 0; base < P; base += kOneCta) {
    const int p = base + threadIdx.x;
    long long rows = 0;
    if (p < P) {
      const PairInfo pi = pair_info(start, B, n_rows, pairs, p);
      info[p] = make_int4(pi.a_lo, pi.n_a, pi.p_lo, pi.n_p);
      out_lengths[2 * p] = pi.n_a;
      out_lengths[2 * p + 1] = pi.n_p;
      rows = (long long)pi.n_a + pi.n_p;
      for (int side = 0; side < 2; ++side) {
        for (int a = 0; a < A.num_axis; ++a)
          rotation(A, p, side, a, R + ((size_t)(2 * p + side) * A.num_axis + a) * 9);
        for (int x = 0; x < 3; ++x)
          shift[(size_t)(2 * p + side) * 3 + x] =
              A.scale_shift ? dadd(-A.shift_range, dmul(dsub(A.shift_range, -A.shift_range),
                                                        uniform(A.seed, p, (unsigned)x, kSlotShift + side)))
                            : 0.0;
      }
      scale[p] = A.scale_shift ? dadd(A.scale_min, dmul(dsub(A.scale_max, A.scale_min),
                                                        uniform(A.seed, p, 0u, kSlotScale)))
                               : 1.0;
    }
    long long total;
    const long long excl = cta_exclusive_scan(rows, &total);
    if (p < P) row_offset[p] = carry + excl;
    carry += total;
  }
  if (threadIdx.x == 0) row_offset[P] = carry;
}

__global__ void __launch_bounds__(256)
aug_points_kernel(const float* __restrict__ points, const int4* __restrict__ info, int P,
                  const long long* __restrict__ row_offset, int capacity, const double* __restrict__ trans, Augment A,
                  const float* __restrict__ R, const double* __restrict__ scale, const double* __restrict__ shift,
                  float* __restrict__ out_points, float* __restrict__ backup) {
  const int r = blockIdx.x * 256 + threadIdx.x;
  if (r >= capacity || (long long)r >= row_offset[P]) return;
  int lo = 0, hi = P - 1;                            // the last pair starting at or before r (it holds r)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (row_offset[mid] <= r) lo = mid; else hi = mid - 1;
  }
  const int p = lo;
  const int4 pi = info[p];
  const int local = (int)(r - row_offset[p]);
  const int side = local < pi.y ? 0 : 1;
  const int lr = side ? local - pi.y : local;
  float x[3];
  load3(points, (side ? pi.z : pi.x) + lr, x);
  double y[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    y[a] = dadd(x[a], dmul(uniform(A.seed, p, (unsigned)lr, kSlotNoise + 3 * side + a), A.noise));
  for (int k = 0; k < A.num_axis; ++k) {
    const float* m = R + ((size_t)(2 * p + side) * A.num_axis + k) * 9;
    double z[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) z[j] = dadd(dadd(dmul(y[0], m[j]), dmul(y[1], m[3 + j])), dmul(y[2], m[6 + j]));
#pragma unroll
    for (int j = 0; j < 3; ++j) y[j] = z[j];
  }
  if (A.scale_shift) {
    const double sc = scale[p];
#pragma unroll
    for (int a = 0; a < 3; ++a) y[a] = dadd(dmul(sc, y[a]), shift[(size_t)(2 * p + side) * 3 + a]);
  }
  double q[3] = {x[0], x[1], x[2]};
  if (side == 0) transform(trans + (size_t)p * 16, x, q);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    out_points[3 * (size_t)r + a] = __double2float_rn(y[a]);
    backup[3 * (size_t)r + a] = __double2float_rn(q[a]);
  }
}

size_t aug_layout(int B, int P, int** start, int4** info, void* base) {
  if (B < 1 || B > kMaxBatch || P < 1 || P > kMaxPairs) return 0;
  Carver cv(base);
  int* s = cv.take<int>(B + 1);
  int4* i = cv.take<int4>(P);
  if (start != nullptr) *start = s;
  if (info != nullptr) *info = i;
  return cv.off;
}

}  // namespace
}  // namespace d3f

// ---- host entry points -------------------------------------------------------------------------------------------

using namespace d3f;

extern "C" size_t d3f_pair_correspondences_workspace_bytes(int N, int B, int P, double distance,
                                                           const float* host_bbox) {
  return corr_layout(N, B, P, distance, host_bbox, nullptr, nullptr);
}

extern "C" int d3f_pair_correspondences_count(const float* points, const int* lengths, int B, int N,
                                              const float* host_bbox, const int* pairs, int P, const double* trans,
                                              double distance, int mode, long long* offset, int* count,
                                              double* overlap, void* workspace, size_t workspace_bytes,
                                              d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const char* who = "pair_correspondences_count";
  CorrWork w;
  int rc = corr_check(who, points, B, N, host_bbox, pairs, P, trans, distance, mode, workspace, workspace_bytes, &w);
  if (rc) return rc;
  D3F_REQUIRE(lengths && offset && count && overlap, D3F_ERR_INVALID, "%s: null pointer", who);
  const float r = grid_radius(distance);
  if (launch_batch_start(lengths, B, w.start, stream)) return D3F_ERR_CUDA;
  rc = radius_neighbors_build(points, lengths, B, N, r, host_bbox, w.nb, w.nb_bytes, stream, nullptr, w.start);
  if (rc) return rc;
  NbView view;
  rc = radius_neighbors_view(w.nb, N, B, r, host_bbox, &view);
  if (rc) return rc;
  corr_prepare_kernel<<<1, kOneCta, 0, stream>>>(N, w.start, B, pairs, P, w.info, w.max_blocks);
  D3F_LAUNCH_CHECK("corr_prepare_kernel");
  const long long items = corr_items(N, P);
  D3F_CUDA(cudaMemsetAsync(w.bcnt, 0, sizeof(long long) * (size_t)std::max(items, 1ll), stream));
  if (items > 0) {
    const int grid = (int)std::min<long long>(items, (long long)kItemCtasPerSM * kNumSMs);
    corr_count_kernel<<<grid, kRows, 0, stream>>>(make_search(points, view, trans, distance, mode), w.info, P,
                                                  w.max_blocks, w.bcnt);
    D3F_LAUNCH_CHECK("corr_count_kernel");
  }
  corr_offsets_kernel<<<1, kOneCta, 0, stream>>>(w.info, P, w.max_blocks, w.bcnt, offset, count, overlap);
  D3F_LAUNCH_CHECK("corr_offsets_kernel");
  return D3F_OK;
}

extern "C" int d3f_pair_correspondences_fill(const float* points, int B, int N, const float* host_bbox,
                                             const int* pairs, int P, const double* trans, double distance, int mode,
                                             int M, int* rows, void* workspace, size_t workspace_bytes,
                                             d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const char* who = "pair_correspondences_fill";
  CorrWork w;
  int rc = corr_check(who, points, B, N, host_bbox, pairs, P, trans, distance, mode, workspace, workspace_bytes, &w);
  if (rc) return rc;
  D3F_REQUIRE(M >= 0 && (rows || M == 0), D3F_ERR_INVALID, "%s: M=%d / null rows", who, M);
  const long long items = corr_items(N, P);
  if (items == 0 || M == 0) return D3F_OK;
  const float r = grid_radius(distance);
  NbView view;
  rc = radius_neighbors_view(w.nb, N, B, r, host_bbox, &view);
  if (rc) return rc;
  const int grid = (int)std::min<long long>(items, (long long)kItemCtasPerSM * kNumSMs);
  corr_fill_kernel<<<grid, kRows, 0, stream>>>(make_search(points, view, trans, distance, mode), w.info, P,
                                               w.max_blocks, w.bcnt, M, rows);
  D3F_LAUNCH_CHECK("corr_fill_kernel");
  return D3F_OK;
}

extern "C" size_t d3f_sample_correspondences_workspace_bytes(int M, int P) {
  return sample_layout(M, P, nullptr, nullptr);
}

extern "C" int d3f_sample_correspondences(const long long* offset, const int* rows, int M, int P, const int* anchor_len,
                                          int k, int replace, int min_count, unsigned long long seed, int* anc,
                                          int* pos, int* valid, void* workspace, size_t workspace_bytes,
                                          d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const char* who = "sample_correspondences";
  D3F_REQUIRE(M >= 0 && P >= 1 && P <= kMaxPairs && k >= 1 && (long long)P * k <= INT32_MAX, D3F_ERR_INVALID,
              "%s: bad shape M=%d P=%d k=%d", who, M, P, k);
  D3F_REQUIRE(replace == 0 || replace == 1, D3F_ERR_INVALID, "%s: replace=%d", who, replace);
  D3F_REQUIRE(offset && (rows || M == 0) && anchor_len && anc && pos && valid && workspace, D3F_ERR_INVALID,
              "%s: null pointer", who);
  SortBuffers sb;
  const size_t need = sample_layout(M, P, &sb, workspace);
  D3F_REQUIRE(workspace_bytes >= need, D3F_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu bytes)", who,
              workspace_bytes, need);
  const uint32_t* sorted = sb.vals[0];
  if (!replace && M > 0) {
    sample_keys_kernel<<<ceil_div(M, 256), 256, 0, stream>>>(offset, P, M, seed, sb.keys[0], sb.vals[0]);
    D3F_LAUNCH_CHECK("sample_keys_kernel");
    const int cur = radix_sort_pairs(sb, M, sort_bits(P), stream);
    if (cur < 0) return cur;
    sorted = sb.vals[cur];
  }
  const long long t = (long long)P * k;
  sample_pick_kernel<<<(int)((t + 255) / 256), 256, 0, stream>>>(offset, rows, M, P, anchor_len, k, replace, min_count,
                                                                 seed, sorted, anc, pos, valid);
  D3F_LAUNCH_CHECK("sample_pick_kernel");
  return D3F_OK;
}

extern "C" size_t d3f_augment_pairs_workspace_bytes(int B, int P) {
  return aug_layout(B, P, nullptr, nullptr, nullptr);
}

extern "C" int d3f_augment_pairs(const float* points, const int* lengths, int B, int N, const int* pairs, int P,
                                 const double* trans, unsigned long long seed, double noise, int num_axis,
                                 int scale_shift, double scale_min, double scale_max, double shift_range, int capacity,
                                 float* out_points, float* backup_points, int* out_lengths, long long* row_offset,
                                 float* R, double* scale, double* shift, void* workspace, size_t workspace_bytes,
                                 d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const char* who = "augment_pairs";
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "%s: B=%d must be in [1,%d]", who, B, kMaxBatch);
  D3F_REQUIRE(N >= 0 && P >= 1 && P <= kMaxPairs && capacity >= 0, D3F_ERR_INVALID,
              "%s: bad shape N=%d P=%d capacity=%d", who, N, P, capacity);
  D3F_REQUIRE(num_axis == 1 || num_axis == 3, D3F_ERR_INVALID, "%s: num_axis=%d must be 1 or 3", who, num_axis);
  D3F_REQUIRE(std::isfinite(noise) && noise >= 0.0, D3F_ERR_INVALID, "%s: noise=%g must be finite and >= 0", who,
              noise);
  D3F_REQUIRE(scale_shift == 0 || (std::isfinite(scale_min) && std::isfinite(scale_max) && scale_min <= scale_max &&
                                   std::isfinite(shift_range) && shift_range >= 0.0),
              D3F_ERR_INVALID, "%s: scale [%g, %g] and shift_range %g must be finite, ordered and >= 0", who,
              scale_min, scale_max, shift_range);
  D3F_REQUIRE((points || N == 0) && lengths && pairs && trans && (out_points || capacity == 0) &&
                  (backup_points || capacity == 0) && out_lengths && row_offset && R && scale && shift && workspace,
              D3F_ERR_INVALID, "%s: null pointer", who);
  int* start;
  int4* info;
  const size_t need = aug_layout(B, P, &start, &info, workspace);
  D3F_REQUIRE(workspace_bytes >= need, D3F_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu bytes)", who,
              workspace_bytes, need);
  const Augment A{seed, noise, num_axis, scale_shift, scale_min, scale_max, shift_range};
  if (launch_batch_start(lengths, B, start, stream)) return D3F_ERR_CUDA;
  aug_prepare_kernel<<<1, kOneCta, 0, stream>>>(N, start, B, pairs, P, A, info, out_lengths, row_offset, R, scale,
                                                shift);
  D3F_LAUNCH_CHECK("aug_prepare_kernel");
  if (capacity == 0) return D3F_OK;
  aug_points_kernel<<<ceil_div(capacity, 256), 256, 0, stream>>>(points, info, P, row_offset, capacity, trans, A, R,
                                                                 scale, shift, out_points, backup_points);
  D3F_LAUNCH_CHECK("aug_points_kernel");
  return D3F_OK;
}

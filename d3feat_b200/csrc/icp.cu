// Point-to-point ICP of cloud pairs over the stacked input clouds -- the refinement every user of a RANSAC pose runs
// next: datasets/KITTI.py:284-301 refines each pair with Open3D's registration_icp(pcd0, pcd1, 0.2, init,
// TransformationEstimationPointToPoint(), ICPConvergenceCriteria(max_iteration=200)) on the host, one pair at a time.
//
// The contract is oracle/icp_np.py, exactly: every step is one correctly rounded fp64 operation in the order written
// there (solver.cuh). Iteration i of pair p transforms every source row by T_i (q = R s + t, residual2's order), finds
// the nearest target row with d^2 < tau^2 (ties to the smaller row), sums the centroids, then the centred
// cross-covariance, then sum d^2 over the corresponding rows in a fixed blocked order (blocks of kBlockRows
// consecutive source rows summed sequentially, then the block sums sequentially in ascending block), scores the pose
// (fitness = n / n_src, inlier_rmse = sqrt(sum d^2 / n)) and updates T_{i+1} = Horn(q, t) T_i. It stops as Open3D does:
// when both scores change by less than the relative thresholds, when n < 3 (the pose is kept), or after I updates.
//
// icp_prepare_kernel     one CTA: validates every pair's clouds, copies init into the pair state, and finds the most
//                        blocks of any source cloud (the extent of the block loops below).
// icp_correspond_kernel  one CTA per (pair, block of kBlockRows source rows), grid-stride over (block, pair): one
//                        thread per row transforms it and finds its nearest target row (nearest_in_cloud, nbgrid.cuh);
//                        seven threads then sum q, t and d^2 over the block's corresponding rows in row order.
// icp_covariance_kernel  the same work items: each CTA sums its pair's block sums to the centroids (every CTA of a
//                        pair in the same order, so they agree bit for bit), then nine threads sum the block's
//                        (q - cq)(t - ct)^T in row order.
// icp_finalize_kernel    one warp per pair: the block sums in block order, the scores, the stopping rule, Horn and the
//                        update, or the outputs of a pair that stops.
// Pairs that have stopped return at the top of every kernel. Launches are sized by (N, B, P, I) only -- the extent of
// the block loops and every count are read on the device -- so a call can be captured into a CUDA graph. For N > 0
// rows a call is 3I + 10 graph nodes: the lengths' scan, the grid build (a memset and five kernels), the prepare kernel,
// then I + 1 correspond, I covariance and I + 1 finalize kernels. For N = 0 it is the scan, two memsets and the
// prepare kernel.
#include <algorithm>
#include <cmath>

#include "nbgrid.cuh"
#include "ops.cuh"
#include "solver.cuh"

namespace d3f {

namespace {

constexpr int kBlockRows = 256;          // the contract's block of consecutive source rows (oracle/icp_np.py BLOCK)
constexpr int kItemCtasPerSM = 4;        // correspond / covariance: persistent CTAs per SM
constexpr int kFinalizeWarps = 4;        // finalize: one warp per pair
constexpr int kPrepareThreads = 1024;

struct PairState {
  Pose T;          // the current pose
  double fit, rmse;  // scores of the previous pose (the stopping rule compares against them)
  int src_lo, n_src, tgt, nblk;
  int active;      // 1 while the pair iterates
  int pad_;
};

// q = R s + t in residual2's order
__device__ __forceinline__ void transform(const Pose& T, const float s[3], double q[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a)
    q[a] = dadd(dadd(dadd(dmul(T.R[a][0], s[0]), dmul(T.R[a][1], s[1])), dmul(T.R[a][2], s[2])), T.t[a]);
}

__device__ __forceinline__ void load3(const float* __restrict__ points, int row, float s[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) s[a] = __ldg(points + 3 * (size_t)row + a);
}

// rows [lo, hi) of cloud b: the lengths' exclusive scan cut at the row count (rows at or past start[B] belong to no
// cloud)
__device__ __forceinline__ void cloud_range(const int* start, int b, int n_rows, int& lo, int& n) {
  lo = min(max(start[b], 0), n_rows);
  n = max(min(max(start[b + 1], 0), n_rows) - lo, 0);
}

__global__ void __launch_bounds__(kPrepareThreads)
icp_prepare_kernel(int N, const int* __restrict__ n_dev, const int* __restrict__ start, int B,
                   const int* __restrict__ pairs, int P, const double* __restrict__ init, PairState* __restrict__ st,
                   int* __restrict__ max_blocks, double* __restrict__ pose, double* __restrict__ fitness,
                   double* __restrict__ inlier_rmse, int* __restrict__ n_corr, int* __restrict__ iterations) {
  __shared__ int mb;
  if (threadIdx.x == 0) mb = 0;
  __syncthreads();
  const int n_rows = cloud_rows(N, n_dev, start, B);
  for (int p = threadIdx.x; p < P; p += kPrepareThreads) {
    const int src = pairs[2 * p], tgt = pairs[2 * p + 1];
    int src_lo = 0, n_src = 0, tgt_lo = 0, n_tgt = 0;
    if (src >= 0 && src < B && tgt >= 0 && tgt < B) {
      cloud_range(start, src, n_rows, src_lo, n_src);
      cloud_range(start, tgt, n_rows, tgt_lo, n_tgt);
    }
    PairState s;
    const double* m = init + (size_t)p * 16;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
      for (int b = 0; b < 3; ++b) s.T.R[a][b] = m[4 * a + b];
      s.T.t[a] = m[4 * a + 3];
    }
    s.fit = s.rmse = 0.0;
    s.src_lo = src_lo;
    s.n_src = n_src;
    s.tgt = tgt;
    s.nblk = ceil_div(n_src, kBlockRows);
    s.active = n_src > 0 && n_tgt > 0;
    s.pad_ = 0;
    st[p] = s;
    if (s.active) {
      atomicMax(&mb, s.nblk);
    } else {                             // a pair without two real clouds keeps init, reads neither
      for (int i = 0; i < 16; ++i) pose[(size_t)p * 16 + i] = m[i];
      fitness[p] = 0.0;
      inlier_rmse[p] = 0.0;
      n_corr[p] = 0;
      iterations[p] = 0;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *max_blocks = mb;
}

struct Items {
  int* corr;        // [items * kBlockRows] nearest target row of every source row of the item, -1 for none
  double* sums;     // [items * 8]: sum q (3), sum t (3), sum d^2 over the block's corresponding rows
  int* counts;      // [items]: corresponding rows of the block
  double* cov;      // [items * 9]: sum (q - cq)(t - ct)^T over the block
};

// work item e = k * P + p: block k of pair p, for k < the most blocks of any pair (read on the device)
__global__ void __launch_bounds__(kBlockRows)
icp_correspond_kernel(const float* __restrict__ points, NbView view, const PairState* __restrict__ st, int P,
                      const int* __restrict__ max_blocks, double tau2, Items it) {
  __shared__ double v[kBlockRows][7];
  __shared__ unsigned char use[kBlockRows];
  const int items = P * __ldg(max_blocks);                  // P * ceil(N / 256) * 256 is within int32 (host check)
  for (int e = blockIdx.x; e < items; e += gridDim.x) {
    const int k = e / P, p = e - k * P;
    if (!st[p].active || k >= st[p].nblk) continue;          // uniform across the CTA
    const int r = k * kBlockRows + threadIdx.x;
    int j = -1;
    if (r < st[p].n_src) {
      float s[3];
      double q[3];
      load3(points, st[p].src_lo + r, s);
      transform(st[p].T, s, q);
      const Nearest nn = nearest_in_cloud(view, st[p].tgt, q[0], q[1], q[2], tau2);
      j = nn.row;
      if (j >= 0) {
        float t[3];
        load3(points, j, t);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          v[threadIdx.x][a] = q[a];
          v[threadIdx.x][3 + a] = t[a];
        }
        v[threadIdx.x][6] = nn.d2;
      }
    }
    use[threadIdx.x] = j >= 0;
    it.corr[(size_t)e * kBlockRows + threadIdx.x] = j;
    const int cnt = __syncthreads_count(j >= 0);
    if (threadIdx.x < 7) {
      double acc = 0.0;
      for (int i = 0; i < kBlockRows; ++i)
        if (use[i]) acc = dadd(acc, v[i][threadIdx.x]);
      it.sums[(size_t)e * 8 + threadIdx.x] = acc;
    }
    if (threadIdx.x == 0) it.counts[e] = cnt;
    __syncthreads();                     // v and use are reused by the next item
  }
}

// sums 0..6 of pair p over its blocks in ascending block order (lane q of the caller sums quantity q)
__device__ __forceinline__ double block_sum(const double* __restrict__ sums, int P, int p, int nblk, int q) {
  double acc = 0.0;
  for (int k = 0; k < nblk; ++k) acc = dadd(acc, sums[((size_t)k * P + p) * 8 + q]);
  return acc;
}

__device__ __forceinline__ int block_count(const int* __restrict__ counts, int P, int p, int nblk) {
  int n = 0;
  for (int k = 0; k < nblk; ++k) n += counts[(size_t)k * P + p];
  return n;
}

__global__ void __launch_bounds__(kBlockRows)
icp_covariance_kernel(const float* __restrict__ points, const PairState* __restrict__ st, int P,
                      const int* __restrict__ max_blocks, Items it) {
  __shared__ double v[kBlockRows][6];
  __shared__ unsigned char use[kBlockRows];
  __shared__ double csum[6];
  __shared__ int cnt;
  const int items = P * __ldg(max_blocks);                  // P * ceil(N / 256) * 256 is within int32 (host check)
  for (int e = blockIdx.x; e < items; e += gridDim.x) {
    const int k = e / P, p = e - k * P;
    if (!st[p].active || k >= st[p].nblk) continue;          // uniform across the CTA
    const int nblk = st[p].nblk;
    if (threadIdx.x < 6) csum[threadIdx.x] = block_sum(it.sums, P, p, nblk, threadIdx.x);
    if (threadIdx.x == 32) cnt = block_count(it.counts, P, p, nblk);
    __syncthreads();
    const int r = k * kBlockRows + threadIdx.x;
    const int j = r < st[p].n_src ? it.corr[(size_t)e * kBlockRows + threadIdx.x] : -1;
    if (j >= 0) {
      const double m = (double)cnt;
      float s[3], t[3];
      double q[3];
      load3(points, st[p].src_lo + r, s);
      load3(points, j, t);
      transform(st[p].T, s, q);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        v[threadIdx.x][a] = dsub(q[a], ddiv(csum[a], m));
        v[threadIdx.x][3 + a] = dsub(t[a], ddiv(csum[3 + a], m));
      }
    }
    use[threadIdx.x] = j >= 0;
    __syncthreads();
    if (threadIdx.x < 9) {
      const int a = threadIdx.x / 3, b = threadIdx.x - 3 * a;
      double acc = 0.0;
      for (int i = 0; i < kBlockRows; ++i)
        if (use[i]) acc = dadd(acc, dmul(v[i][a], v[i][3 + b]));
      it.cov[(size_t)e * 9 + threadIdx.x] = acc;
    }
    __syncthreads();                     // v, use, csum and cnt are reused by the next item
  }
}

// evaluation `iter` (0 .. I) of every active pair: the scores of its current pose, then stop or update
__global__ void __launch_bounds__(kFinalizeWarps * 32)
icp_finalize_kernel(PairState* __restrict__ st, int P, Items it, int iter, int I, double rel_fitness,
                    double rel_rmse, const double* __restrict__ init, double* __restrict__ pose,
                    double* __restrict__ fitness, double* __restrict__ inlier_rmse, int* __restrict__ n_corr,
                    int* __restrict__ iterations) {
  __shared__ double sums[kFinalizeWarps][16];
  __shared__ int cnts[kFinalizeWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int p = blockIdx.x * kFinalizeWarps + warp;
  if (p >= P || !st[p].active) return;                         // uniform across the warp
  const int nblk = st[p].nblk;
  if (lane < 7) sums[warp][lane] = block_sum(it.sums, P, p, nblk, lane);
  if (lane == 7) cnts[warp] = block_count(it.counts, P, p, nblk);
  if (lane >= 8 && lane < 17 && iter < I) {     // the cross-covariance (no covariance pass after the last update)
    double acc = 0.0;
    for (int k = 0; k < nblk; ++k) acc = dadd(acc, it.cov[((size_t)k * P + p) * 9 + (lane - 8)]);
    sums[warp][lane - 1] = acc;                 // H[a][b] at 7 + 3a + b
  }
  __syncwarp();
  if (lane != 0) return;
  PairState s = st[p];
  const int n = cnts[warp];
  const double m = (double)n;
  const double fit = ddiv(m, (double)s.n_src);
  const double rmse = n > 0 ? dsqrt(ddiv(sums[warp][6], m)) : 0.0;
  bool stop = iter > 0 && fabs(dsub(fit, s.fit)) < rel_fitness && fabs(dsub(rmse, s.rmse)) < rel_rmse;
  stop = stop || iter == I || n < 3;
  if (stop) {
    double* out = pose + (size_t)p * 16;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
      for (int b = 0; b < 3; ++b) out[4 * a + b] = s.T.R[a][b];
      out[4 * a + 3] = s.T.t[a];
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) out[12 + b] = init[(size_t)p * 16 + 12 + b];   // U T keeps the last row of T
    fitness[p] = fit;
    inlier_rmse[p] = rmse;
    n_corr[p] = n;
    iterations[p] = iter;
    st[p].active = 0;
    return;
  }
  double cs[3], ct[3], H[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    cs[a] = ddiv(sums[warp][a], m);
    ct[a] = ddiv(sums[warp][3 + a], m);
#pragma unroll
    for (int b = 0; b < 3; ++b) H[a][b] = sums[warp][7 + 3 * a + b];
  }
  Pose U;
  pose_from_moments(cs, ct, H, U);
  // T_{i+1} = U T_i: R' = Ru R, t' = Ru t + tu, each entry ((x_0 y_0 + x_1 y_1) + x_2 y_2) (+ tu)
  Pose T;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int b = 0; b < 3; ++b)
      T.R[a][b] = dadd(dadd(dmul(U.R[a][0], s.T.R[0][b]), dmul(U.R[a][1], s.T.R[1][b])), dmul(U.R[a][2], s.T.R[2][b]));
    T.t[a] = dadd(dadd(dadd(dmul(U.R[a][0], s.T.t[0]), dmul(U.R[a][1], s.T.t[1])), dmul(U.R[a][2], s.T.t[2])), U.t[a]);
  }
  st[p].T = T;
  st[p].fit = fit;
  st[p].rmse = rmse;
}

struct Work {
  int* start;
  int* max_blocks;
  PairState* st;
  Items it;
  void* nb;
  size_t nb_bytes;
};

// fp32 grid radius: tau rounded up, so that the grid's cells cover tau (nbgrid.cuh)
float grid_radius(double distance) {
  float r = (float)distance;
  if ((double)r < distance) r = nextafterf(r, INFINITY);
  return r;
}

long long item_count(int N, int P) { return (long long)P * ((N + kBlockRows - 1) / kBlockRows); }

// every size the workspace depends on, or 0
size_t workspace_layout(int N, int B, int P, double distance, const float* host_bbox, Work* w, void* base) {
  if (N < 0 || B < 1 || B > kMaxBatch || P < 1 || host_bbox == nullptr || !std::isfinite(distance) || !(distance > 0))
    return 0;
  const long long items = item_count(N, P);
  if (items * kBlockRows > INT32_MAX) return 0;
  const float r = grid_radius(distance);
  const NbGrid g = make_grid(host_bbox, r);
  if (g.ncells * B > kMaxGridCells || !nearest_lookup_exact(g, host_bbox)) return 0;
  const size_t nb = d3f_radius_neighbors_workspace_bytes(N, B, r, host_bbox);
  if (nb == 0) return 0;
  Carver cv(base);
  Work x;
  x.start = cv.take<int>(B + 1);
  x.max_blocks = cv.take<int>(1);
  x.st = cv.take<PairState>(P);
  x.it.corr = cv.take<int>((size_t)items * kBlockRows);
  x.it.sums = cv.take<double>((size_t)items * 8);
  x.it.counts = cv.take<int>((size_t)items);
  x.it.cov = cv.take<double>((size_t)items * 9);
  x.nb = cv.take<char>(nb);
  x.nb_bytes = nb;
  if (w != nullptr) *w = x;
  return cv.off;
}

}  // namespace
}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_icp_pairs_workspace_bytes(int N, int B, int P, double distance, const float* host_bbox) {
  return workspace_layout(N, B, P, distance, host_bbox, nullptr, nullptr);
}

extern "C" int d3f_icp_pairs(const float* points, const int* lengths, int B, int N, const int* n_dev,
                             const float* host_bbox, const int* pairs, int P, const double* init, double distance,
                             int max_iterations, double relative_fitness, double relative_rmse, double* pose,
                             double* fitness, double* inlier_rmse, int* n_corr, int* iterations, void* workspace,
                             size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "icp_pairs: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(N >= 0 && P >= 1, D3F_ERR_INVALID, "icp_pairs: bad shape N=%d P=%d", N, P);
  D3F_REQUIRE(max_iterations >= 0 && max_iterations <= 1024, D3F_ERR_INVALID,
              "icp_pairs: max_iterations=%d must be in [0,1024]", max_iterations);
  D3F_REQUIRE(std::isfinite(distance) && distance > 0.0, D3F_ERR_INVALID,
              "icp_pairs: distance=%g must be finite and > 0", distance);
  D3F_REQUIRE(std::isfinite(relative_fitness) && relative_fitness >= 0.0 && std::isfinite(relative_rmse) &&
                  relative_rmse >= 0.0,
              D3F_ERR_INVALID, "icp_pairs: relative_fitness=%g and relative_rmse=%g must be finite and >= 0",
              relative_fitness, relative_rmse);
  D3F_REQUIRE(points && lengths && host_bbox && pairs && init && pose && fitness && inlier_rmse && n_corr &&
                  iterations && workspace,
              D3F_ERR_INVALID, "icp_pairs: null pointer");
  D3F_REQUIRE(item_count(N, P) * kBlockRows <= INT32_MAX, D3F_ERR_INVALID,
              "icp_pairs: P*ceil(N/256)*256 exceeds int32 (N=%d P=%d)", N, P);
  const float r = grid_radius(distance);
  const NbGrid g = make_grid(host_bbox, r);
  D3F_REQUIRE(g.ncells * B <= kMaxGridCells, D3F_ERR_INVALID,
              "icp_pairs: grid %d x %d x %d x %d clouds at distance %g exceeds %lld cells", g.nx, g.ny, g.nz, B,
              distance, kMaxGridCells);
  D3F_REQUIRE(nearest_lookup_exact(g, host_bbox), D3F_ERR_INVALID,
              "icp_pairs: host_bbox coordinates beyond 1024 cells (of distance * 1.001) from the origin");
  Work w;
  const size_t need = workspace_layout(N, B, P, distance, host_bbox, &w, workspace);
  D3F_REQUIRE(workspace_bytes >= need, D3F_ERR_WORKSPACE, "icp_pairs: workspace too small (%zu < %zu bytes)",
              workspace_bytes, need);
  if (launch_batch_start(lengths, B, w.start, stream)) return D3F_ERR_CUDA;
  int rc = radius_neighbors_build(points, lengths, B, N, r, host_bbox, w.nb, w.nb_bytes, stream, n_dev, w.start);
  if (rc) return rc;
  NbView view;
  rc = radius_neighbors_view(w.nb, N, B, r, host_bbox, &view);
  if (rc) return rc;
  icp_prepare_kernel<<<1, kPrepareThreads, 0, stream>>>(N, n_dev, w.start, B, pairs, P, init, w.st, w.max_blocks,
                                                        pose, fitness, inlier_rmse, n_corr, iterations);
  D3F_LAUNCH_CHECK("icp_prepare_kernel");
  const long long items = item_count(N, P);
  if (items == 0) return D3F_OK;         // no rows: every pair keeps init
  const int grid = (int)std::min<long long>(items, (long long)kItemCtasPerSM * kNumSMs);
  const double tau2 = distance * distance;
  for (int iter = 0; iter <= max_iterations; ++iter) {
    icp_correspond_kernel<<<grid, kBlockRows, 0, stream>>>(points, view, w.st, P, w.max_blocks, tau2, w.it);
    D3F_LAUNCH_CHECK("icp_correspond_kernel");
    if (iter < max_iterations) {
      icp_covariance_kernel<<<grid, kBlockRows, 0, stream>>>(points, w.st, P, w.max_blocks, w.it);
      D3F_LAUNCH_CHECK("icp_covariance_kernel");
    }
    icp_finalize_kernel<<<ceil_div(P, kFinalizeWarps), kFinalizeWarps * 32, 0, stream>>>(
        w.st, P, w.it, iter, max_iterations, relative_fitness, relative_rmse, init, pose, fitness, inlier_rmse, n_corr,
        iterations);
    D3F_LAUNCH_CHECK("icp_finalize_kernel");
  }
  return D3F_OK;
}

// The hash grid of neighbors.cu (cell edge = radius * 1.001, one dense cell table per cloud) and the fp64 queries
// over it that ICP (icp.cu) and the training-pair correspondences (correspond.cu) use. The fp32 radius queries live
// in neighbors.cu.
#pragma once
#include <math.h>

#include "common.cuh"

namespace d3f {

struct NbGrid {
  float minx, miny, minz, inv_cell;
  int nx, ny, nz;
  long long ncells;  // per cloud
};

static NbGrid make_grid(const float* host_bbox, float radius) {
  NbGrid g;
  float cell = radius * 1.001f;
  g.inv_cell = 1.0f / cell;
  g.minx = host_bbox[0];
  g.miny = host_bbox[1];
  g.minz = host_bbox[2];
  auto dim = [&](int a) {
    double ext = (double)host_bbox[3 + a] - (double)host_bbox[a];
    if (!(ext >= 0)) ext = 0;
    double n = floor(ext / (double)cell) + 2.0;
    return n > 2.0e9 ? 2000000000 : (int)n;
  };
  g.nx = dim(0);
  g.ny = dim(1);
  g.nz = dim(2);
  g.ncells = (long long)g.nx * g.ny * g.nz;
  return g;
}

constexpr long long kMaxGridCells = 1ll << 27;  // 128 Mi cells total (2 x 4 B tables = 1 GiB)

// Why the 27 cells around a query's cell hold every support with fp32 d2 < r2 (the radius search of neighbors.cu),
// and up to which axis length. Queries and supports are fp32 points, r2 = fl(r * r), cell edge c = fl(r * 1.001f),
// inv = fl(1 / c), and along one axis the cell of v is
//   idx(v) = clamp(floor(Y(v)), 0, n - 1),   Y(v) = fl(fl(v - mn) * inv),
// monotone in v. A hit has fl(dx * dx) <= d2 < r2 (fp32 sums of non-negative terms), so |fl(q - s)| < r (1 + 2^-24)
// and |q - s| < r (1 + 2^-23) on every axis. With E(v) = (v - mn) / c exact, (b - a) * inv (1 + 2^-24)^2 <
// (1 + 3.5 2^-24) / 1.001f < 0.9990012 cells for a hit's coordinates a < b. Each of Y's two roundings has relative
// error at most u = 2^-24, so Y(b) - Y(a) < 0.9990012 + 4 u E(a): below one cell, and the floors at most one apart,
// while E(a) < 9.988e-4 / (4 u) = 4189 cells. That covers every pair when n <= 4189 cells per axis: if E(a) >= n,
// Y(a) >= n (1 - 2u) > n - 1, so a and every b >= a clamp to the edge cell n - 1; if a < mn, E(b) < 1 and Y(b) < 1,
// so both clamp to cell 0 or b is in cell 0. kMaxScanAxisCells = 4096 keeps a margin; past it a pair inside the
// radius can sit two cells apart. Distance from the origin does not enter: v and mn are fp32, so only the extent in
// cells does. Grids past the bound are refused on the host (neighbors.cu).
constexpr int kMaxScanAxisCells = 4096;

static inline bool radius_scan_complete(const NbGrid& g) {
  return g.nx <= kMaxScanAxisCells && g.ny <= kMaxScanAxisCells && g.nz <= kMaxScanAxisCells;
}

__device__ __forceinline__ int cell_coord(float v, float mn, float inv, int n) {
  int c = (int)floorf((v - mn) * inv);
  return min(max(c, 0), n - 1);
}

// A built grid: sorted_pts[Ns] = (x, y, z, bits(row)) in cell order, the run of cell c = [cell_start[c], cell_start[c+1]).
struct NbView {
  NbGrid g;
  const float4* sorted_pts;
  const int* cell_start;
};

// ---- the rows of one cloud around an fp64 query ---------------------------------------------------------------
// The query q is fp64 (a transformed fp32 point); d^2 = (e_0^2 + e_1^2) + e_2^2 with e_a = q_a - s_a, one rounding per
// operation, as residual2 in solver.cuh. visit_cloud_rows calls f(row, d^2) for every row of cloud b in the 27 cells
// around the cell of (float)q; the callers keep the rows with d^2 < tau2 (a NaN d^2 never qualifies). The nearest row
// (nearest_in_cloud) is the one with the smallest d^2 < tau2, ties to the smaller row.
//
// Why the 27 cells around the cell of (float)q hold every row with d^2 < tau2 -- all of them, not only the nearest
// (tau2 = tau * tau, grid radius r >= tau as an fp32, cell edge c = fl(r * 1.001f)): along one axis the cell index is
//   idx(x) = clamp(floor(fl(fl(fl32(x) - mn) * inv)), 0, n - 1),   inv = fl(1 / c),
// a composition of monotone maps (round to fp32, subtract / multiply by positive constants with round to nearest,
// floor, clamp), so it is monotone in the real x. Every row s with d^2 < tau2 has |q_a - s_a| <= tau (1 + 2^-50) on
// every axis, so idx(s_a) lies between idx(q_a - tau') and idx(q_a + tau'); the scan is conservative when any two reals
// a < b with b - a <= tau' get indices at most one apart. Exactly, (b - a) * inv <= tau' / (r * 1.001 (1 - 2^-24))
// (1 + 2^-24) < 0.999002 cells, leaving a margin of 9.98e-4 cells for the roundings. If every bbox coordinate lies
// within M = 1024 cells of the origin (checked on the host, nearest_lookup_exact), a point x within two cells of the
// box has |x| <= (M + 2) c and |x - mn| <= (2M + 4) c, so its three roundings move fl(...) by at most
// 2^-24 ((M + 2) + 2 (2M + 4)) < 3.1e-4 cells, 6.2e-4 for the two points: below the margin, so the floors differ by at
// most one. A point more than two cells outside the box pins, with the other point (within one cell of it), both
// indices to the same edge cell or to the edge cell and its neighbour (monotonicity, and fl(...) of a point one cell
// outside the box is within 1e-3 of its exact value), so the clamp keeps them within one. Non-finite queries have no
// row within tau and are not looked up; a query beyond the fp32 range rounds to +-inf and clamps to an edge cell.
static inline bool nearest_lookup_exact(const NbGrid& g, const float* host_bbox) {
  for (int a = 0; a < 3; ++a) {
    const double m = fmax(fabs((double)host_bbox[a]), fabs((double)host_bbox[3 + a]));
    if (!(m * (double)g.inv_cell <= 1024.0)) return false;
  }
  return true;
}

struct Nearest {
  int row;       // -1: no row with d^2 < tau2
  double d2;     // tau2 when there is none
};

template <typename F>
__device__ __forceinline__ void visit_cloud_rows(const NbView& v, int b, double q0, double q1, double q2, F&& f) {
  const double q[3] = {q0, q1, q2};
  if (isfinite(q0) && isfinite(q1) && isfinite(q2)) {
    const NbGrid& g = v.g;
    const int cx = cell_coord((float)q[0], g.minx, g.inv_cell, g.nx);
    const int cy = cell_coord((float)q[1], g.miny, g.inv_cell, g.ny);
    const int cz = cell_coord((float)q[2], g.minz, g.inv_cell, g.nz);
    const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.nx - 1);
    for (int zz = max(cz - 1, 0); zz <= min(cz + 1, g.nz - 1); ++zz) {
      for (int yy = max(cy - 1, 0); yy <= min(cy + 1, g.ny - 1); ++yy) {
        // cells x0..x1 of one (y, z) row are adjacent in the table: one contiguous run of sorted_pts
        const int row = b * (int)g.ncells + (zz * g.ny + yy) * g.nx;
        const int e = __ldg(v.cell_start + row + x1 + 1);
        for (int i = __ldg(v.cell_start + row + x0); i < e; ++i) {
          const float4 s = __ldg(v.sorted_pts + i);
          const double e0 = __dsub_rn(q[0], (double)s.x), e1 = __dsub_rn(q[1], (double)s.y);
          const double e2 = __dsub_rn(q[2], (double)s.z);
          const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(e0, e0), __dmul_rn(e1, e1)), __dmul_rn(e2, e2));
          f((int)__float_as_uint(s.w), d2);
        }
      }
    }
  }
}

// nearest_in_cloud walks the cells itself: written over visit_cloud_rows, ICP's correspond kernel takes a stack frame
__device__ __forceinline__ Nearest nearest_in_cloud(const NbView& v, int b, double q0, double q1, double q2,
                                                    double tau2) {
  const double q[3] = {q0, q1, q2};
  double best_d2 = tau2;
  int best = -1;                        // d2 == tau2 never wins: no row is below -1
  if (isfinite(q0) && isfinite(q1) && isfinite(q2)) {
    const NbGrid& g = v.g;
    const int cx = cell_coord((float)q[0], g.minx, g.inv_cell, g.nx);
    const int cy = cell_coord((float)q[1], g.miny, g.inv_cell, g.ny);
    const int cz = cell_coord((float)q[2], g.minz, g.inv_cell, g.nz);
    const int x0 = max(cx - 1, 0), x1 = min(cx + 1, g.nx - 1);
    for (int zz = max(cz - 1, 0); zz <= min(cz + 1, g.nz - 1); ++zz) {
      for (int yy = max(cy - 1, 0); yy <= min(cy + 1, g.ny - 1); ++yy) {
        // cells x0..x1 of one (y, z) row are adjacent in the table: one contiguous run of sorted_pts
        const int row = b * (int)g.ncells + (zz * g.ny + yy) * g.nx;
        const int e = __ldg(v.cell_start + row + x1 + 1);
        for (int i = __ldg(v.cell_start + row + x0); i < e; ++i) {
          const float4 s = __ldg(v.sorted_pts + i);
          const double e0 = __dsub_rn(q[0], (double)s.x), e1 = __dsub_rn(q[1], (double)s.y);
          const double e2 = __dsub_rn(q[2], (double)s.z);
          const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(e0, e0), __dmul_rn(e1, e1)), __dmul_rn(e2, e2));
          const int j = (int)__float_as_uint(s.w);
          if (d2 < best_d2 || (d2 == best_d2 && j < best)) {
            best_d2 = d2;
            best = j;
          }
        }
      }
    }
  }
  return Nearest{best, best_d2};
}

}  // namespace d3f

/* TEST INFRASTRUCTURE ONLY -- not part of the product path.
 *
 * CPU restatement ("port") of Open3D 0.7's VoxelDownSample (Geometry/DownSample.cpp) over stacked clouds, the
 * contract of d3f_voxel_down_sample (include/d3feat_b200.h). Written from the semantics of that function; Open3D is
 * not part of the reference tree and no Open3D binary was run against it.
 *
 * The literal loop, per cloud: bounds over the finite rows, one fp64 voxel index per row, fp64 accumulation per voxel
 * in input order, then the canonical order (ascending (iz, iy, ix)) instead of std::unordered_map's.
 *
 * Compile: gcc -std=c11 -O2 -ffp-contract=off (no FMA contraction: every operation rounds separately).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef struct {
  int64_t ix, iy, iz;
  int32_t row;
} VoxelRow;

static int cmp_voxel_row(const void* a, const void* b) {
  const VoxelRow* x = (const VoxelRow*)a;
  const VoxelRow* y = (const VoxelRow*)b;
  if (x->iz != y->iz) return x->iz < y->iz ? -1 : 1;
  if (x->iy != y->iy) return x->iy < y->iy ? -1 : 1;
  if (x->ix != y->ix) return x->ix < y->ix ? -1 : 1;
  return (x->row > y->row) - (x->row < y->row);
}

/* pts[N,3]; lengths[B]: cloud b holds rows [start_b, start_b + lengths[b]) cut at N (start = exclusive scan).
 * out_pts holds N rows (upper bound), out_lengths[B]. Returns the number of voxels M. */
int orc_voxel_down_sample(const float* pts, int N, const int* lengths, int B, double v, float* out_pts,
                          int* out_lengths) {
  VoxelRow* rows = (VoxelRow*)malloc(sizeof(VoxelRow) * (size_t)(N > 0 ? N : 1));
  int64_t start = 0;
  int M = 0;
  for (int b = 0; b < B; ++b) {
    int64_t s = start < N ? start : N;
    int64_t e = start + lengths[b];
    if (e > N) e = N;
    if (e < s) e = s;
    start += lengths[b];
    out_lengths[b] = 0;
    /* bounds of the finite rows: min_bound - voxel_size * 0.5 */
    double mn[3] = {INFINITY, INFINITY, INFINITY};
    int n = 0;
    for (int64_t i = s; i < e; ++i) {
      const float* p = pts + 3 * i;
      if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) continue;
      for (int a = 0; a < 3; ++a)
        if ((double)p[a] < mn[a]) mn[a] = (double)p[a];
      ++n;
    }
    if (n == 0) continue;
    double lo[3];
    for (int a = 0; a < 3; ++a) lo[a] = mn[a] - v * 0.5;
    n = 0;
    for (int64_t i = s; i < e; ++i) {
      const float* p = pts + 3 * i;
      if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) continue;
      rows[n].ix = (int64_t)floor(((double)p[0] - lo[0]) / v);
      rows[n].iy = (int64_t)floor(((double)p[1] - lo[1]) / v);
      rows[n].iz = (int64_t)floor(((double)p[2] - lo[2]) / v);
      rows[n].row = (int32_t)i;
      ++n;
    }
    qsort(rows, (size_t)n, sizeof(VoxelRow), cmp_voxel_row);
    for (int i = 0; i < n;) {
      double sum[3] = {0.0, 0.0, 0.0};
      int j = i;
      for (; j < n && rows[j].ix == rows[i].ix && rows[j].iy == rows[i].iy && rows[j].iz == rows[i].iz; ++j)
        for (int a = 0; a < 3; ++a) sum[a] += (double)pts[3 * (int64_t)rows[j].row + a];
      for (int a = 0; a < 3; ++a) out_pts[3 * (int64_t)M + a] = (float)(sum[a] / (double)(j - i));
      ++M;
      ++out_lengths[b];
      i = j;
    }
  }
  free(rows);
  return M;
}

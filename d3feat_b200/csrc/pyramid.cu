// The input pyramid of the encoder as ONE host call: mirror of the loop in Dataset.tf_descriptor_input
// (datasets/common.py:1325-1397) with big_neighborhood_filter (:399-406) folded in.
//
// Per level: conv neighbours, grid subsampling, pool neighbours, upsample neighbours. A hash grid is keyed by
// (level, radius) and reused by every search over the same supports and radius (the reference's 13 radius searches
// need 5 grids for the standard architecture). The only device->host reads are the cell counts after each
// subsampling (the next level's launch sizes depend on them).
#include <math.h>

#include "ops.cuh"

namespace d3f {

namespace {

struct GridSlot {
  int level;
  float radius;
  void* ws;
  size_t bytes;
  bool built;   // set by the build when it first searches this grid
};

inline bool same_radius(float a, float b) { return fabsf(a - b) <= 1e-6f * fmaxf(fabsf(a), fabsf(b)); }

struct PyramidWs {
  void* sub;   // the subsampling workspace, sized for level 0 and reused by every level
  size_t sub_bytes;
  int* starts;   // [D3F_MAX_LEVELS][B + 1] exclusive scans of every level's lengths
  int* counts;   // [D3F_MAX_LEVELS] level row counts, when the caller keeps none
  int* status;   // [1], when the caller keeps none
  GridSlot slots[3 * D3F_MAX_LEVELS];   // in build order
  int n_slots;
};

// The grids are listed in the order the build first uses them: per level l the conv grid over level l, then, when
// level l is subsampled into level l + 1, the pool grid over level l and the upsample grid over level l + 1. A grid is
// keyed by (level, radius) and sized with the row capacity of its level; a radius <= 0 has none.
size_t pyramid_layout(int B, const d3f_pyramid_spec* spec, const int* capacity, const float* host_bbox, void* base,
                      PyramidWs* w_out) {
  if (spec == nullptr || capacity == nullptr || host_bbox == nullptr) return 0;
  const int L = spec->n_levels;
  if (L < 1 || L > D3F_MAX_LEVELS) return 0;
  Carver cv(base);
  PyramidWs w;
  w.sub_bytes = d3f_grid_subsample_workspace_bytes(capacity[0], B);
  w.sub = cv.take<char>(w.sub_bytes);
  w.starts = cv.take<int>((size_t)D3F_MAX_LEVELS * (B + 1));
  w.counts = cv.take<int>(D3F_MAX_LEVELS);
  w.status = cv.take<int>(1);
  w.n_slots = 0;
  auto add = [&](int l, float radius) {
    if (!(radius > 0.f)) return true;
    for (int i = 0; i < w.n_slots; ++i)
      if (w.slots[i].level == l && same_radius(w.slots[i].radius, radius)) return true;
    const size_t nb = d3f_radius_neighbors_workspace_bytes(capacity[l], B, radius, host_bbox);
    if (nb == 0) return false;
    GridSlot& g = w.slots[w.n_slots++];
    g.level = l;
    g.radius = radius;
    g.ws = cv.take<char>(nb);
    g.bytes = nb;
    g.built = false;
    return true;
  };
  for (int l = 0; l < L; ++l) {
    if (!add(l, spec->conv_radius[l])) return 0;
    if (spec->sub_dl[l] > 0.f && l + 1 < L && !(add(l, spec->pool_radius[l]) && add(l + 1, spec->up_radius[l])))
      return 0;
  }
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

}  // namespace

__global__ void set_count_kernel(int* __restrict__ dst, int value, const int* __restrict__ src) {
  *dst = src ? *src : value;
}

}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_pyramid_workspace_bytes(int B, const d3f_pyramid_spec* spec, const int* capacity,
                                              const float* host_bbox) {
  return pyramid_layout(B, spec, capacity, host_bbox, nullptr, nullptr);
}

// Two ways to run it:
//  * exact (out_level_sizes != nullptr): after every subsampling the number of cells is read back (one host
//    synchronisation per level) so that the next level's launches and the caller's tensor views have exact sizes --
//    what the TF ops do, and what the stand-alone op mirrors / parity tests use;
//  * static (out_level_sizes == nullptr): nothing is read back. Every launch is sized by capacity[l], every kernel
//    takes its row count from d_counts[l] in device memory, errors (more cells than capacity[l+1], a cloud wider than the
//    bbox) are OR-ed into *d_status. The launch sequence then depends on nothing but (B, capacity, spec, bbox): it
//    can be captured once as a CUDA graph and replayed for every batch of the bucket.
// d_counts[0] is N0, or *n0_dev when the caller keeps the level-0 count on the device (graph replay: N0 = capacity[0]).
extern "C" int d3f_pyramid_build(const float* points, const int* lengths, int B, int N0, const d3f_pyramid_spec* spec,
                                 const float* host_bbox, float* const* out_points, int* const* out_lengths,
                                 int* const* out_neighbors, int* const* out_pools, int* const* out_upsamples,
                                 const int* capacity, int* out_level_sizes, void* workspace, size_t workspace_bytes,
                                 d3f_stream_t stream_, int* d_counts, int* d_status, const int* n0_dev) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE((points != nullptr || N0 == 0) && lengths != nullptr && out_points && out_lengths && out_neighbors &&
                  out_pools && out_upsamples && workspace,
              D3F_ERR_INVALID, "d3f_pyramid_build: null pointer");
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "d3f_pyramid_build: B=%d", B);
  D3F_REQUIRE(spec != nullptr && capacity != nullptr && host_bbox != nullptr, D3F_ERR_INVALID,
              "pyramid_build: null argument");
  const bool exact = out_level_sizes != nullptr;
  D3F_REQUIRE(exact || (d_counts != nullptr && d_status != nullptr), D3F_ERR_INVALID,
              "pyramid_build: the static form needs d_counts and d_status");
  const int L = spec->n_levels;
  D3F_REQUIRE(L >= 1 && L <= D3F_MAX_LEVELS, D3F_ERR_INVALID, "pyramid_build: n_levels=%d", L);
  D3F_REQUIRE(N0 >= 0 && N0 <= capacity[0], D3F_ERR_CAPACITY, "pyramid_build: N0=%d exceeds capacity %d", N0, capacity[0]);
  PyramidWs w;
  const size_t need = pyramid_layout(B, spec, capacity, host_bbox, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE,
              "pyramid_build: workspace too small (or grid too large)");

  // start[l][b] = first row of cloud b at level l: scanned ONCE per level (every grid build, search and subsampling
  // of that level used to launch its own scan: 22 launches per step instead of 5)
  int* starts = w.starts;
  if (launch_batch_start(lengths, B, starts, stream)) return D3F_ERR_CUDA;
  // level counts and status live in the caller's buffers, or (exact form without them) in the workspace
  int* counts = d_counts != nullptr ? d_counts : w.counts;
  int* status = d_status != nullptr ? d_status : w.status;
  if (d_status == nullptr) D3F_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  set_count_kernel<<<1, 1, 0, stream>>>(counts, N0, n0_dev);
  D3F_LAUNCH_CHECK("set_count_kernel");

  const float* lvl_pts[D3F_MAX_LEVELS];
  const int* lvl_len[D3F_MAX_LEVELS];
  int lvl_n[D3F_MAX_LEVELS];   // launch size of level l: exact form = its row count, static form = its capacity
  lvl_pts[0] = points;
  lvl_len[0] = lengths;
  lvl_n[0] = exact ? N0 : capacity[0];

  // returns the grid of the layout over level `l` at `radius`, building it on first use
  auto grid_for = [&](int l, float radius, GridSlot** out) -> int {
    for (int i = 0; i < w.n_slots; ++i) {
      GridSlot& g = w.slots[i];
      if (g.level != l || !same_radius(g.radius, radius)) continue;
      *out = &g;
      if (g.built) return D3F_OK;
      g.built = true;
      return radius_neighbors_build(lvl_pts[l], lvl_len[l], B, lvl_n[l], radius, host_bbox, g.ws, g.bytes, stream,
                                    counts + l, starts + (size_t)l * (B + 1));
    }
    d3f::set_error("pyramid_build: radius=%g at level %d must be > 0", (double)radius, l);
    return D3F_ERR_INVALID;
  };
  // the workspace of a grid is carved with the CAPACITY of its level (the query side re-derives the same layout)
  auto fill = [&](int lq, int ls, GridSlot* g, int lim, int* out) -> int {
    return radius_neighbors_fill(lvl_pts[lq], lvl_len[lq], lvl_n[lq], B, lvl_n[ls], g->radius, host_bbox, g->ws, lim,
                                 lvl_n[ls], out, stream, counts + lq, counts + ls, starts + (size_t)lq * (B + 1));
  };

  for (int l = 0; l < L; ++l) {
    const int lim = spec->limit[l];
    D3F_REQUIRE(lim >= 1, D3F_ERR_INVALID, "pyramid_build: limit[%d]=%d", l, lim);
    if (exact) out_level_sizes[l] = lvl_n[l];
    GridSlot* g = nullptr;
    if (spec->conv_radius[l] > 0.f) {
      int rc = grid_for(l, spec->conv_radius[l], &g);
      if (rc) return rc;
      rc = fill(l, l, g, lim, out_neighbors[l]);
      if (rc) return rc;
    }
    if (spec->sub_dl[l] > 0.f && l + 1 < L) {
      D3F_REQUIRE(out_points[l + 1] != nullptr && out_lengths[l + 1] != nullptr, D3F_ERR_INVALID,
                  "pyramid_build: missing output buffers for level %d", l + 1);
      int* d_M = counts + l + 1;
      int rc = grid_subsample(lvl_pts[l], lvl_len[l], B, lvl_n[l], spec->sub_dl[l], nullptr, 0, nullptr, 0, host_bbox,
                              out_points[l + 1], nullptr, nullptr, out_lengths[l + 1], d_M, w.sub, w.sub_bytes,
                              stream, counts + l, capacity[l + 1], status, starts + (size_t)l * (B + 1));
      if (rc) return rc;
      if (launch_batch_start(out_lengths[l + 1], B, starts + (size_t)(l + 1) * (B + 1), stream)) return D3F_ERR_CUDA;
      int M = capacity[l + 1];
      if (exact) {
        D3F_CUDA(cudaMemcpyAsync(&M, d_M, sizeof(int), cudaMemcpyDeviceToHost, stream));
        D3F_CUDA(cudaStreamSynchronize(stream));
        D3F_REQUIRE(M != -1, D3F_ERR_CAPACITY, "pyramid_build: a cloud at level %d is wider than the supplied bbox allows", l);
        D3F_REQUIRE(M >= 0, D3F_ERR_CAPACITY, "pyramid_build: level %d exceeds its capacity %d", l + 1, capacity[l + 1]);
      }
      lvl_pts[l + 1] = out_points[l + 1];
      lvl_len[l + 1] = out_lengths[l + 1];
      lvl_n[l + 1] = M;
      // pool: queries = level l+1, supports = level l
      rc = grid_for(l, spec->pool_radius[l], &g);
      if (rc) return rc;
      rc = fill(l + 1, l, g, lim, out_pools[l]);
      if (rc) return rc;
      // upsample: queries = level l, supports = level l+1
      rc = grid_for(l + 1, spec->up_radius[l], &g);
      if (rc) return rc;
      rc = fill(l, l + 1, g, lim, out_upsamples[l]);
      if (rc) return rc;
    } else if (l + 1 < L) {
      D3F_REQUIRE(false, D3F_ERR_INVALID, "pyramid_build: level %d has no subsampling but is not the last level", l);
    }
  }
  return D3F_OK;
}

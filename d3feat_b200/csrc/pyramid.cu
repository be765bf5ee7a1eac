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
};

struct PyramidPlan {
  int L;
  const d3f_pyramid_spec* spec;
};

inline bool same_radius(float a, float b) { return fabsf(a - b) <= 1e-6f * fmaxf(fabsf(a), fabsf(b)); }

}  // namespace

__global__ void set_count_kernel(int* __restrict__ dst, int value, const int* __restrict__ src) {
  *dst = src ? *src : value;
}

}  // namespace d3f

using namespace d3f;

// Workspace: one subsampling workspace (level-0 sized) + one grid workspace per distinct (level, radius) pair,
// sized with the per-level row capacity.
extern "C" size_t d3f_pyramid_workspace_bytes(int B, const d3f_pyramid_spec* spec, const int* capacity,
                                              const float* host_bbox) {
  if (spec == nullptr || capacity == nullptr || host_bbox == nullptr) return 0;
  int L = spec->n_levels;
  if (L < 1 || L > D3F_MAX_LEVELS) return 0;
  size_t total = align_up(d3f_grid_subsample_workspace_bytes(capacity[0], B) + 512, 256);
  total += align_up(sizeof(int) * (size_t)D3F_MAX_LEVELS * (B + 1), 256);   // exclusive scans of every level's lengths
  for (int l = 0; l < L; ++l) {
    float radii[3] = {spec->conv_radius[l], spec->sub_dl[l] > 0.f ? spec->pool_radius[l] : -1.f,
                      (l > 0 && spec->sub_dl[l - 1] > 0.f) ? spec->up_radius[l - 1] : -1.f};
    for (int a = 0; a < 3; ++a) {
      if (!(radii[a] > 0.f)) continue;
      bool dup = false;
      for (int b = 0; b < a; ++b) dup = dup || (radii[b] > 0.f && same_radius(radii[a], radii[b]));
      if (dup) continue;
      size_t nb = d3f_radius_neighbors_workspace_bytes(capacity[l], B, radii[a], host_bbox);
      if (nb == 0) return 0;
      total += align_up(nb, 256);
    }
  }
  return total + 1024;
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
  D3F_REQUIRE(workspace_bytes >= d3f_pyramid_workspace_bytes(B, spec, capacity, host_bbox) &&
                  d3f_pyramid_workspace_bytes(B, spec, capacity, host_bbox) > 0,
              D3F_ERR_WORKSPACE, "pyramid_build: workspace too small (or grid too large)");

  char* base = (char*)workspace;
  size_t off = 0;
  void* sub_ws = base;
  size_t sub_bytes = align_up(d3f_grid_subsample_workspace_bytes(capacity[0], B) + 512, 256);
  off += sub_bytes;
  // start[l][b] = first row of cloud b at level l: scanned ONCE per level (every grid build, search and subsampling
  // of that level used to launch its own scan: 22 launches per step instead of 5)
  int* starts = (int*)(base + off);
  off += align_up(sizeof(int) * (size_t)D3F_MAX_LEVELS * (B + 1), 256);
  if (launch_batch_start(lengths, B, starts, stream)) return D3F_ERR_CUDA;
  // level counts live in the caller's buffer, or (exact form without one) in the tail of the subsampling region
  int* counts = d_counts != nullptr ? d_counts : (int*)((char*)sub_ws + sub_bytes - 256);
  int* status = d_status != nullptr ? d_status : counts + D3F_MAX_LEVELS;
  if (d_status == nullptr) D3F_CUDA(cudaMemsetAsync(status, 0, sizeof(int), stream));
  set_count_kernel<<<1, 1, 0, stream>>>(counts, N0, n0_dev);
  D3F_LAUNCH_CHECK("set_count_kernel");

  GridSlot slots[3 * D3F_MAX_LEVELS];
  int n_slots = 0;
  const float* lvl_pts[D3F_MAX_LEVELS];
  const int* lvl_len[D3F_MAX_LEVELS];
  int lvl_n[D3F_MAX_LEVELS];   // launch size of level l: exact form = its row count, static form = its capacity
  lvl_pts[0] = points;
  lvl_len[0] = lengths;
  lvl_n[0] = exact ? N0 : capacity[0];

  // returns the grid over level `l` at `radius`, building it on first use
  auto grid_for = [&](int l, float radius, GridSlot** out) -> int {
    for (int i = 0; i < n_slots; ++i)
      if (slots[i].level == l && same_radius(slots[i].radius, radius)) {
        *out = &slots[i];
        return D3F_OK;
      }
    GridSlot& g = slots[n_slots];
    g.level = l;
    g.radius = radius;
    g.bytes = align_up(d3f_radius_neighbors_workspace_bytes(capacity[l], B, radius, host_bbox), 256);
    g.ws = base + off;
    off += g.bytes;
    D3F_REQUIRE(off <= workspace_bytes, D3F_ERR_WORKSPACE, "pyramid_build: workspace exhausted");
    int rc = radius_neighbors_build(lvl_pts[l], lvl_len[l], B, lvl_n[l], radius, host_bbox, g.ws, g.bytes, stream,
                                    counts + l, starts + (size_t)l * (B + 1));
    if (rc) return rc;
    ++n_slots;
    *out = &g;
    return D3F_OK;
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
                              out_points[l + 1], nullptr, nullptr, out_lengths[l + 1], d_M, sub_ws, sub_bytes - 256,
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

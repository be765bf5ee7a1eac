/* d3feat_b200 -- C ABI of the Hopper-native (sm_90a) D3Feat hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / TF types. Every entry point
 *   - takes DEVICE pointers unless a parameter is explicitly marked "host",
 *   - takes an explicit CUDA stream (cudaStream_t passed as void*), enqueues its work there and
 *     returns without synchronising unless stated otherwise,
 *   - never frees or allocates caller-visible memory: scratch comes from the caller-supplied
 *     workspace (size from the matching *_workspace_bytes query),
 *   - returns 0 (D3F_OK) or a negative D3F_ERR_* code; d3f_last_error() gives the message
 *     (thread-local). No exception crosses the boundary.
 *   - keeps no global mutable state: re-entrant across host threads and streams (the reference's
 *     OpKernels are invoked concurrently by the tf.data map pool, datasets/common.py:600,744).
 *
 * Reference interfaces replaced (paths relative to the D3Feat repository):
 *   d3f_grid_subsample        tf_custom_ops/tf_subsampling/tf_batch_subsampling.cpp:8-20,30-122
 *                             tf_custom_ops/tf_subsampling/tf_subsampling.cpp:8-17 (B = 1)
 *                             cpp_wrappers/cpp_subsampling/wrapper.cpp:58-286 (features / classes)
 *   d3f_voxel_down_sample     open3d.voxel_down_sample of the raw scans: datasets/ThreeDMatch.py:349 (0.03 m),
 *                             datasets/ETH.py:169 (0.0625 m), datasets/KITTI.py:314-315 (first_subsampling_dl),
 *                             demo_registration.py:24 (0.03 m)
 *   d3f_radius_neighbors_*    tf_custom_ops/tf_neighbors/tf_batch_neighbors.cpp:8-30,40-116
 *                             tf_custom_ops/tf_neighbors/tf_neighbors.cpp:8-18 (B = 1, pad = -1)
 *   d3f_kpconv_forward        kernels/convolution_ops.py:161-255 (KPConv_ops) + BN/LeakyReLU epilogue
 *                             models/network_blocks.py:149-165,185-186
 *   d3f_kpconv_deform_forward kernels/convolution_ops.py:379-499 (KPConv_deform_ops)
 *   d3f_unary_forward         kernels/convolution_ops.py:90-99 + models/network_blocks.py:207-219,
 *                             :343-368 (conv3 + shortcut add + LeakyReLU)
 *   d3f_kpconv_backward,      feature and weight gradients of KPConv_ops and unary_convolution (what tf.gradients
 *   d3f_unary_backward        gives the training scripts, training_3DMatch.py / utils/trainer.py)
 *   d3f_ind_max_pool          models/network_blocks.py:51-66
 *   d3f_closest_pool          models/network_blocks.py:69-83
 *   d3f_l2_normalize          models/D3Feat.py:65
 *   d3f_select_keypoints      utils/tester.py:209-213, 281-290 (host argsort of the detection scores)
 *   d3f_match_descriptors     geometric_registration/evaluate.py:11-27 (build_correspondence: mutual nearest
 *                             neighbours of two fragments' keypoint descriptors)
 *   d3f_register_pairs        geometric_registration/evaluate.py:84-99, utils/tester.py:305-316,
 *                             demo_registration.py:184-192 (Open3D's RANSAC over the keypoint correspondences,
 *                             with the edge-length and distance checkers)
 *   d3f_icp_pairs             datasets/KITTI.py:284-301 (Open3D's point-to-point registration_icp)
 *   d3f_pair_correspondences_* datasets/KITTI.py:35-48,319-327 (get_matching_indices), datasets/cal_overlap.py:78-126
 *                             (the BFMatcher overlap table of 3DMatch's training pairs)
 *   d3f_sample_correspondences datasets/KITTI.py:184-189, datasets/ThreeDMatch.py:218-229 (the keypoint draw)
 *   d3f_augment_pairs         datasets/ThreeDMatch.py:24-45,266-273, datasets/KITTI.py:191-206 (noise, rotate, scale,
 *                             shift; the backup points the loss measures on)
 *   d3f_evaluate_pairs        geometric_registration/evaluate.py:67-82,207, repeatability/evaluate_3dmatch_our.py:30-41,
 *                             evaluate_kitti_our.py:12-23, utils/tester.py:326-342, 3dmatch/evaluate.m with
 *                             mrEvaluateRegistration.m (FMR, repeatability, RTE / RRE, registration recall)
 *   d3f_momentum_clip_update  utils/trainer.py:116-156 (tf.clip_by_norm per gradient + tf.train.MomentumOptimizer)
 *   d3f_rank_mean             the data-parallel mean of gradients and batch statistics over ranks (no counterpart:
 *                             the reference trains on one GPU)
 */
#ifndef D3FEAT_B200_H_
#define D3FEAT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define D3F_OK 0
#define D3F_ERR_INVALID (-1)   /* bad argument (shape, enum, null pointer)            */
#define D3F_ERR_CAPACITY (-2)  /* caller-supplied output capacity / grid budget too small */
#define D3F_ERR_CUDA (-3)      /* CUDA runtime error (message in d3f_last_error)       */
#define D3F_ERR_WORKSPACE (-4) /* workspace smaller than *_workspace_bytes             */

/* KP_influence / aggregation_mode enums (kernels/convolution_ops.py:208-232) */
#define D3F_INFLUENCE_CONSTANT 0
#define D3F_INFLUENCE_LINEAR 1
#define D3F_INFLUENCE_GAUSSIAN 2
#define D3F_MODE_SUM 0
#define D3F_MODE_CLOSEST 1

typedef void* d3f_stream_t; /* cudaStream_t */

int d3f_version(void);
const char* d3f_last_error(void);
/* number of kernels this library has launched from the calling host thread (bench.py "gpu_launches") */
long long d3f_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * Bounding box of a stacked cloud: out_bbox[6] = {minx,miny,minz,maxx,maxy,maxz} (device floats).
 * Used to bound the hash grids of the two ops below without a host round trip per call.
 * ------------------------------------------------------------------------------------------- */
int d3f_bbox(const float* pts, int N, float* out_bbox, d3f_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Grid subsampling (voxel barycenters), stacked clouds.
 *   pts[N,3], batch_len[B] (device int32), dl: cell size.
 *   feats[N,fdim] / classes[N,ldim] optional (NULL, 0): the cpp_wrappers signature.
 *   Row i belongs to cloud b when start[b] <= i < start[b+1] (start = exclusive scan of batch_len). Rows at or
 *     past start[B] (lengths summing to less than N) belong to no cloud and are never read; lengths summing to more
 *     than N cut the last cloud at N.
 *   host_bbox: host float[6] bounding ALL points (from d3f_bbox or known a priori). It only bounds
 *     the sort-key width; the per-cloud origin is recomputed exactly on the device. A cloud merely displaced
 *     outside host_bbox is still subsampled exactly; a cloud whose own extent needs more cells than host_bbox
 *     allows overflows the sort key and is reported as out_M = -1.
 *   Outputs (capacity N rows each): out_pts[<=N,3], out_feats, out_classes, out_batch_len[B],
 *     out_M[1] (device int32: total number of cells). Cells are emitted per cloud in ascending
 *     reference cell key iX + NX*iY + NX*NY*iZ (grid_subsampling.cpp:53-56); barycenters are
 *     bit-identical to the reference (fp32 sums in input order, * (float)(1.0/count)).
 *   classes follow the reference literally: the LARGEST label present in the cell
 *     (std::max_element over map pairs, grid_subsampling.cpp:97-101).
 * ------------------------------------------------------------------------------------------- */
size_t d3f_grid_subsample_workspace_bytes(int N, int B);
int d3f_grid_subsample(const float* pts, const int* batch_len, int B, int N, float dl,
                       const float* feats, int fdim, const int* classes, int ldim,
                       const float* host_bbox, float* out_pts, float* out_feats, int* out_classes,
                       int* out_batch_len, int* out_M, void* workspace, size_t workspace_bytes,
                       d3f_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Voxel down-sampling of raw scans, stacked clouds: Open3D 0.7's voxel_down_sample (Geometry/DownSample.cpp), the
 * input stage of every reference entry point. Per cloud b, from its fp32 rows widened exactly to fp64, each step one
 * IEEE fp64 operation (true division, no fused multiply-add):
 *     min_b = per-axis minimum of the cloud's finite rows - voxel_size * 0.5
 *     i_a   = (int)floor((p_a - min_b,a) / voxel_size)                    (>= 0)
 *     voxel point = (sum of its rows in fp64, sequentially in input order) / (double)count, rounded to nearest fp32.
 *   voxel_size is a DOUBLE: voxel_down_sample(x, 0.03) uses the double 0.03; float(0.03) voxelises differently.
 *   Deviations from Open3D: voxels are emitted per cloud in ascending (iz, iy, ix), not in hash-map order; the output
 *   is fp32; a row with a non-finite coordinate is dropped (in no voxel, not in the bounds); a voxel_size that is not
 *   finite and > 0 is D3F_ERR_INVALID (Open3D returns an empty cloud).
 *   pts[N,3], lengths[B] (device int32), B in [1, 1024]; clouds as in d3f_grid_subsample (rows at or past start[B]
 *   belong to no cloud, lengths summing past the row count cut the last cloud). n_dev (device, optional): the raw row
 *   count, N then being the capacity of pts and of every launch.
 *   host_bbox: host float[6] bounding the clouds. It sizes the sort key: each axis gets the index width of the host
 *   extent / voxel_size plus a margin, at most 30 bits (so every index fits an int and Open3D's voxel_size * INT_MAX <
 *   extent guard cannot trigger), and cloud + three axes at most 62 bits; otherwise D3F_ERR_CAPACITY. A cloud merely
 *   displaced outside host_bbox is still voxelised exactly; one whose own extent needs wider indices overflows.
 *   Outputs: out_pts[out_capacity,3] (out_capacity < 0: N), out_lengths[B], out_M[1] (device int32).
 *   Exact form (d_status == NULL): *out_M = the number of voxels, -1 for a key overflow, -2 for more voxels than
 *   out_capacity; the caller reads it back (the output size is data dependent).
 *   Static form (d_status != NULL): nothing is read back. *out_M = min(voxels, out_capacity); no row at or past
 *   out_capacity is written; out_lengths count the written voxels; bit 0 of *d_status is OR-ed for a key overflow,
 *   bit 1 for more voxels than out_capacity. The launch sequence depends only on (B, N, out_capacity, host_bbox,
 *   voxel_size): it can be captured in a CUDA graph.
 *   Argument errors (D3F_ERR_INVALID / _CAPACITY / _WORKSPACE) are returned before any CUDA call.
 * ------------------------------------------------------------------------------------------- */
size_t d3f_voxel_down_sample_workspace_bytes(int N, int B);
int d3f_voxel_down_sample(const float* pts, const int* lengths, int B, int N, const int* n_dev, double voxel_size,
                          const float* host_bbox, float* out_pts, int* out_lengths, int* out_M, int out_capacity,
                          int* d_status, void* workspace, size_t workspace_bytes, d3f_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Radius neighbours, stacked clouds (hash grid over the supports, 27-cell scan per query).
 *   Result-set semantics of the reference (neighbors.cpp:211-332 / nanoflann.hpp:249-253,432-440):
 *   supports of the same cloud with d2 < radius*radius, d2 = ((dx*dx)+dy*dy)+dz*dz in fp32 without
 *   FMA contraction, rows sorted by ascending (d2, index), global support indices, rows padded with
 *   pad_value (Ns for the batch op, -1 for the non-batch op).
 *   Clouds as in d3f_grid_subsample: supports at or past the end of the last support cloud are in no cloud and
 *   never returned; a query at or past the end of the last query cloud gets count 0 and a row of padding; lengths
 *   summing past the row count cut the last cloud there. host_bbox sizes the grid; points outside it are clamped
 *   into its edge cells, which only adds candidates, so results stay exact. A host_bbox with more than 4096
 *   cells of radius * 1.001 on one axis is refused (D3F_ERR_INVALID; workspace_bytes returns 0): past that length
 *   fp32 cell indices can put two points within the radius two cells apart (nbgrid.cuh).
 *
 *   Two-phase use for the exact reference shape [Nq, max count]:
 *     d3f_radius_neighbors_build  -> grid over the supports in `workspace`
 *     d3f_radius_neighbors_count  -> counts[Nq] and out_max[1] (device); caller reads out_max
 *     d3f_radius_neighbors_fill   -> out_idx[Nq, cols]; rows longer than cols keep the nearest cols
 *   Single-phase use with a known column cap (the pyramid's neighborhood_limits,
 *   datasets/common.py:399-406): build + fill with cols = cap (count optional).
 * ------------------------------------------------------------------------------------------- */
size_t d3f_radius_neighbors_workspace_bytes(int Ns, int B, float radius, const float* host_bbox);
int d3f_radius_neighbors_build(const float* supports, const int* s_batch_len, int B, int Ns,
                               float radius, const float* host_bbox, void* workspace,
                               size_t workspace_bytes, d3f_stream_t stream);
int d3f_radius_neighbors_count(const float* queries, const int* q_batch_len, int Nq,
                               const float* supports, const int* s_batch_len, int B, int Ns,
                               float radius, const float* host_bbox, const void* workspace,
                               int* counts, int* out_max, d3f_stream_t stream);
/* out_order[Ns]: the support indices in hash-grid cell order (a spatially coherent visiting order). Passing it
 * as `query_order` to d3f_kpconv_forward when queries == supports makes neighbouring queries share their
 * gathered rows in L1/L2; results are unchanged (each query still writes its own output row). */
int d3f_radius_neighbors_order(const void* workspace, int Ns, int B, float radius,
                               const float* host_bbox, int* out_order, d3f_stream_t stream);
int d3f_radius_neighbors_fill(const float* queries, const int* q_batch_len, int Nq,
                              const float* supports, const int* s_batch_len, int B, int Ns,
                              float radius, const float* host_bbox, const void* workspace, int cols,
                              int pad_value, int* out_idx, d3f_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * The whole input pyramid of the encoder in ONE call: the loop of Dataset.tf_descriptor_input
 * (datasets/common.py:1325-1397) with the neighbourhood caps of big_neighborhood_filter (:399-406).
 * Level l: neighbors[l] = search(points_l, points_l, conv_radius[l]) (skipped if conv_radius <= 0);
 * if sub_dl[l] > 0: points_{l+1} = grid_subsample(points_l, sub_dl[l]); pools[l] = search(points_{l+1}, points_l,
 * pool_radius[l]); upsamples[l] = search(points_l, points_{l+1}, up_radius[l]). Every index matrix has exactly
 * limit[l] columns (nearest first, padded with the number of supports). Output buffers are caller-allocated with
 * `capacity[l]` rows per level. Level-0 rows at or past the end of the last cloud (N0 > sum of lengths) belong to
 * no cloud: they are not subsampled, no search returns them, and their neighbour and upsample rows are all padding.
 *   Exact form (out_level_sizes != NULL, a HOST int[n_levels]): receives the actual row counts; the call synchronises
 *   the stream once per subsampled level (the next level's launch sizes depend on the cell count) -- what the TF ops
 *   do (their output shapes are data dependent, tf_batch_subsampling.cpp:99-104).
 *   Static form (out_level_sizes == NULL): no device->host read at all. Launches are sized by capacity[l], every
 *   kernel reads its row count from d_counts[l] (DEVICE int[n_levels], written by this call), conditions that the exact
 *   form reports as errors are OR-ed into *d_status (DEVICE int: bit 0 = a cloud whose extent needs more subsampling
 *   cells than host_bbox allows, so its sort key overflows; bit 1 = a level has more cells than capacity[l+1]). A
 *   cloud that is only displaced outside host_bbox sets no bit: its cells are keyed from its own origin and the
 *   neighbour grids clamp it into their edge cells, so its pyramid is still exact. The launch sequence depends only on (B, capacity, spec, host_bbox), so a
 *   caller may capture it in a CUDA graph and replay it for every batch of the same bucket. d_counts[0] = N0, or
 *   *n0_dev when n0_dev != NULL (the level-0 count kept on the device; N0 is then the capacity of `points`).
 *   d_counts / d_status may be NULL in the exact form.
 * ------------------------------------------------------------------------------------------- */
#define D3F_MAX_LEVELS 8
typedef struct {
  int n_levels;
  float conv_radius[D3F_MAX_LEVELS];
  float sub_dl[D3F_MAX_LEVELS];
  float pool_radius[D3F_MAX_LEVELS];
  float up_radius[D3F_MAX_LEVELS];
  int limit[D3F_MAX_LEVELS];
} d3f_pyramid_spec;
size_t d3f_pyramid_workspace_bytes(int B, const d3f_pyramid_spec* spec, const int* capacity,
                                   const float* host_bbox);
int d3f_pyramid_build(const float* points, const int* lengths, int B, int N0,
                      const d3f_pyramid_spec* spec, const float* host_bbox, float* const* out_points,
                      int* const* out_lengths, int* const* out_neighbors, int* const* out_pools,
                      int* const* out_upsamples, const int* capacity, int* out_level_sizes,
                      void* workspace, size_t workspace_bytes, d3f_stream_t stream, int* d_counts,
                      int* d_status, const int* n0_dev);

/* ---------------------------------------------------------------------------------------------
 * Device-side row counts. Every row-wise entry point below takes trailing `const int* ..._dev` arguments (all may
 * be NULL). When given, the integer row count (Nq / Ns / N / N1 / N2) is the CAPACITY of the buffers and of the launch,
 * and the kernels read the actual count from device memory (e.g. &d_counts[l] of d3f_pyramid_build) -- rows beyond
 * it are neither read nor written, and the shadow index is the actual count. This is what lets a whole step be
 * enqueued (or graph-replayed) without the host ever knowing the level sizes.
 * ------------------------------------------------------------------------------------------- */

/* ---------------------------------------------------------------------------------------------
 * Static weights for the tensor-core path. A weight matrix W[K,N] (row-major; for KPConv the [K*Cin, Cout]
 * view of K_values[K,Cin,Cout]) is packed ONCE into the K-major TF32 hi/lo images the wgmma kernels
 * consume (3xTF32 split: fp32-level accuracy on the 5th-gen tensor cores). Every forward entry point takes
 * the packed image as an optional `W_packed` argument: NULL selects the CUDA-core fp32 path (same results
 * within rounding), non-NULL the wgmma path.
 * ------------------------------------------------------------------------------------------- */
size_t d3f_packed_weight_floats(int K, int N);
int d3f_pack_weight(const float* W, int K, int N, float* packed, d3f_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Rigid KPConv forward (KPConv_ops, convolution_ops.py:161-255), fused with the block epilogue.
 *   q[Nq,3], s[Ns,3], idx[Nq,H] (shadow index = Ns), feat[Ns,Cin], Kp[K,3], W[K,Cin,Cout].
 *   out[Nq,Cout] = epilogue( (sum_k (sum_h w[n,h,k] feat[idx[n,h]]) W_k) / nn[n] )
 *   nn = max(#neighbours whose feature-row sum > 0, 1)   (normalize != 0; :249-253)
 *   epilogue: y = x*bn_scale[c] + bn_shift[c] (if bn_scale != NULL; inference batch norm folded by
 *   the caller: scale = gamma/sqrt(var+1e-6), shift = beta - mean*scale), then + bias[c] (if
 *   bias != NULL), then LeakyReLU(leaky_alpha) if leaky_alpha >= 0 (pass -1 for none).
 *   shadow_xyz: coordinate of the shadow support (1e6 rigid :190, 1000 deformable :414).
 *   K = num_kernel_points (utils/config.py): any value in [1, 64]; K = 15 (the D3Feat configuration) runs the
 *   specialised tensor-core kernels, other values a generic CUDA-core stage 1.
 * ------------------------------------------------------------------------------------------- */
size_t d3f_kpconv_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout);
int d3f_kpconv_forward(const float* q, const float* s, const int* idx, const float* feat,
                       const float* Kp, const float* W, const float* W_packed, const int* query_order,
                       int Nq, int Ns, int H, int K, int Cin,
                       int Cout, float extent, int influence, int mode, int normalize,
                       const float* bn_scale, const float* bn_shift, const float* bias,
                       float leaky_alpha, float* out, void* workspace, size_t workspace_bytes,
                       d3f_stream_t stream, const int* nq_dev, const int* ns_dev);

/* Deformable KPConv second stage (KPConv_deform_ops, :379-499): per-query kernel points
 * Kp + offsets[n,K,3]; influence distance /extent (no factor 2); neighbours in range of no kernel
 * point are dropped (:435-451); optional modulations[n,K]; no neighbour-count normalisation. */
int d3f_kpconv_deform_forward(const float* q, const float* s, const int* idx, const float* feat,
                              const float* Kp, const float* offsets, const float* modulations,
                              const float* W, const float* W_packed, const int* query_order, int Nq,
                              int Ns, int H, int K, int Cin, int Cout,
                              float extent, int influence, int mode, const float* bn_scale,
                              const float* bn_shift, const float* bias, float leaky_alpha,
                              float* out, void* workspace, size_t workspace_bytes,
                              d3f_stream_t stream, const int* nq_dev, const int* ns_dev);

/* ---------------------------------------------------------------------------------------------
 * Unary convolution (features @ W) with fused epilogue:
 *   y = x@W; y = y*bn_scale + bn_shift (opt); y += bias (opt); y += residual[N,Cout] (opt);
 *   y = LeakyReLU(y) if leaky_alpha >= 0.
 * ------------------------------------------------------------------------------------------- */
int d3f_unary_forward(const float* x, const float* W, const float* W_packed, int N, int Cin, int Cout,
                      const float* bn_scale, const float* bn_shift, const float* bias,
                      const float* residual, float leaky_alpha, float* out, d3f_stream_t stream,
                      const int* n_dev);

/* ---------------------------------------------------------------------------------------------
 * Gradients of rigid KPConv (d3f_kpconv_forward without epilogue or bias) and of the unary convolution.
 *   G[q,o] = dout[q,o] / nn[q] (nn as the forward counts it; normalize = 0: 1), held constant
 *   dW[k,c,o] = sum_q wf[q,k,c] G[q,o]          wf[q,k,c] = sum_h w(q,h,k) feat[idx[q,h],c]
 *   dfeat[s,c] = sum_{(q,h): idx[q,h]=s} sum_k w(q,h,k) sum_o G[q,o] W[k,c,o]
 * Points, kernel points and indices get no gradient. Shadow entries, rows at or past nq_dev and indices at or past
 * ns_dev contribute nothing; dfeat rows no query reaches and rows at or past ns_dev are zero; dout rows at or past
 * nq_dev are never read. dfeat or dW may be NULL (not computed). Bitwise deterministic (no float atomics).
 * The feature gradient is a forward KPConv over the transposed neighbourhood, whose width Hr (the largest number of
 * (q, h) entries naming one support) depends on the data:
 *   d3f_kpconv_reverse_width  computes Hr and copies it to the host int *width: it SYNCHRONISES the stream. Its
 *                             workspace is d3f_kpconv_backward_workspace_bytes(Nq, Ns, H, K, Cin, Cout, 0) or more.
 *   d3f_kpconv_backward       takes that Hr (a smaller value drops reverse entries) and a workspace of
 *                             d3f_kpconv_backward_workspace_bytes(..., Hr). Does not synchronise.
 * tensor_cores != 0: the transposed contraction runs on the 3xTF32 wgmma GEMM (as a non-NULL W_packed selects in the
 * forward), 0: the CUDA-core fp32 GEMM. The weight gradient is fp32 FFMA, fresh accumulators every 64 rows, partials
 * of 2048 rows summed in float64 in a fixed order.
 * Unary: dx = dout @ W^T (rows at or past n_dev stay zero), dW = x^T @ dout over the rows below n_dev.
 * ------------------------------------------------------------------------------------------- */
size_t d3f_kpconv_backward_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout, int Hr);
int d3f_kpconv_reverse_width(const int* idx, int Nq, int Ns, int H, int* width, void* workspace,
                             size_t workspace_bytes, d3f_stream_t stream, const int* nq_dev, const int* ns_dev);
int d3f_kpconv_backward(const float* q, const float* s, const int* idx, const float* feat, const float* Kp,
                        const float* W, const float* dout, int Nq, int Ns, int H, int Hr, int K, int Cin, int Cout,
                        float extent, int influence, int mode, int normalize, int tensor_cores, float* dfeat,
                        float* dW, void* workspace, size_t workspace_bytes, d3f_stream_t stream, const int* nq_dev,
                        const int* ns_dev);
size_t d3f_unary_backward_workspace_bytes(int N, int Cin, int Cout);
int d3f_unary_backward(const float* x, const float* W, const float* dout, int N, int Cin, int Cout, int tensor_cores,
                       float* dx, float* dW, void* workspace, size_t workspace_bytes, d3f_stream_t stream,
                       const int* n_dev);

/* out[N2,C] = max_h x'[inds[n,h]] with x' = x || colmin(x) (shadow index = N1).
 * workspace: C floats. */
size_t d3f_ind_max_pool_workspace_bytes(int C);
int d3f_ind_max_pool(const float* x, const int* inds, int N1, int N2, int H, int C, float* out,
                     void* workspace, size_t workspace_bytes, d3f_stream_t stream, const int* n1_dev,
                     const int* n2_dev);

/* out[N2,C] = x'[inds[n,0]] with x' = x || zeros. `ld_inds` = row stride of inds (H). */
int d3f_closest_pool(const float* x, const int* inds, int N1, int N2, int ld_inds, int C,
                     float* out, d3f_stream_t stream, const int* n1_dev, const int* n2_dev);

/* out[n,:] = x[n,:] * rsqrt(max(sum x^2, eps)) (tf.nn.l2_normalize, models/D3Feat.py:65) */
int d3f_l2_normalize(const float* x, int N, int C, float eps, float* out, d3f_stream_t stream,
                     const int* n_dev);

/* Two unary convolutions that are summed -- the tail of every resnetb block (network_blocks.py:343-368: conv3 + BN,
 * shortcut unary + BN, add, LeakyReLU) -- as ONE tensor-core GEMM over the concatenated K:
 *   out = leaky([x1 | x2] @ W + shift),  W_packed = d3f_pack_weight of the [Cin1 + Cin2, Cout] matrix whose rows
 * are the two weight matrices with their batch-norm scales folded in, shift = the sum of the two BN shifts.
 * Neither the shortcut tensor nor the [x1 | x2] concatenation is ever materialised. Cin1 % 32 == 0, Cin2 % 4 == 0. */
int d3f_unary_pair_forward(const float* x1, int Cin1, const float* x2, int Cin2, const float* W_packed, int N,
                           int Cout, const float* shift, float leaky_alpha, float* out, d3f_stream_t stream,
                           const int* n_dev);

/* Detection score of D3Feat (models/D3Feat.py:67-115) for B stacked clouds: feats[N,D] are the decoder outputs BEFORE
 * l2 normalisation, neighbors[N,H] the level-0 conv neighbours (shadow index = N), lengths[B] the stack lengths.
 * out_scores[N]. The reference hard-codes B = 2 (anchor || positive); the result is identical for B = 2.
 * A cloud reaching past the row count n (lengths summing to more than n) is cut there. Rows past the last cloud
 * (lengths summing to less than n) belong to no cloud: they enter no cloud's maximum, so they change no real row's
 * score, and their own score is unspecified. */
size_t d3f_detection_scores_workspace_bytes(int N, int B);
int d3f_detection_scores(const float* feats, const int* neighbors, const int* lengths, int B, int N,
                         int H, int D, float* out_scores, void* workspace, size_t workspace_bytes,
                         d3f_stream_t stream, const int* n_dev);

/* Stand-alone block epilogue for callers that do not use the fused forms
 * (models/network_blocks.py:149-165 batch_norm inference form, :185-186 leaky_relu, :368 residual add):
 * y = x*scale[c] + shift[c] (if scale) ; y += residual (if) ; LeakyReLU(leaky_alpha) if >= 0. */
int d3f_affine_leaky(const float* x, int N, int C, const float* scale, const float* shift,
                     const float* residual, float leaky_alpha, float* out, d3f_stream_t stream,
                     const int* n_dev);

/* ---------------------------------------------------------------------------------------------
 * Training (models/network_blocks.py and models/D3Feat.py with training = True, what tf.gradients gives
 * utils/trainer.py). Exact shapes only: no device row counts. No float atomics: cross-row sums are float64 partials of
 * fixed 2048-row blocks added in block order, a row scattered to by several outputs sums its own list (the reverse
 * table of the indices) in ascending (q, h). Results are bitwise identical run to run and across streams. None of
 * these synchronises.
 *
 * Batch norm in training mode, tf.layers.batch_normalization(training=True) on x[N,C] (unfused):
 *   mean = sum x / N, var = sum (x - mean)^2 / N, invstd = 1/sqrt(var + eps),
 *   out = leaky(x * gamma*invstd + (beta - mean*gamma*invstd) + residual)   (residual optional, leaky_alpha < 0: none)
 *   moving_mean -= (moving_mean - mean) * decay, moving_var -= (moving_var - var) * decay   (decay = 1 - momentum)
 * mean[C] and invstd[C] are written for the backward. gamma = NULL: use_batch_norm = False, out = leaky(x + beta +
 * residual) with no statistics (moving_*, mean, invstd unused). N = 0: nothing is written, the moving statistics stay
 * (TF would write NaN into them).
 * Backward (dout[N,C], the forward's out): dz = dout * LeakyReluGrad (out > 0), dbeta = sum dz, dgamma = sum dz*xhat,
 * dx = gamma*invstd*(dz - dbeta/N - xhat*dgamma/N) (gamma = NULL: dx = dz), dresidual = dz. Any output may be NULL;
 * N = 0 gives dgamma = dbeta = 0. Workspace of both: d3f_batch_norm_train_workspace_bytes(N, C). */
size_t d3f_batch_norm_train_workspace_bytes(int N, int C);
int d3f_batch_norm_train_forward(const float* x, int N, int C, const float* gamma, const float* beta,
                                 float* moving_mean, float* moving_var, float decay, float eps, const float* residual,
                                 float leaky_alpha, float* out, float* mean, float* invstd, void* workspace,
                                 size_t workspace_bytes, d3f_stream_t stream);
int d3f_batch_norm_train_backward(const float* x, const float* out, const float* dout, int N, int C,
                                  const float* gamma, const float* mean, const float* invstd, float leaky_alpha,
                                  float* dx, float* dresidual, float* dgamma, float* dbeta, void* workspace,
                                  size_t workspace_bytes, d3f_stream_t stream);

/* Gradient of d3f_ind_max_pool (TF: reduce_max over h of gather(x || colmin(x), inds)), given its output out[N2,C]:
 * every entry equal to out[q,c] gets dout[q,c] / (number of such entries among the H of (q, c)); an entry whose index
 * is not in [0, N1) is the shadow row, valued colmin(x); the shadow's shares are summed and split evenly among the rows
 * of x equal to the column minimum (reduce_min's gradient). dx[N1,C]. */
size_t d3f_ind_max_pool_backward_workspace_bytes(int N1, int N2, int H, int C);
int d3f_ind_max_pool_backward(const float* x, const int* inds, const float* out, const float* dout, int N1, int N2,
                              int H, int C, float* dx, void* workspace, size_t workspace_bytes, d3f_stream_t stream);

/* Gradient of a row gather out[q] = x'[inds[q]], x' = x || zeros (d3f_closest_pool on its first index column, and
 * tf.gather): dx[s,c] = sum of dout[q,c] over the q with inds[q] == s, ascending q, rounded once. inds[N2] is one
 * contiguous column; entries outside [0, N1) are the shadow, whose gradient is dropped. */
size_t d3f_gather_rows_backward_workspace_bytes(int N1, int N2);
int d3f_gather_rows_backward(const int* inds, const float* dout, int N1, int N2, int C, float* dx, void* workspace,
                             size_t workspace_bytes, d3f_stream_t stream);

/* Gradient of d3f_l2_normalize, s = sum x^2 per row: s >= eps: dx = (dout - y (y.dout)) / sqrt(s), else
 * dx = dout / sqrt(eps). Needs no workspace. */
int d3f_l2_normalize_backward(const float* x, const float* dout, int N, int C, float eps, float* dx,
                              d3f_stream_t stream);

/* Gradient of d3f_detection_scores for dscores[N]: ties of the channel maxima and of each cloud's maximum split
 * evenly (reduce_max), the neighbour count is held constant (count_nonzero), softplus' = sigmoid. Rows of no cloud
 * pass no gradient; the gradient reaching the shadow row is dropped. dfeats[N,D]. */
size_t d3f_detection_scores_backward_workspace_bytes(int N, int H, int B, int D);
int d3f_detection_scores_backward(const float* feats, const int* neighbors, const int* lengths, const float* dscores,
                                  int B, int N, int H, int D, float* dfeats, void* workspace, size_t workspace_bytes,
                                  d3f_stream_t stream);

/* Keypoint selection by detection score for B stacked clouds (utils/tester.py:209-213, the 3DMatch tester: every
 * point in ascending score order; :281-290, the KITTI tester: the top k per cloud, ascending).
 *   scores[N] (N = capacity with n_dev), lengths[B] (device), optional points[N,3] and descriptors[N,D].
 *   Order contract: within each cloud, ascending score with ties by ascending row -- np.argsort(kind="stable") --
 *   where every NaN (either sign) ranks above +inf and -0.0 equals +0.0.
 *   Outputs (each optional, at least one required):
 *     out_order[N]       every row: clouds in stack order, ascending score within each (rows >= n untouched)
 *     out_index[B,k]     global rows of cloud b's top min(k, len_b), ascending score (= argsort(s_b)[-k:] + start_b)
 *     out_count[B]       min(k, len_b)
 *     out_points[B,k,3], out_descriptors[B,k,D], out_scores[B,k]   the selected rows
 *   Slots j >= count_b hold index -1 and zero rows. A cloud reaching past n (lengths summing to more than n) is cut at
 *   n: no row >= n is read. Rows past the last cloud (lengths summing to less than n) belong to no cloud and come
 *   last in out_order. k >= 1 when a per-cloud output is requested; D >= 1 with descriptors. Graph-capturable. */
size_t d3f_select_keypoints_workspace_bytes(int N, int B);
int d3f_select_keypoints(const float* scores, const int* lengths, int B, int N, int k, const float* points,
                         const float* descriptors, int D, int* out_order, int* out_index, int* out_count,
                         float* out_points, float* out_descriptors, float* out_scores, void* workspace,
                         size_t workspace_bytes, d3f_stream_t stream, const int* n_dev);

/* Descriptor matching between the keypoint sets of P cloud pairs (geometric_registration/evaluate.py:11-27).
 *   desc[B,k,D], count[B] (device) in the d3f_select_keypoints layout: slot j of cloud b is real iff
 *   j < clamp(count[b], 0, k). pairs[P,2] (device) = (src cloud, tgt cloud).
 *   For pair p with a = desc[src, :n_s], b = desc[tgt, :n_t]:
 *     s_ij = 0.0f, then for c = 0 .. D-1 in ascending order s_ij = fadd_rn(s_ij, fmul_rn(a_ic, b_jc)) -- fp32, no FMA.
 *     nn_st[p,i] = argmax_j s_ij, sim_st[p,i] = s[i, nn_st[p,i]]; nn_ts[p,j] = argmax_i s_ij, sim_ts likewise.
 *     argmax has numpy's semantics: NaN above everything, -0.0 equal to +0.0, ties to the smallest slot. A NaN
 *     similarity is reported as the positive quiet NaN 0x7fc00000.
 *     matches[p,m,:] = (i, nn_st[p,i]) for every real i with nn_ts[p, nn_st[p,i]] == i, in ascending i;
 *     n_matches[p] = their number. Unused match rows hold -1.
 *   Slots i >= n_s get nn = -1 and sim = 0, and so does every slot when the other cloud is empty. Slots at or past
 *   the count are never read; neither is a cloud outside [0, B), and a pair naming one matches nothing.
 *   On unit descriptors argmax s is the reference's argmin sqrt(2 - 2s), except where the rounding of 2 - 2s merges
 *   distinct similarities.
 *   Returns D3F_ERR_INVALID for B outside [1, 1024], k < 1, D < 1, P < 1, P*k beyond int32 or a null pointer (every
 *   output is required), D3F_ERR_WORKSPACE for a short workspace. Graph-capturable. */
size_t d3f_match_descriptors_workspace_bytes(int k, int P);
int d3f_match_descriptors(const float* desc, const int* count, int B, int k, int D, const int* pairs, int P,
                          int* nn_st, float* sim_st, int* nn_ts, float* sim_ts, int* matches, int* n_matches,
                          void* workspace, size_t workspace_bytes, d3f_stream_t stream);

/* Rigid registration of P cloud pairs by deterministic RANSAC over keypoint correspondences
 * (geometric_registration/evaluate.py:84-99, utils/tester.py:305-316, demo_registration.py:184-192, which call
 * Open3D's registration_ransac_based_on_* with CorrespondenceCheckerBasedOnEdgeLength / OnDistance).
 *   points[B,k,3] fp32, count[B] (device) in the d3f_select_keypoints layout: slot j of cloud b is real iff
 *   j < clamp(count[b], 0, k). pairs[P,2] (device) = (src cloud, tgt cloud). corr[P,L,2] (device) = (source slot,
 *   target slot) rows, of which the first n_c = clamp(n_corr[p], 0, L) are real.
 *   Contract (exact; oracle/register_np.py restates it in numpy): every step is one correctly rounded fp64 operation
 *   in a fixed order (no fused multiply-add), sums sequential in ascending index, points widened from fp32 exactly.
 *     hypothesis h in [0, max_iterations) samples idx_m, m < ransac_n: c = ((p << 32) | h) * 8 + m,
 *       z = splitmix64(seed + c * 0x9E3779B97F4A7C15), idx_m = ((z >> 32) * n_c) >> 32 (uint64, wrapping);
 *       a repeated index rejects it; the edge checker rejects it if |s_a - s_b| < edge_ratio * |t_a - t_b| or the
 *       reverse for any a < b; the pose is Horn's quaternion method (centroids, centred cross-covariance, cyclic
 *       Jacobi on the 4x4 matrix, 6 sweeps, exact-zero pivots skipped); every sample row must then have
 *       |R s + t - t'|^2 <= distance^2. Only the first max_validation validated hypotheses in ascending h are scored.
 *     A row is an inlier if |R s + t - t'|^2 < distance^2. The best hypothesis has the most inliers, then the smaller
 *     sequential sum of inlier d^2, then the smaller h; the pose is refit over its inliers in ascending row order
 *     (kept as it is if it has none).
 *   Outputs: pose[P,4,4] fp64 (t' ~ R s + t, row-major, last row 0 0 0 1), n_inliers[P], hypothesis[P] (the best h)
 *   and n_validated[P] (the number scored). A pair naming a cloud outside [0, B), or with a real row naming a slot at
 *   or past its cloud's count, registers nothing and reads neither; so does a pair with n_c < ransac_n or without a
 *   validated hypothesis: identity, 0, -1 and its validated count.
 *   Limits: B in [1, 1024]; k, L, P >= 1; ransac_n in [3, 8]; max_iterations in [1, 2^24]; max_validation in
 *   [1, max_iterations]; distance finite and > 0; edge_ratio in (0, 1]; B*k*3, P*L*2 and P*max_iterations within
 *   int32. Otherwise, or for a null pointer, D3F_ERR_INVALID before any CUDA call; D3F_ERR_WORKSPACE for a short
 *   workspace. Graph-capturable: counts, n_corr and pair ids are read on the device. */
size_t d3f_register_pairs_workspace_bytes(int L, int P, int max_iterations, int max_validation);
int d3f_register_pairs(const float* points, const int* count, int B, int k, const int* corr, const int* n_corr, int L,
                       const int* pairs, int P, int ransac_n, int max_iterations, int max_validation, double distance,
                       double edge_ratio, unsigned long long seed, double* pose, int* n_inliers, int* hypothesis,
                       int* n_validated, void* workspace, size_t workspace_bytes, d3f_stream_t stream);

/* Point-to-point ICP refinement of P cloud pairs over stacked clouds (datasets/KITTI.py:284-301, which calls
 * Open3D's registration_icp with TransformationEstimationPointToPoint and ICPConvergenceCriteria).
 *   points[N,3] fp32 and lengths[B] (device, >= 0) stacked as in d3f_radius_neighbors_build: cloud b holds the rows
 *   [start[b], start[b+1]) of the lengths' exclusive scan, cut at the row count; rows at or past start[B] belong to no
 *   cloud. n_dev (device, optional): the row count, N then being the capacity. host_bbox (host, 6 floats) sizes the
 *   target grid as in the neighbour search; points outside it stay exact. pairs[P,2] (device) = (source cloud,
 *   target cloud); init[P,4,4] (device, fp64, row-major) maps source points onto the target, t' ~ R s + t.
 *   Contract (exact; oracle/icp_np.py restates it in numpy): every step is one correctly rounded fp64 operation in a
 *   fixed order (no fused multiply-add), points widened from fp32 exactly. Evaluation i of pair p, pose T_i (T_0 =
 *   init): every source row s becomes q = R s + t; its correspondence is the target row j with the smallest
 *   d^2 = |q - t_j|^2 < distance^2 (strict; ties to the smaller row; NaN never corresponds). Over the n corresponding
 *   rows, in blocks of 256 consecutive source rows summed sequentially and then the block sums sequentially: the
 *   centroids, the centred cross-covariance and sum d^2. fitness = n / n_src, inlier_rmse = sqrt(sum d^2 / n) (0 for
 *   n = 0). The pair stops after evaluation i > 0 when |fitness_i - fitness_{i-1}| < relative_fitness and
 *   |rmse_i - rmse_{i-1}| < relative_rmse, when n < 3 (the pose is kept) or when i = max_iterations; otherwise
 *   T_{i+1} = U T_i with U Horn's quaternion pose of (q, t_j) (6 cyclic Jacobi sweeps, as d3f_register_pairs).
 *   Outputs, all for the final pose: pose[P,4,4] fp64 (rows 0-2 from T, row 3 copied from init), fitness[P],
 *   inlier_rmse[P] (fp64), n_corr[P] and iterations[P] (the number of updates). A pair naming a cloud outside [0, B),
 *   or with an empty source or target, keeps init with 0 correspondences and 0 iterations, and neither cloud is read.
 *   Limits: B in [1, 1024]; N >= 0; P >= 1; max_iterations in [0, 1024]; distance finite and > 0; relative_fitness
 *   and relative_rmse finite and >= 0; P * ceil(N / 256) * 256 within int32; the target grid (cell edge
 *   distance * 1.001) within 2^27 cells over all clouds, and every host_bbox coordinate within 1024 cells of the origin
 *   (the fp32 cell lookup of an fp64 query is then provably conservative). Otherwise, or for a null pointer (n_dev
 *   excepted), D3F_ERR_INVALID before any CUDA call; D3F_ERR_WORKSPACE for a short workspace; the workspace query
 *   returns 0 for arguments outside these limits. Graph-capturable: counts, pair ids and the stopping rule are
 *   evaluated on the device; a call is 3 * max_iterations + 10 graph nodes (4 for N = 0). */
size_t d3f_icp_pairs_workspace_bytes(int N, int B, int P, double distance, const float* host_bbox);
int d3f_icp_pairs(const float* points, const int* lengths, int B, int N, const int* n_dev, const float* host_bbox,
                  const int* pairs, int P, const double* init, double distance, int max_iterations,
                  double relative_fitness, double relative_rmse, double* pose, double* fitness, double* inlier_rmse,
                  int* n_corr, int* iterations, void* workspace, size_t workspace_bytes, d3f_stream_t stream);

/* Ground-truth metrics of P matched and registered cloud pairs (geometric_registration/evaluate.py:67-82 and :207:
 * feature-match recall; repeatability/evaluate_3dmatch_our.py:30-41, evaluate_kitti_our.py:12-23: repeatability;
 * utils/tester.py:326-342: RTE / RRE / success; 3dmatch/evaluate.m with mrEvaluateRegistration.m: registration
 * recall).
 *   points[B,k,3] fp32 and count[B] (device) in the d3f_select_keypoints layout: cloud b's real slots are
 *   [0, clamp(count[b], 0, k)) in ascending score, so its top n are the last n of them; no other slot is read.
 *   matches[P,L,2] and n_matches[P] (device) as d3f_match_descriptors writes them. pairs[P,2] (device) = (source
 *   cloud, target cloud). truth_pose[P,4,4] (device, fp64) maps source points onto the target (t ~ R s + t, the
 *   convention of d3f_register_pairs; a 3DMatch gt.log holds the inverse). truth_info[P,6,6] (device, fp64, nullable):
 *   Choi's information matrices. truth_flags[P] (device): bit 0 = the pair has truth, bit 1 = it counts for
 *   registration recall. poses (host array of S device pointers, S in [0, 2]): [P,4,4] fp64 pose sets to score.
 *   levels (host, R in [0, 14]): repeatability levels, strictly ascending within [1, k].
 *   Contract (exact; oracle/evaluate_np.py restates it in numpy): every step is one correctly rounded fp64 operation
 *   in a fixed order (no fused multiply-add), keypoints widened from fp32, q = R s + t in d3f_register_pairs' order,
 *   every distance test d^2 < tau^2 (strict; the reference compares sqrt(d^2) < tau, which differs only at rounding
 *   ties). A pair is evaluated when flags bit 0 is set and both cloud ids lie in [0, B):
 *     n_match_inliers counts the rows m < clamp(n_matches, 0, L) whose real slots have d^2(G s_i, t_j) < fmr_distance^2;
 *     inlier_ratio = n_match_inliers / n_matches (0 without matches); fmr_hit = inlier_ratio > fmr_ratio.
 *     n_repeated[p,r] counts the target slots among the top levels[r] whose smallest d^2 over the top levels[r] source
 *     slots is < repeat_distance^2 with no NaN d^2 among them; repeatability = n_repeated / levels[r].
 *     Per pose set: rte = |t - t_G|; c = (tr(R^T R_G) - 1) / 2 clamped to [-1, 1]; rre_deg = acos(c) * 180 / pi
 *     (acos is not correctly rounded: within a few ulp of the oracle); success = rte < rte_max and
 *     c > cos(rre_max_deg). With flags bit 1 and truth_info: E = G inv(pose), er = [t_E; -q_v] (dcm2quat),
 *     rmse2 = er^T info er / info_00, recall_hit = rmse2 <= err2 (NaN is a miss). A non-finite entry in rows 0-2 of G
 *     or of the pose gives NaN rte, rre_deg and rmse2: a miss in every pose test.
 *   Outputs (device, every element written): valid, n_match_inliers, fmr_hit [P] int32, inlier_ratio [P] fp64;
 *   n_repeated [P,R] int32, repeatability [P,R] fp64; rte, rre_deg, rmse2 [S,P] fp64, success, recall_hit [S,P] int32
 *   (NaN where undefined); totals [4 + R + 7 S] fp64, summed over the evaluated pairs sequentially in pair order:
 *   pairs, FMR hits, sum inlier_ratio, sum n_match_inliers, sum repeatability per level, then per pose set:
 *   successes, sum rte over rte < rte_max and that count, sum rre_deg over c > cos(rre_max_deg) and that count,
 *   recall hits, recall pairs. A pair that is not evaluated reads nothing: valid 0, zeros, NaN rte / rre_deg / rmse2.
 *   Limits: B in [1, 1024]; k, L, P >= 1; P*k, P*L*2 and B*k*3 within int32; fmr_distance, repeat_distance, err2 and
 *   rte_max finite and > 0; fmr_ratio in [0, 1); rre_max_deg in (0, 180]. Otherwise, or for a null pointer
 *   (truth_info excepted; the repeatability outputs when R = 0 and the pose outputs when S = 0),
 *   D3F_ERR_INVALID before any CUDA call; D3F_ERR_WORKSPACE for a short workspace. Graph-capturable: counts, pair
 *   ids, flags and truth are read on the device; a call is 2 to 4 kernels. */
size_t d3f_evaluate_pairs_workspace_bytes(int P, int S);
int d3f_evaluate_pairs(const float* points, const int* count, int B, int k, const int* matches, const int* n_matches,
                       int L, const int* pairs, int P, const double* truth_pose, const double* truth_info,
                       const int* truth_flags, const double* const* poses, int S, const int* levels, int R,
                       double fmr_distance, double fmr_ratio, double repeat_distance, double err2, double rte_max,
                       double rre_max_deg, int* valid, int* n_match_inliers, double* inlier_ratio, int* fmr_hit,
                       int* n_repeated, double* repeatability, double* rte, double* rre_deg, double* rmse2,
                       int* success, int* recall_hit, double* totals, void* workspace, size_t workspace_bytes,
                       d3f_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Training pairs (datasets/KITTI.py and datasets/ThreeDMatch.py's generators, datasets/cal_overlap.py). Contract:
 * oracle/pairs_np.py, exactly. points[N,3] fp32 and lengths[B] (device, B in [1, 1024]) stacked as in d3f_icp_pairs;
 * pairs[P,2] (device) = (anchor cloud, positive cloud), P in [1, 2^24]; trans[P,4,4] (device, fp64, row-major) maps
 * anchor points onto the positive (GroundTruth.pose's convention). A pair naming a cloud outside [0, B) reads neither.
 *
 * Correspondences. Anchor row s becomes q = R s + t (fp64, one rounding per operation in d3f_icp_pairs' order, no
 * fused multiply-add); d^2 = ((e_0^2 + e_1^2) + e_2^2) against the widened positive rows, tau^2 = distance * distance.
 *   mode D3F_CORR_RADIUS: every positive row with d^2 < tau^2 (strict); D3F_CORR_NEAREST: the row with the smallest
 *   d^2 < tau^2, ties to the smaller row. A non-finite q matches nothing.
 *   d3f_pair_correspondences_count  builds the grid over the clouds in `workspace` and writes offset[P+1] (int64):
 *                                   pair p's rows are [offset[p], offset[p+1]); count[P] (int32, saturating) and
 *                                   overlap[P] = count / anchor rows (fp64, 0 for an empty anchor). The caller reads
 *                                   M = offset[P] back to size `rows`.
 *   d3f_pair_correspondences_fill   with the same arguments and workspace, after the count: rows[M,2] int32 =
 *                                   (anchor row, positive row), cloud-local, ascending in (anchor, positive) per pair.
 *   Limits: N >= 0; P * ceil(N / 256) * 256 within int32; distance finite and > 0; the grid (cell distance rounded
 *   up to fp32, * 1.001) within 2^27 cells over all clouds and 4096 per axis, and every host_bbox coordinate within 1024
 *   cells of the origin; otherwise, or for a null pointer, D3F_ERR_INVALID before any CUDA call (the workspace query
 *   returns 0).
 * Sampling, d3f_sample_correspondences: pair p's candidates are rows [offset[p], offset[p+1]) of rows[M,2] (offset
 *   nondecreasing from 0 to M, as the count writes it; any other table gives an unspecified but in-bounds sample),
 *   n = their number. valid[p] = n >= max(min_count, 1), and without replacement n >= k. replace = 1: draw m is
 *   ((z >> 32) * n) >> 32 of its counter; replace = 0: the k candidates with the smallest (32-bit key, candidate), in
 *   that order. anc[P,k] = the anchor row, pos[P,k] = the positive row + anchor_len[p] (device int32 [P]), -1 for an
 *   invalid pair. Never synchronises.
 * Augmentation, d3f_augment_pairs: for every pair and each of its two clouds (side 0: anchor, 1: positive), from the
 *   fp32 row widened to fp64, one rounding per operation: x += u * noise per axis; num_axis (1 or 3) rotations
 *   x_j = ((x_0 R_0j + x_1 R_1j) + x_2 R_2j) by the reference's float32 R (theta = (u * 2) * pi, R from fp64 cos / sin
 *   rounded to fp32, row and column `axis` those of the identity; axis = floor(3 u') for num_axis = 1, 0, 1, 2 for 3);
 *   with scale_shift: x = scale * x + shift, scale = scale_min + (scale_max - scale_min) u per pair and
 *   shift_a = -shift_range + (2 shift_range) u per cloud; then one rounding to fp32. Outputs: out_points and
 *   backup_points [capacity,3] (pair p's anchor then positive rows from row_offset[p]; backup = fp32 of q = trans s for
 *   the anchor, the point itself for the positive; rows at or past min(row_offset[P], capacity) are not written),
 *   out_lengths[P,2], row_offset[P+1] (int64), R[2P,num_axis,3,3] fp32, scale[P] and shift[2P,3] fp64 (1 and 0 without
 *   scale_shift). Never synchronises.
 * Counters: every draw is z = splitmix64(seed + c * 0x9E3779B97F4A7C15), c = (pair << 36) | (index << 4) | slot, and
 *   u = (z >> 11) * 2^-53. Slots: 0-5 noise (3 * side + axis; index = cloud-local row), 6-7 rotation angle (+ side;
 *   index = rotation), 8-9 rotation axis (+ side), 10 scale, 11-12 shift (+ side; index = axis), 13 draw with
 *   replacement (index = m), 14 key without replacement (index = candidate; key = z >> 32).
 * ------------------------------------------------------------------------------------------- */
#define D3F_CORR_RADIUS 0
#define D3F_CORR_NEAREST 1
size_t d3f_pair_correspondences_workspace_bytes(int N, int B, int P, double distance, const float* host_bbox);
int d3f_pair_correspondences_count(const float* points, const int* lengths, int B, int N, const float* host_bbox,
                                   const int* pairs, int P, const double* trans, double distance, int mode,
                                   long long* offset, int* count, double* overlap, void* workspace,
                                   size_t workspace_bytes, d3f_stream_t stream);
int d3f_pair_correspondences_fill(const float* points, int B, int N, const float* host_bbox, const int* pairs, int P,
                                  const double* trans, double distance, int mode, int M, int* rows, void* workspace,
                                  size_t workspace_bytes, d3f_stream_t stream);
size_t d3f_sample_correspondences_workspace_bytes(int M, int P);
int d3f_sample_correspondences(const long long* offset, const int* rows, int M, int P, const int* anchor_len, int k,
                               int replace, int min_count, unsigned long long seed, int* anc, int* pos, int* valid,
                               void* workspace, size_t workspace_bytes, d3f_stream_t stream);
size_t d3f_augment_pairs_workspace_bytes(int B, int P);
int d3f_augment_pairs(const float* points, const int* lengths, int B, int N, const int* pairs, int P,
                      const double* trans, unsigned long long seed, double noise, int num_axis, int scale_shift,
                      double scale_min, double scale_max, double shift_range, int capacity, float* out_points,
                      float* backup_points, int* out_lengths, long long* row_offset, float* R, double* scale,
                      double* shift, void* workspace, size_t workspace_bytes, d3f_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * The training update (utils/trainer.py:116-156): tf.clip_by_norm on each gradient on its own (TF 1.12
 * clip_ops.clip_by_norm), then tf.train.MomentumOptimizer (ApplyMomentum, use_nesterov = False). Contract:
 * oracle/optim_np.py, exactly. table[T] (device) names T tensors; per tensor, in fp32 with one rounding per operation
 * and no fused multiply-add:
 *   l2sum = sum of g^2 in fp64: each 2048-element block (from element 0) summed sequentially, the blocks added in
 *           block order. TF sums g*g in fp32 in an unspecified order: the one deviation.
 *   norm  = fl32(sqrt(l2sum)), 0 when l2sum = 0 (TF's where(l2sum > 0, ...)); M = (norm < c) ? c : norm
 *   gc    = fl32(fl32(g * c) / M)          (clip_norm = c <= 0: gc = g, trainer.py:150-153, and no norm is taken)
 *   accum = fl32(fl32(accum * momentum) + gc);   var = fl32(var - fl32(accum * lr))
 * Two kernels for all tensors together (one without clipping): block partials over the flat element space, then
 * per-tensor finalise and update. No float atomics, no host synchronisation: graph-capturable, bitwise identical run to
 * run and across streams. numel_total (host) must equal the sum of the table's numel: the workspace is sized from it
 * (d3f_momentum_clip_workspace_bytes(T, numel_total)); any other table gives an unspecified update but never writes
 * outside the workspace or the named tensors. A numel < 0 counts as 0. T in [0, 1024], numel_total >= 0; var, accum
 * and grad of one tensor must not overlap. Otherwise, or for a null pointer, D3F_ERR_INVALID before any CUDA call.
 *
 * d3f_rank_mean: the data-parallel reduction of a gathered x[R, P] (device, fp32, rank-major):
 *   out[p] = fl32((x[0,p] + x[1,p] + ... + x[R-1,p]) / R), summed in fp64 in rank order from x[0,p]
 * (R = 1: out = x bit for bit; for R > 1 a NaN comes out as the canonical NaN). out may be x's row 0. R >= 1,
 * P >= 0. One kernel (none for P = 0).
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  float* var;
  float* accum;
  const float* grad;
  long long numel;
} d3f_momentum_tensor;
size_t d3f_momentum_clip_workspace_bytes(int T, long long numel_total);
int d3f_momentum_clip_update(const d3f_momentum_tensor* table, int T, long long numel_total, float lr,
                             float momentum, float clip_norm, void* workspace, size_t workspace_bytes,
                             d3f_stream_t stream);
int d3f_rank_mean(const float* x, int R, long long P, float* out, d3f_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* D3FEAT_B200_H_ */

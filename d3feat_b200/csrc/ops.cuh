// Internal (C++) interface between the translation units of the library. The public C ABI is api.cu.
#pragma once
#include "common.cuh"

namespace d3f {

// ---- gemm.cu ----------------------------------------------------------------------------------------
struct Epilogue {
  const float* rowscale;  // [M] or null
  const float* bn_scale;  // [N] or null
  const float* bn_shift;  // [N] or null (used with bn_scale)
  const float* bias;      // [N] or null
  const float* residual;  // [M,N] or null
  float leaky_alpha;      // < 0: none
  const int* row_map;     // [M] or null: GEMM row m is written to output row row_map[m]
  const int* m_dev = nullptr;   // optional: actual row count in device memory (M is then the launch capacity)
  int m_off = 0;                // rows of *m_dev that precede this GEMM's row 0 (KPConv query chunks)
};
int gemm_f32(const float* A, const float* B, float* C, int M, int N, int K, const Epilogue& ep, cudaStream_t stream);

// ---- tc_gemm.cu (wgmma, 3xTF32) ---------------------------------------------------------------------
size_t tc_packed_floats(int K, int N);
int tc_padded_n(int N);
int tc_pack_weight(const float* W, int K, int N, float* packed, cudaStream_t stream);
bool tc_gemm_supported(const float* A, int K);
int tc_gemm(const float* A, const float* Bp, float* C, int M, int N, int K, const Epilogue& ep, cudaStream_t stream,
            float* split_ws = nullptr, const float* A2 = nullptr, int K1 = 0);
int tc_gemm_splits(int M, int N, int K);
size_t tc_gemm_split_ws_floats(int M, int N, int K);

// ---- grid.cu ----------------------------------------------------------------------------------------
int launch_batch_start(const int* len, int B, int* start, cudaStream_t stream);
int bbox_device(const float* pts, int N, float* out_bbox, cudaStream_t stream);
size_t grid_subsample_workspace_bytes(int N, int B);
int grid_subsample(const float* pts, const int* batch_len, int B, int N, float dl, const float* feats, int fdim,
                   const int* classes, int ldim, const float* host_bbox, float* out_pts, float* out_feats,
                   int* out_classes, int* out_batch_len, int* out_M, void* workspace, size_t workspace_bytes,
                   cudaStream_t stream, const int* n_dev = nullptr, int out_capacity = -1, int* status = nullptr,
                   const int* start_pre = nullptr);

// ---- voxel.cu ---------------------------------------------------------------------------------------
size_t voxel_down_sample_workspace_bytes(int N, int B);
int voxel_down_sample(const float* pts, const int* lengths, int B, int N, const int* n_dev, double voxel_size,
                      const float* host_bbox, float* out_pts, int* out_lengths, int* out_M, int out_capacity,
                      int* d_status, void* workspace, size_t workspace_bytes, cudaStream_t stream);

// ---- neighbors.cu -----------------------------------------------------------------------------------
size_t radius_neighbors_workspace_bytes(int Ns, int B, float radius, const float* host_bbox);
// ns_dev / nq_dev / pad_dev (optional): actual row counts / the shadow index in device memory; Ns / Nq are then capacities
int radius_neighbors_build(const float* supports, const int* s_batch_len, int B, int Ns, float radius,
                           const float* host_bbox, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                           const int* ns_dev = nullptr, const int* s_start_pre = nullptr);
int radius_neighbors_count(const float* queries, const int* q_batch_len, int Nq, int B, int Ns, float radius,
                           const float* host_bbox, const void* workspace, int* counts, int* out_max,
                           cudaStream_t stream);
int radius_neighbors_order(const void* workspace, int Ns, int B, float radius, const float* host_bbox, int* out_order,
                           cudaStream_t stream);
int radius_neighbors_fill(const float* queries, const int* q_batch_len, int Nq, int B, int Ns, float radius,
                          const float* host_bbox, const void* workspace, int cols, int pad_value, int* out_idx,
                          cudaStream_t stream, const int* nq_dev = nullptr, const int* pad_dev = nullptr,
                          const int* q_start_pre = nullptr);
struct NbView;   // nbgrid.cuh: the built grid, for nearest_in_cloud
int radius_neighbors_view(const void* workspace, int Ns, int B, float radius, const float* host_bbox, NbView* out);

// ---- pyramid.cu -------------------------------------------------------------------------------------
size_t pyramid_workspace_bytes(int B, const d3f_pyramid_spec* spec, const int* capacity, const float* host_bbox);
int pyramid_build(const float* points, const int* lengths, int B, int N0, const d3f_pyramid_spec* spec,
                  const float* host_bbox, float* const* out_points, int* const* out_lengths,
                  int* const* out_neighbors, int* const* out_pools, int* const* out_upsamples, const int* capacity,
                  int* out_level_sizes, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                  int* d_counts = nullptr, int* d_status = nullptr, const int* n0_dev = nullptr);

// ---- kpconv.cu --------------------------------------------------------------------------------------
size_t kpconv_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout);
int kpconv_forward_impl(bool deform, const float* q, const float* s, const int* idx, const float* feat,
                        const float* Kp, const float* offsets, const float* modulations, const float* W,
                        const float* W_packed, const int* query_order, int Nq,
                        int Ns, int H, int K, int Cin, int Cout, float extent, int influence, int mode, int normalize,
                        const float* bn_scale, const float* bn_shift, const float* bias, float leaky_alpha,
                        float* out, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                        const int* nq_dev = nullptr, const int* ns_dev = nullptr);

// building blocks the backward pass shares with the forward (kpconv.cu)
int kpconv_chunk_queries(int K, int Cin);
int kpconv_prep_supports(bool deform, const float* s, const float* feat, int Ns, const int* ns_dev, int K, int Cin,
                         int normalize, float4* s4, cudaStream_t stream);
int kpconv_stage1_wf(const float* q, const float4* s4, const int* idx, const float* feat, const float* Kp, int Nq, int Ns,
                     int H, int K, int Cin, float extent, int influence, int mode, int n0, int n1, float* wf,
                     cudaStream_t stream, const int* nq_dev = nullptr, const int* ns_dev = nullptr);

// ---- kpconv_grad.cu (feature and weight gradients of rigid KPConv and of the unary convolution) ----------
size_t kpconv_backward_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout, int Hr);
int kpconv_reverse_width(const int* idx, int Nq, int Ns, int H, int* width, void* workspace, size_t workspace_bytes,
                         cudaStream_t stream, const int* nq_dev, const int* ns_dev);
int kpconv_backward(const float* q, const float* s, const int* idx, const float* feat, const float* Kp, const float* W,
                    const float* dout, int Nq, int Ns, int H, int Hr, int K, int Cin, int Cout, float extent,
                    int influence, int mode, int normalize, int tensor_cores, float* dfeat, float* dW, void* workspace,
                    size_t workspace_bytes, cudaStream_t stream, const int* nq_dev, const int* ns_dev);
size_t unary_backward_workspace_bytes(int N, int Cin, int Cout);
int unary_backward(const float* x, const float* W, const float* dout, int N, int Cin, int Cout, int tensor_cores,
                   float* dx, float* dW, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                   const int* n_dev);
// Reverse neighbour table of idx[Nq, H] as a CSR, with no read-back: *sorted_q lists the query of every entry in
// ascending (s, q, h); support s owns [offs[s], offs[s] + counts[s]). Entries that are not real (q at or past the row
// count, idx < 0 or at or past the support count) sort last, are not counted and fill [offs[Ns], Nq * H). Sort
// buffers for Nq * H pairs (keys[0] / vals[0] are the input), counts and offs of Ns + 1 ints, scan_scratch of
// scan_num_blocks(Ns + 1) + 1 ints.
struct SortBuffers;
int reverse_csr(const int* idx, int Nq, int Ns, int H, const int* nq_dev, const int* ns_dev, const SortBuffers& sb,
                int* counts, int* offs, int* scan_scratch, const uint32_t** sorted_q, cudaStream_t stream);

// ---- train_ops.cu (training-mode batch norm; backward of the pools, l2_normalize and detection_scores) -------
size_t batch_norm_train_workspace_bytes(int N, int C);
int batch_norm_train_forward(const float* x, int N, int C, const float* gamma, const float* beta, float* moving_mean,
                             float* moving_var, float decay, float eps, const float* residual, float alpha, float* out,
                             float* mean, float* invstd, void* workspace, size_t workspace_bytes, cudaStream_t stream);
int batch_norm_train_backward(const float* x, const float* out, const float* dout, int N, int C, const float* gamma,
                              const float* mean, const float* invstd, float alpha, float* dx, float* dresidual,
                              float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes,
                              cudaStream_t stream);
size_t ind_max_pool_backward_workspace_bytes(int N1, int N2, int H, int C);
int ind_max_pool_backward(const float* x, const int* inds, const float* out, const float* dout, int N1, int N2, int H,
                          int C, float* dx, void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t gather_rows_backward_workspace_bytes(int N1, int N2);
int gather_rows_backward(const int* inds, const float* dout, int N1, int N2, int C, float* dx, void* workspace,
                         size_t workspace_bytes, cudaStream_t stream);
int l2_normalize_backward(const float* x, const float* dout, int N, int C, float eps, float* dx, cudaStream_t stream);
size_t detection_scores_backward_workspace_bytes(int N, int H, int B, int D);
int detection_scores_backward(const float* feats, const int* neighbors, const int* lengths, const float* dscores, int B,
                              int N, int H, int D, float* dfeats, void* workspace, size_t workspace_bytes,
                              cudaStream_t stream);

// ---- kpconv_fused.cu (one persistent kernel per layer: gather + correlation + wgmma contraction) -------
bool kpconv_fused_supported(int Nq, int H, int K, int Cin, int Cout, int influence, int mode, const float* feat,
                            const float* W, const float* out, const int* query_order);
size_t kpconv_fused_workspace_bytes();
int kpconv_fused_forward(const float* q, const float4* s4, const int* idx, const float* feat, const float* Kp,
                         const float* W, float* w_img, int Nq, int Ns, int H, int Cout, float extent, int normalize,
                         const float* bn_scale, const float* bn_shift, const float* bias, float leaky_alpha, float* out,
                         cudaStream_t stream, const int* nq_dev = nullptr, const int* ns_dev = nullptr);

// ---- pool.cu ----------------------------------------------------------------------------------------
int ind_max_pool(const float* x, const int* inds, int N1, int N2, int H, int C, float* out, void* workspace,
                 size_t workspace_bytes, cudaStream_t stream, const int* n1_dev = nullptr, const int* n2_dev = nullptr);
int closest_pool(const float* x, const int* inds, int N1, int N2, int ld_inds, int C, float* out,
                 cudaStream_t stream, const int* n1_dev = nullptr, const int* n2_dev = nullptr);
int l2_normalize(const float* x, int N, int C, float eps, float* out, cudaStream_t stream, const int* n_dev = nullptr);
size_t detection_scores_workspace_bytes(int N, int B);
int detection_scores(const float* feats, const int* neighbors, const int* lengths, int B, int N, int H, int D,
                     float* out_scores, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                     const int* n_dev = nullptr);
int affine_leaky(const float* x, int N, int C, const float* scale, const float* shift, const float* residual,
                 float alpha, float* out, cudaStream_t stream, const int* n_dev = nullptr);

// ---- keypoints.cu -----------------------------------------------------------------------------------
size_t select_keypoints_workspace_bytes(int N, int B);
int select_keypoints(const float* scores, const int* lengths, int B, int N, int k, const float* points,
                     const float* descriptors, int D, int* out_order, int* out_index, int* out_count, float* out_points,
                     float* out_descriptors, float* out_scores, void* workspace, size_t workspace_bytes,
                     cudaStream_t stream, const int* n_dev = nullptr);

// ---- matching.cu ------------------------------------------------------------------------------------
size_t match_descriptors_workspace_bytes(int k, int P);
int match_descriptors(const float* desc, const int* count, int B, int k, int D, const int* pairs, int P, int* nn_st,
                      float* sim_st, int* nn_ts, float* sim_ts, int* matches, int* n_matches, void* workspace,
                      size_t workspace_bytes, cudaStream_t stream);

// ---- registration.cu --------------------------------------------------------------------------------
size_t register_pairs_workspace_bytes(int L, int P, int max_iterations, int max_validation);
int register_pairs(const float* points, const int* count, int B, int k, const int* corr, const int* n_corr, int L,
                   const int* pairs, int P, int ransac_n, int max_iterations, int max_validation, double distance,
                   double edge_ratio, unsigned long long seed, double* pose, int* n_inliers, int* hypothesis,
                   int* n_validated, void* workspace, size_t workspace_bytes, cudaStream_t stream);

// ---- icp.cu -----------------------------------------------------------------------------------------
size_t icp_pairs_workspace_bytes(int N, int B, int P, double distance, const float* host_bbox);
int icp_pairs(const float* points, const int* lengths, int B, int N, const int* n_dev, const float* host_bbox,
              const int* pairs, int P, const double* init, double distance, int max_iterations,
              double relative_fitness, double relative_rmse, double* pose, double* fitness, double* inlier_rmse,
              int* n_corr, int* iterations, void* workspace, size_t workspace_bytes, cudaStream_t stream);

// ---- evaluation.cu ----------------------------------------------------------------------------------
size_t evaluate_pairs_workspace_bytes(int P, int S);
int evaluate_pairs(const float* points, const int* count, int B, int k, const int* matches, const int* n_matches,
                   int L, const int* pairs, int P, const double* truth_pose, const double* truth_info,
                   const int* truth_flags, const double* const* poses, int S, const int* levels, int R,
                   double fmr_distance, double fmr_ratio, double repeat_distance, double err2, double rte_max,
                   double rre_max_deg, int* valid, int* n_match_inliers, double* inlier_ratio, int* fmr_hit,
                   int* n_repeated, double* repeatability, double* rte, double* rre_deg, double* rmse2, int* success,
                   int* recall_hit, double* totals, void* workspace, size_t workspace_bytes, cudaStream_t stream);

}  // namespace d3f

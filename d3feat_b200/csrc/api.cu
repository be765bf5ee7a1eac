// extern "C" entry points of libd3feat_b200.so (declared in include/d3feat_b200.h).
#include <stdarg.h>

#include "ops.cuh"

namespace d3f {

static thread_local char g_err[512] = "";
static thread_local long long g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return D3F_ERR_CUDA;
}

void count_launch(int n) { g_launches += n; }

}  // namespace d3f

using namespace d3f;

extern "C" {

int d3f_version(void) { return 100; }

const char* d3f_last_error(void) { return g_err; }

long long d3f_launch_count(void) { return g_launches; }

int d3f_bbox(const float* pts, int N, float* out_bbox, d3f_stream_t stream) {
  D3F_REQUIRE(pts != nullptr || N == 0, D3F_ERR_INVALID, "d3f_bbox: null points");
  D3F_REQUIRE(out_bbox != nullptr && N >= 0, D3F_ERR_INVALID, "d3f_bbox: bad arguments");
  return bbox_device(pts, N, out_bbox, (cudaStream_t)stream);
}

size_t d3f_grid_subsample_workspace_bytes(int N, int B) { return grid_subsample_workspace_bytes(N, B); }

int d3f_grid_subsample(const float* pts, const int* batch_len, int B, int N, float dl, const float* feats, int fdim,
                       const int* classes, int ldim, const float* host_bbox, float* out_pts, float* out_feats,
                       int* out_classes, int* out_batch_len, int* out_M, void* workspace, size_t workspace_bytes,
                       d3f_stream_t stream) {
  D3F_REQUIRE((pts != nullptr || N == 0) && batch_len != nullptr && out_pts != nullptr && out_batch_len != nullptr &&
                  out_M != nullptr && workspace != nullptr,
              D3F_ERR_INVALID, "d3f_grid_subsample: null pointer");
  D3F_REQUIRE((fdim == 0 || out_feats != nullptr) && (ldim == 0 || out_classes != nullptr), D3F_ERR_INVALID,
              "d3f_grid_subsample: missing feature / class output");
  return grid_subsample(pts, batch_len, B, N, dl, feats, fdim, classes, ldim, host_bbox, out_pts, out_feats,
                        out_classes, out_batch_len, out_M, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_voxel_down_sample_workspace_bytes(int N, int B) { return voxel_down_sample_workspace_bytes(N, B); }

int d3f_voxel_down_sample(const float* pts, const int* lengths, int B, int N, const int* n_dev, double voxel_size,
                          const float* host_bbox, float* out_pts, int* out_lengths, int* out_M, int out_capacity,
                          int* d_status, void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  return voxel_down_sample(pts, lengths, B, N, n_dev, voxel_size, host_bbox, out_pts, out_lengths, out_M, out_capacity,
                           d_status, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_radius_neighbors_workspace_bytes(int Ns, int B, float radius, const float* host_bbox) {
  return radius_neighbors_workspace_bytes(Ns, B, radius, host_bbox);
}

int d3f_radius_neighbors_build(const float* supports, const int* s_batch_len, int B, int Ns, float radius,
                               const float* host_bbox, void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  D3F_REQUIRE((supports != nullptr || Ns == 0) && s_batch_len != nullptr && workspace != nullptr, D3F_ERR_INVALID,
              "d3f_radius_neighbors_build: null pointer");
  return radius_neighbors_build(supports, s_batch_len, B, Ns, radius, host_bbox, workspace, workspace_bytes,
                                (cudaStream_t)stream);
}

int d3f_radius_neighbors_count(const float* queries, const int* q_batch_len, int Nq, const float* supports,
                               const int* s_batch_len, int B, int Ns, float radius, const float* host_bbox,
                               const void* workspace, int* counts, int* out_max, d3f_stream_t stream) {
  (void)supports;
  (void)s_batch_len;
  D3F_REQUIRE((queries != nullptr || Nq == 0) && q_batch_len != nullptr && workspace != nullptr, D3F_ERR_INVALID,
              "d3f_radius_neighbors_count: null pointer");
  return radius_neighbors_count(queries, q_batch_len, Nq, B, Ns, radius, host_bbox, workspace, counts, out_max,
                                (cudaStream_t)stream);
}

int d3f_radius_neighbors_fill(const float* queries, const int* q_batch_len, int Nq, const float* supports,
                              const int* s_batch_len, int B, int Ns, float radius, const float* host_bbox,
                              const void* workspace, int cols, int pad_value, int* out_idx, d3f_stream_t stream) {
  (void)supports;
  (void)s_batch_len;
  D3F_REQUIRE((queries != nullptr || Nq == 0) && q_batch_len != nullptr && workspace != nullptr, D3F_ERR_INVALID,
              "d3f_radius_neighbors_fill: null pointer");
  return radius_neighbors_fill(queries, q_batch_len, Nq, B, Ns, radius, host_bbox, workspace, cols, pad_value, out_idx,
                               (cudaStream_t)stream);
}

int d3f_radius_neighbors_order(const void* workspace, int Ns, int B, float radius, const float* host_bbox,
                               int* out_order, d3f_stream_t stream) {
  D3F_REQUIRE(workspace != nullptr && (out_order != nullptr || Ns == 0), D3F_ERR_INVALID,
              "d3f_radius_neighbors_order: null pointer");
  return radius_neighbors_order(workspace, Ns, B, radius, host_bbox, out_order, (cudaStream_t)stream);
}

size_t d3f_kpconv_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout) {
  return kpconv_workspace_bytes(Nq, Ns, H, K, Cin, Cout);
}

size_t d3f_pyramid_workspace_bytes(int B, const d3f_pyramid_spec* spec, const int* capacity, const float* host_bbox) {
  return pyramid_workspace_bytes(B, spec, capacity, host_bbox);
}

int d3f_pyramid_build(const float* points, const int* lengths, int B, int N0, const d3f_pyramid_spec* spec,
                      const float* host_bbox, float* const* out_points, int* const* out_lengths,
                      int* const* out_neighbors, int* const* out_pools, int* const* out_upsamples, const int* capacity,
                      int* out_level_sizes, void* workspace, size_t workspace_bytes, d3f_stream_t stream,
                      int* d_counts, int* d_status, const int* n0_dev) {
  D3F_REQUIRE((points != nullptr || N0 == 0) && lengths != nullptr && out_points && out_lengths && out_neighbors &&
                  out_pools && out_upsamples && workspace,
              D3F_ERR_INVALID, "d3f_pyramid_build: null pointer");
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "d3f_pyramid_build: B=%d", B);
  return pyramid_build(points, lengths, B, N0, spec, host_bbox, out_points, out_lengths, out_neighbors, out_pools,
                       out_upsamples, capacity, out_level_sizes, workspace, workspace_bytes, (cudaStream_t)stream,
                       d_counts, d_status, n0_dev);
}

size_t d3f_packed_weight_floats(int K, int N) { return tc_packed_floats(K, N); }

int d3f_pack_weight(const float* W, int K, int N, float* packed, d3f_stream_t stream) {
  return tc_pack_weight(W, K, N, packed, (cudaStream_t)stream);
}

int d3f_kpconv_forward(const float* q, const float* s, const int* idx, const float* feat, const float* Kp,
                       const float* W, const float* W_packed, const int* query_order, int Nq, int Ns, int H, int K, int Cin, int Cout, float extent, int influence,
                       int mode, int normalize, const float* bn_scale, const float* bn_shift, const float* bias,
                       float leaky_alpha, float* out, void* workspace, size_t workspace_bytes, d3f_stream_t stream,
                       const int* nq_dev, const int* ns_dev) {
  // an empty support set (Ns == 0: every index is the shadow point) has no coordinates or features to point at
  D3F_REQUIRE(Nq == 0 || (q && idx && Kp && W && out && workspace && (Ns == 0 || (s && feat))), D3F_ERR_INVALID,
              "d3f_kpconv_forward: null pointer");
  return kpconv_forward_impl(false, q, s, idx, feat, Kp, nullptr, nullptr, W, W_packed, query_order, Nq, Ns, H, K, Cin, Cout, extent,
                             influence, mode, normalize, bn_scale, bn_shift, bias, leaky_alpha, out, workspace,
                             workspace_bytes, (cudaStream_t)stream, nq_dev, ns_dev);
}

int d3f_kpconv_deform_forward(const float* q, const float* s, const int* idx, const float* feat, const float* Kp,
                              const float* offsets, const float* modulations, const float* W, const float* W_packed,
                              const int* query_order, int Nq, int Ns, int H, int K, int Cin, int Cout, float extent, int influence, int mode, const float* bn_scale,
                              const float* bn_shift, const float* bias, float leaky_alpha, float* out,
                              void* workspace, size_t workspace_bytes, d3f_stream_t stream, const int* nq_dev,
                              const int* ns_dev) {
  D3F_REQUIRE(Nq == 0 || (q && idx && Kp && W && out && workspace && offsets && (Ns == 0 || (s && feat))),
              D3F_ERR_INVALID, "d3f_kpconv_deform_forward: null pointer");
  return kpconv_forward_impl(true, q, s, idx, feat, Kp, offsets, modulations, W, W_packed, query_order, Nq, Ns, H, K, Cin, Cout, extent,
                             influence, mode, 0, bn_scale, bn_shift, bias, leaky_alpha, out, workspace,
                             workspace_bytes, (cudaStream_t)stream, nq_dev, ns_dev);
}

int d3f_unary_forward(const float* x, const float* W, const float* W_packed, int N, int Cin, int Cout,
                      const float* bn_scale,
                      const float* bn_shift, const float* bias, const float* residual, float leaky_alpha, float* out,
                      d3f_stream_t stream, const int* n_dev) {
  D3F_REQUIRE(N >= 0 && Cin >= 1 && Cout >= 1, D3F_ERR_INVALID, "d3f_unary_forward: bad shape N=%d Cin=%d Cout=%d", N,
              Cin, Cout);
  D3F_REQUIRE(N == 0 || (x && W && out), D3F_ERR_INVALID, "d3f_unary_forward: null pointer");
  D3F_REQUIRE((bn_scale == nullptr) == (bn_shift == nullptr), D3F_ERR_INVALID,
              "d3f_unary_forward: bn_scale/bn_shift mismatch");
  Epilogue ep;
  ep.rowscale = nullptr;
  ep.bn_scale = bn_scale;
  ep.bn_shift = bn_shift;
  ep.bias = bias;
  ep.residual = residual;
  ep.leaky_alpha = leaky_alpha;
  ep.row_map = nullptr;
  ep.m_dev = n_dev;
  if (W_packed != nullptr && tc_gemm_supported(x, Cin))
    return tc_gemm(x, W_packed, out, N, Cout, Cin, ep, (cudaStream_t)stream);
  return gemm_f32(x, W, out, N, Cout, Cin, ep, (cudaStream_t)stream);
}

int d3f_unary_pair_forward(const float* x1, int Cin1, const float* x2, int Cin2, const float* W_packed, int N,
                           int Cout, const float* shift, float leaky_alpha, float* out, d3f_stream_t stream,
                           const int* n_dev) {
  D3F_REQUIRE(N >= 0 && Cin1 >= 1 && Cin2 >= 1 && Cout >= 1, D3F_ERR_INVALID,
              "d3f_unary_pair_forward: bad shape N=%d Cin=%d+%d Cout=%d", N, Cin1, Cin2, Cout);
  D3F_REQUIRE(N == 0 || (x1 && x2 && W_packed && out), D3F_ERR_INVALID, "d3f_unary_pair_forward: null pointer");
  D3F_REQUIRE(Cin1 % 32 == 0 && Cin2 % 4 == 0, D3F_ERR_INVALID,
              "d3f_unary_pair_forward: Cin1 must be a multiple of 32 and Cin2 of 4 (got %d, %d)", Cin1, Cin2);
  Epilogue ep;
  ep.rowscale = nullptr;
  ep.bn_scale = nullptr;
  ep.bn_shift = nullptr;
  ep.bias = shift;
  ep.residual = nullptr;
  ep.leaky_alpha = leaky_alpha;
  ep.row_map = nullptr;
  ep.m_dev = n_dev;
  return tc_gemm(x1, W_packed, out, N, Cout, Cin1 + Cin2, ep, (cudaStream_t)stream, nullptr, x2, Cin1);
}

size_t d3f_kpconv_backward_workspace_bytes(int Nq, int Ns, int H, int K, int Cin, int Cout, int Hr) {
  return kpconv_backward_workspace_bytes(Nq, Ns, H, K, Cin, Cout, Hr);
}

int d3f_kpconv_reverse_width(const int* idx, int Nq, int Ns, int H, int* width, void* workspace,
                             size_t workspace_bytes, d3f_stream_t stream, const int* nq_dev, const int* ns_dev) {
  return kpconv_reverse_width(idx, Nq, Ns, H, width, workspace, workspace_bytes, (cudaStream_t)stream, nq_dev, ns_dev);
}

int d3f_kpconv_backward(const float* q, const float* s, const int* idx, const float* feat, const float* Kp,
                        const float* W, const float* dout, int Nq, int Ns, int H, int Hr, int K, int Cin, int Cout,
                        float extent, int influence, int mode, int normalize, int tensor_cores, float* dfeat,
                        float* dW, void* workspace, size_t workspace_bytes, d3f_stream_t stream, const int* nq_dev,
                        const int* ns_dev) {
  D3F_REQUIRE(Nq == 0 || Ns == 0 || (dfeat == nullptr && dW == nullptr) ||
                  (q && s && idx && feat && Kp && W && dout && workspace),
              D3F_ERR_INVALID, "d3f_kpconv_backward: null pointer");
  return kpconv_backward(q, s, idx, feat, Kp, W, dout, Nq, Ns, H, Hr, K, Cin, Cout, extent, influence, mode, normalize,
                         tensor_cores, dfeat, dW, workspace, workspace_bytes, (cudaStream_t)stream, nq_dev, ns_dev);
}

size_t d3f_unary_backward_workspace_bytes(int N, int Cin, int Cout) {
  return unary_backward_workspace_bytes(N, Cin, Cout);
}

int d3f_unary_backward(const float* x, const float* W, const float* dout, int N, int Cin, int Cout, int tensor_cores,
                       float* dx, float* dW, void* workspace, size_t workspace_bytes, d3f_stream_t stream,
                       const int* n_dev) {
  D3F_REQUIRE(N == 0 || (dx == nullptr && dW == nullptr) || (x && W && dout && workspace), D3F_ERR_INVALID,
              "d3f_unary_backward: null pointer");
  return unary_backward(x, W, dout, N, Cin, Cout, tensor_cores, dx, dW, workspace, workspace_bytes,
                        (cudaStream_t)stream, n_dev);
}

size_t d3f_ind_max_pool_workspace_bytes(int C) { return sizeof(unsigned) * ((size_t)(C > 0 ? C : 1) + 1); }

int d3f_ind_max_pool(const float* x, const int* inds, int N1, int N2, int H, int C, float* out, void* workspace,
                     size_t workspace_bytes, d3f_stream_t stream, const int* n1_dev, const int* n2_dev) {
  D3F_REQUIRE(N2 == 0 || (x && inds && out && workspace), D3F_ERR_INVALID, "d3f_ind_max_pool: null pointer");
  return ind_max_pool(x, inds, N1, N2, H, C, out, workspace, workspace_bytes, (cudaStream_t)stream, n1_dev, n2_dev);
}

int d3f_closest_pool(const float* x, const int* inds, int N1, int N2, int ld_inds, int C, float* out,
                     d3f_stream_t stream, const int* n1_dev, const int* n2_dev) {
  D3F_REQUIRE(N2 == 0 || (x && inds && out), D3F_ERR_INVALID, "d3f_closest_pool: null pointer");
  return closest_pool(x, inds, N1, N2, ld_inds, C, out, (cudaStream_t)stream, n1_dev, n2_dev);
}

int d3f_l2_normalize(const float* x, int N, int C, float eps, float* out, d3f_stream_t stream, const int* n_dev) {
  D3F_REQUIRE(N == 0 || (x && out), D3F_ERR_INVALID, "d3f_l2_normalize: null pointer");
  return l2_normalize(x, N, C, eps, out, (cudaStream_t)stream, n_dev);
}

size_t d3f_detection_scores_workspace_bytes(int N, int B) { return detection_scores_workspace_bytes(N, B); }

int d3f_detection_scores(const float* feats, const int* neighbors, const int* lengths, int B, int N, int H, int D,
                         float* out_scores, void* workspace, size_t workspace_bytes, d3f_stream_t stream,
                         const int* n_dev) {
  D3F_REQUIRE(N == 0 || (feats && (neighbors || H == 0) && lengths && out_scores && workspace), D3F_ERR_INVALID,
              "d3f_detection_scores: null pointer");
  return detection_scores(feats, neighbors, lengths, B, N, H, D, out_scores, workspace, workspace_bytes,
                          (cudaStream_t)stream, n_dev);
}

int d3f_affine_leaky(const float* x, int N, int C, const float* scale, const float* shift, const float* residual,
                     float leaky_alpha, float* out, d3f_stream_t stream, const int* n_dev) {
  D3F_REQUIRE(N == 0 || (x && out), D3F_ERR_INVALID, "d3f_affine_leaky: null pointer");
  return affine_leaky(x, N, C, scale, shift, residual, leaky_alpha, out, (cudaStream_t)stream, n_dev);
}

size_t d3f_batch_norm_train_workspace_bytes(int N, int C) { return batch_norm_train_workspace_bytes(N, C); }

int d3f_batch_norm_train_forward(const float* x, int N, int C, const float* gamma, const float* beta,
                                 float* moving_mean, float* moving_var, float decay, float eps, const float* residual,
                                 float leaky_alpha, float* out, float* mean, float* invstd, void* workspace,
                                 size_t workspace_bytes, d3f_stream_t stream) {
  return batch_norm_train_forward(x, N, C, gamma, beta, moving_mean, moving_var, decay, eps, residual, leaky_alpha, out,
                                  mean, invstd, workspace, workspace_bytes, (cudaStream_t)stream);
}

int d3f_batch_norm_train_backward(const float* x, const float* out, const float* dout, int N, int C,
                                  const float* gamma, const float* mean, const float* invstd, float leaky_alpha,
                                  float* dx, float* dresidual, float* dgamma, float* dbeta, void* workspace,
                                  size_t workspace_bytes, d3f_stream_t stream) {
  return batch_norm_train_backward(x, out, dout, N, C, gamma, mean, invstd, leaky_alpha, dx, dresidual, dgamma, dbeta,
                                   workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_ind_max_pool_backward_workspace_bytes(int N1, int N2, int H, int C) {
  return ind_max_pool_backward_workspace_bytes(N1, N2, H, C);
}

int d3f_ind_max_pool_backward(const float* x, const int* inds, const float* out, const float* dout, int N1, int N2,
                              int H, int C, float* dx, void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  return ind_max_pool_backward(x, inds, out, dout, N1, N2, H, C, dx, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_gather_rows_backward_workspace_bytes(int N1, int N2) { return gather_rows_backward_workspace_bytes(N1, N2); }

int d3f_gather_rows_backward(const int* inds, const float* dout, int N1, int N2, int C, float* dx, void* workspace,
                             size_t workspace_bytes, d3f_stream_t stream) {
  return gather_rows_backward(inds, dout, N1, N2, C, dx, workspace, workspace_bytes, (cudaStream_t)stream);
}

int d3f_l2_normalize_backward(const float* x, const float* dout, int N, int C, float eps, float* dx,
                              d3f_stream_t stream) {
  return l2_normalize_backward(x, dout, N, C, eps, dx, (cudaStream_t)stream);
}

size_t d3f_detection_scores_backward_workspace_bytes(int N, int H, int B, int D) {
  return detection_scores_backward_workspace_bytes(N, H, B, D);
}

int d3f_detection_scores_backward(const float* feats, const int* neighbors, const int* lengths, const float* dscores,
                                  int B, int N, int H, int D, float* dfeats, void* workspace, size_t workspace_bytes,
                                  d3f_stream_t stream) {
  return detection_scores_backward(feats, neighbors, lengths, dscores, B, N, H, D, dfeats, workspace, workspace_bytes,
                                   (cudaStream_t)stream);
}

size_t d3f_select_keypoints_workspace_bytes(int N, int B) { return select_keypoints_workspace_bytes(N, B); }

int d3f_select_keypoints(const float* scores, const int* lengths, int B, int N, int k, const float* points,
                         const float* descriptors, int D, int* out_order, int* out_index, int* out_count,
                         float* out_points, float* out_descriptors, float* out_scores, void* workspace,
                         size_t workspace_bytes, d3f_stream_t stream, const int* n_dev) {
  return select_keypoints(scores, lengths, B, N, k, points, descriptors, D, out_order, out_index, out_count, out_points,
                          out_descriptors, out_scores, workspace, workspace_bytes, (cudaStream_t)stream, n_dev);
}

size_t d3f_match_descriptors_workspace_bytes(int k, int P) { return match_descriptors_workspace_bytes(k, P); }

int d3f_match_descriptors(const float* desc, const int* count, int B, int k, int D, const int* pairs, int P,
                          int* nn_st, float* sim_st, int* nn_ts, float* sim_ts, int* matches, int* n_matches,
                          void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  return match_descriptors(desc, count, B, k, D, pairs, P, nn_st, sim_st, nn_ts, sim_ts, matches, n_matches, workspace,
                           workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_register_pairs_workspace_bytes(int L, int P, int max_iterations, int max_validation) {
  return register_pairs_workspace_bytes(L, P, max_iterations, max_validation);
}

int d3f_register_pairs(const float* points, const int* count, int B, int k, const int* corr, const int* n_corr, int L,
                       const int* pairs, int P, int ransac_n, int max_iterations, int max_validation, double distance,
                       double edge_ratio, unsigned long long seed, double* pose, int* n_inliers, int* hypothesis,
                       int* n_validated, void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  return register_pairs(points, count, B, k, corr, n_corr, L, pairs, P, ransac_n, max_iterations, max_validation,
                        distance, edge_ratio, seed, pose, n_inliers, hypothesis, n_validated, workspace,
                        workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_icp_pairs_workspace_bytes(int N, int B, int P, double distance, const float* host_bbox) {
  return icp_pairs_workspace_bytes(N, B, P, distance, host_bbox);
}

int d3f_icp_pairs(const float* points, const int* lengths, int B, int N, const int* n_dev, const float* host_bbox,
                  const int* pairs, int P, const double* init, double distance, int max_iterations,
                  double relative_fitness, double relative_rmse, double* pose, double* fitness, double* inlier_rmse,
                  int* n_corr, int* iterations, void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  return icp_pairs(points, lengths, B, N, n_dev, host_bbox, pairs, P, init, distance, max_iterations,
                   relative_fitness, relative_rmse, pose, fitness, inlier_rmse, n_corr, iterations, workspace,
                   workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_evaluate_pairs_workspace_bytes(int P, int S) { return evaluate_pairs_workspace_bytes(P, S); }

int d3f_evaluate_pairs(const float* points, const int* count, int B, int k, const int* matches, const int* n_matches,
                       int L, const int* pairs, int P, const double* truth_pose, const double* truth_info,
                       const int* truth_flags, const double* const* poses, int S, const int* levels, int R,
                       double fmr_distance, double fmr_ratio, double repeat_distance, double err2, double rte_max,
                       double rre_max_deg, int* valid, int* n_match_inliers, double* inlier_ratio, int* fmr_hit,
                       int* n_repeated, double* repeatability, double* rte, double* rre_deg, double* rmse2,
                       int* success, int* recall_hit, double* totals, void* workspace, size_t workspace_bytes,
                       d3f_stream_t stream) {
  return evaluate_pairs(points, count, B, k, matches, n_matches, L, pairs, P, truth_pose, truth_info, truth_flags,
                        poses, S, levels, R, fmr_distance, fmr_ratio, repeat_distance, err2, rte_max, rre_max_deg,
                        valid, n_match_inliers, inlier_ratio, fmr_hit, n_repeated, repeatability, rte, rre_deg, rmse2,
                        success, recall_hit, totals, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_pair_correspondences_workspace_bytes(int N, int B, int P, double distance, const float* host_bbox) {
  return pair_correspondences_workspace_bytes(N, B, P, distance, host_bbox);
}

int d3f_pair_correspondences_count(const float* points, const int* lengths, int B, int N, const float* host_bbox,
                                   const int* pairs, int P, const double* trans, double distance, int mode,
                                   long long* offset, int* count, double* overlap, void* workspace,
                                   size_t workspace_bytes, d3f_stream_t stream) {
  return pair_correspondences_count(points, lengths, B, N, host_bbox, pairs, P, trans, distance, mode, offset, count,
                                    overlap, workspace, workspace_bytes, (cudaStream_t)stream);
}

int d3f_pair_correspondences_fill(const float* points, int B, int N, const float* host_bbox, const int* pairs, int P,
                                  const double* trans, double distance, int mode, int M, int* rows, void* workspace,
                                  size_t workspace_bytes, d3f_stream_t stream) {
  return pair_correspondences_fill(points, B, N, host_bbox, pairs, P, trans, distance, mode, M, rows, workspace,
                                   workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_sample_correspondences_workspace_bytes(int M, int P) { return sample_correspondences_workspace_bytes(M, P); }

int d3f_sample_correspondences(const long long* offset, const int* rows, int M, int P, const int* anchor_len, int k,
                               int replace, int min_count, unsigned long long seed, int* anc, int* pos, int* valid,
                               void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  return sample_correspondences(offset, rows, M, P, anchor_len, k, replace, min_count, seed, anc, pos, valid,
                                workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t d3f_augment_pairs_workspace_bytes(int B, int P) { return augment_pairs_workspace_bytes(B, P); }

int d3f_augment_pairs(const float* points, const int* lengths, int B, int N, const int* pairs, int P,
                      const double* trans, unsigned long long seed, double noise, int num_axis, int scale_shift,
                      double scale_min, double scale_max, double shift_range, int capacity, float* out_points,
                      float* backup_points, int* out_lengths, long long* row_offset, float* R, double* scale,
                      double* shift, void* workspace, size_t workspace_bytes, d3f_stream_t stream) {
  return augment_pairs(points, lengths, B, N, pairs, P, trans, seed, noise, num_axis, scale_shift, scale_min, scale_max,
                       shift_range, capacity, out_points, backup_points, out_lengths, row_offset, R, scale, shift,
                       workspace, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"

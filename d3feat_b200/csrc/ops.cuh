// Internal (C++) interface between the translation units of the library. The public C ABI is include/d3feat_b200.h;
// each of its entry points is defined, extern "C", in the .cu file that implements it.
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
bool tc_gemm_supported(const float* A, int K);
int tc_gemm(const float* A, const float* Bp, float* C, int M, int N, int K, const Epilogue& ep, cudaStream_t stream,
            float* split_ws = nullptr, const float* A2 = nullptr, int K1 = 0);
size_t tc_gemm_split_ws_floats(int M, int N, int K);

// ---- grid.cu ----------------------------------------------------------------------------------------
int launch_batch_start(const int* len, int B, int* start, cudaStream_t stream);
int grid_subsample(const float* pts, const int* batch_len, int B, int N, float dl, const float* feats, int fdim,
                   const int* classes, int ldim, const float* host_bbox, float* out_pts, float* out_feats,
                   int* out_classes, int* out_batch_len, int* out_M, void* workspace, size_t workspace_bytes,
                   cudaStream_t stream, const int* n_dev = nullptr, int out_capacity = -1, int* status = nullptr,
                   const int* start_pre = nullptr);

// ---- neighbors.cu -----------------------------------------------------------------------------------
// ns_dev / nq_dev / pad_dev (optional): actual row counts / the shadow index in device memory; Ns / Nq are then capacities
int radius_neighbors_build(const float* supports, const int* s_batch_len, int B, int Ns, float radius,
                           const float* host_bbox, void* workspace, size_t workspace_bytes, cudaStream_t stream,
                           const int* ns_dev = nullptr, const int* s_start_pre = nullptr);
int radius_neighbors_fill(const float* queries, const int* q_batch_len, int Nq, int B, int Ns, float radius,
                          const float* host_bbox, const void* workspace, int cols, int pad_value, int* out_idx,
                          cudaStream_t stream, const int* nq_dev = nullptr, const int* pad_dev = nullptr,
                          const int* q_start_pre = nullptr);
struct NbView;   // nbgrid.cuh: the built grid, for nearest_in_cloud
int radius_neighbors_view(const void* workspace, int Ns, int B, float radius, const float* host_bbox, NbView* out);

// ---- kpconv.cu --------------------------------------------------------------------------------------
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
// Reverse neighbour table of idx[Nq, H] as a CSR, with no read-back: *sorted_q lists the query of every entry in
// ascending (s, q, h); support s owns [offs[s], offs[s] + counts[s]). Entries that are not real (q at or past the row
// count, idx < 0 or at or past the support count) sort last, are not counted and fill [offs[Ns], Nq * H). Sort
// buffers for Nq * H pairs (keys[0] / vals[0] are the input), counts and offs of Ns + 1 ints, scan_scratch of
// scan_num_blocks(Ns + 1) + 1 ints.
struct SortBuffers;
int reverse_csr(const int* idx, int Nq, int Ns, int H, const int* nq_dev, const int* ns_dev, const SortBuffers& sb,
                int* counts, int* offs, int* scan_scratch, const uint32_t** sorted_q, cudaStream_t stream);

// ---- kpconv_fused.cu (one persistent kernel per layer: gather + correlation + wgmma contraction) -------
bool kpconv_fused_supported(int Nq, int H, int K, int Cin, int Cout, int influence, int mode, const float* feat,
                            const float* W, const float* out, const int* query_order);
size_t kpconv_fused_image_floats();
int kpconv_fused_forward(const float* q, const float4* s4, const int* idx, const float* feat, const float* Kp,
                         const float* W, float* w_img, int Nq, int Ns, int H, int Cout, float extent, int normalize,
                         const float* bn_scale, const float* bn_shift, const float* bias, float leaky_alpha, float* out,
                         cudaStream_t stream, const int* nq_dev = nullptr, const int* ns_dev = nullptr);

}  // namespace d3f

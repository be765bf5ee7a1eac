// Ground-truth metrics of matched and registered cloud pairs -- the last stage of every reference test script, run
// there per pair on the host:
//   geometric_registration/evaluate.py:67-82, :207    feature-match recall (inlier ratio of the mutual matches)
//   repeatability/evaluate_3dmatch_our.py:30-41,       keypoint repeatability at 4 .. 512 keypoints
//   repeatability/evaluate_kitti_our.py:12-23
//   utils/tester.py:326-342                           KITTI RTE / RRE / success
//   3dmatch/evaluate.m, mrEvaluateRegistration.m       registration recall (Choi's error with the gt.info matrices)
//
// The contract is oracle/evaluate_np.py, exactly: every step is one correctly rounded fp64 operation in the order
// written there (solver.cuh), keypoints widened from fp32, every distance test d^2 < tau^2. rre_deg alone goes through
// acos, which is not correctly rounded, and agrees within a few ulp.
//
// eval_match_kernel   one warp per pair: whether the pair is evaluated, its FMR inliers over the mutual matches, the
//                     inlier ratio; it also zeroes the pair's repeatability counters.
// eval_repeat_kernel  one CTA per (pair, tile of kRepThreads target slots among the top n_max), grid-stride: the top
//                     n_max source keypoints, transformed by G, go through shared memory in chunks from the highest
//                     rank down; each target thread keeps a running min d^2 and a NaN flag and records its hit bit at
//                     every level boundary. Hits are counted with ballot / popc and one integer atomicAdd per (CTA,
//                     level), which is exact whatever the tile split.
// eval_pose_kernel    one thread per (pose set, pair): rte, the clamped cosine, rre_deg, success and Choi's error.
// eval_totals_kernel  one CTA: the per-pair contributions go through shared memory a pass of pairs at a time, and one
//                     lane per total of its first warp sums them sequentially in pair order (it also writes the
//                     per-pair repeatability).
// Launches are sized by (P, k, R, S) and the levels only; counts, pair ids, flags and truth are read on the device, so
// a call can be captured into a CUDA graph.
#include <cmath>

#include "ops.cuh"
#include "solver.cuh"

namespace d3f {

namespace {

constexpr int kMaxLevels = 14;           // 4 + 14 + 7 * 2 = 32 totals: one lane each
constexpr int kMaxPoseSets = 2;
constexpr int kPairWarps = 8;            // match kernel: one warp per pair
constexpr int kRepThreads = 128;         // repeatability: target slots per CTA
constexpr int kRepChunk = 256;           // repeatability: source ranks staged per chunk
constexpr int kRepCtasPerSM = 16;
constexpr int kPoseThreads = 128;
constexpr int kTotalsThreads = 128;     // totals: pairs staged per pass
constexpr double kRad2Deg = 180.0 / 3.141592653589793;   // 180 / pi, as the oracle's RAD2DEG

// bits of the per-(pose set, pair) decisions the totals kernel reads
constexpr int kRteOk = 1, kRreOk = 2, kRecallPair = 4, kRecallHit = 8;

struct EvalParams {
  int levels[kMaxLevels];
  int R, S;
  const double* pose[kMaxPoseSets];
  double tau_fmr2, fmr_ratio, tau_rep2, err2, rte_max, cos_max;
};

struct Outputs {
  int* valid;
  int* n_match_inliers;
  double* inlier_ratio;
  int* fmr_hit;
  int* n_repeated;
  double* repeatability;
  double* rte;
  double* rre_deg;
  double* rmse2;
  int* success;
  int* recall_hit;
  double* totals;
  int* bits;          // workspace [S, P]
};

// real slots of cloud b: clamp(count[b], 0, k)
__device__ __forceinline__ int real_slots(const int* __restrict__ count, int k, int b) {
  const int n = __ldg(count + b);
  return n < 0 ? 0 : (n < k ? n : k);
}

// flags bit 0 set and both cloud ids in [0, B)
__device__ __forceinline__ bool evaluated(const int* __restrict__ pairs, const int* __restrict__ flags, int B, int p,
                                          int& src, int& tgt) {
  src = __ldg(pairs + 2 * p);
  tgt = __ldg(pairs + 2 * p + 1);
  return (__ldg(flags + p) & 1) && src >= 0 && src < B && tgt >= 0 && tgt < B;
}

__device__ __forceinline__ void load_pose(const double* __restrict__ m, Pose& T) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int b = 0; b < 3; ++b) T.R[a][b] = m[4 * a + b];
    T.t[a] = m[4 * a + 3];
  }
}

__device__ __forceinline__ bool finite_pose(const Pose& T) {
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int b = 0; b < 3; ++b) ok = ok && isfinite(T.R[a][b]);
    ok = ok && isfinite(T.t[a]);
  }
  return ok;
}

__device__ __forceinline__ void load3(const float* __restrict__ points, size_t slot, float v[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) v[a] = __ldg(points + 3 * slot + a);
}

__global__ void __launch_bounds__(kPairWarps * 32)
eval_match_kernel(const float* __restrict__ points, const int* __restrict__ count, int B, int k,
                  const int* __restrict__ matches, const int* __restrict__ n_matches, int L,
                  const int* __restrict__ pairs, const int* __restrict__ flags, const double* __restrict__ truth, int P,
                  int R, double tau2, double fmr_ratio, Outputs o) {
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * kPairWarps + (threadIdx.x >> 5);
  if (p >= P) return;                                          // uniform across the warp
  if (lane < R) o.n_repeated[(size_t)p * R + lane] = 0;       // counted by eval_repeat_kernel
  int src, tgt;
  if (!evaluated(pairs, flags, B, p, src, tgt)) {
    if (lane == 0) {
      o.valid[p] = 0;
      o.n_match_inliers[p] = 0;
      o.inlier_ratio[p] = 0.0;
      o.fmr_hit[p] = 0;
    }
    return;
  }
  Pose G;
  load_pose(truth + (size_t)p * 16, G);
  const int ns = real_slots(count, k, src), nt = real_slots(count, k, tgt);
  const int nm = min(max(__ldg(n_matches + p), 0), L);
  const int* row = matches + (size_t)p * L * 2;
  int n = 0;
  for (int m = lane; m < nm; m += 32) {
    const int i = __ldg(row + 2 * m), j = __ldg(row + 2 * m + 1);
    if (i >= 0 && i < ns && j >= 0 && j < nt) {                // a row naming a slot that is not real: no inlier
      float s[3], t[3];
      load3(points, (size_t)src * k + i, s);
      load3(points, (size_t)tgt * k + j, t);
      n += residual2(G, s, t) < tau2;
    }
  }
  n = __reduce_add_sync(0xffffffffu, n);
  if (lane == 0) {
    const double ratio = nm > 0 ? ddiv((double)n, (double)nm) : 0.0;
    o.valid[p] = 1;
    o.n_match_inliers[p] = n;
    o.inlier_ratio[p] = ratio;
    o.fmr_hit[p] = ratio > fmr_ratio;
  }
}

__global__ void __launch_bounds__(kRepThreads)
eval_repeat_kernel(const float* __restrict__ points, const int* __restrict__ count, int B, int k,
                   const int* __restrict__ pairs, const int* __restrict__ flags, const double* __restrict__ truth,
                   int P, int tiles, const __grid_constant__ EvalParams prm, int* __restrict__ n_repeated) {
  __shared__ double qs[kRepChunk][3];
  __shared__ int hits[kMaxLevels];
  const int R = prm.R, n_max = prm.levels[R - 1];
  const int items = P * tiles;                                 // P * k is within int32 (host check)
  for (int e = blockIdx.x; e < items; e += gridDim.x) {
    const int p = e / tiles, tile = e - p * tiles;
    int src, tgt;
    if (!evaluated(pairs, flags, B, p, src, tgt)) continue;   // uniform across the CTA
    const int ns = real_slots(count, k, src), nt = real_slots(count, k, tgt);
    const int j0 = max(0, nt - n_max) + tile * kRepThreads;
    if (ns == 0 || j0 >= nt) continue;                         // no source slot, or no target slot in this tile
    Pose G;
    load_pose(truth + (size_t)p * 16, G);
    const int j = j0 + threadIdx.x;
    const bool has = j < nt;
    float t[3] = {0.f, 0.f, 0.f};
    if (has) load3(points, (size_t)tgt * k + j, t);
    if (threadIdx.x < R) hits[threadIdx.x] = 0;
    double mn = INFINITY;
    bool nan = false;
    unsigned bits = 0;
    int r = 0, bound = min(prm.levels[0], ns);                 // level r is recorded after `bound` source ranks
    const int m_end = min(n_max, ns);
    for (int c0 = 0; c0 < m_end; c0 += kRepChunk) {
      const int c1 = min(m_end, c0 + kRepChunk);
      __syncthreads();                                         // the previous chunk is consumed; hits is zeroed
      for (int m = c0 + threadIdx.x; m < c1; m += kRepThreads) {
        float s[3];
        load3(points, (size_t)src * k + (ns - 1 - m), s);      // rank m: the m-th highest score
#pragma unroll
        for (int a = 0; a < 3; ++a)
          qs[m - c0][a] = dadd(dadd(dadd(dmul(G.R[a][0], s[0]), dmul(G.R[a][1], s[1])), dmul(G.R[a][2], s[2])), G.t[a]);
      }
      __syncthreads();
      for (int m = c0; m < c1; ++m) {
        if (has) {
          const double e0 = dsub(qs[m - c0][0], t[0]), e1 = dsub(qs[m - c0][1], t[1]), e2 = dsub(qs[m - c0][2], t[2]);
          const double d2 = dadd(dadd(dmul(e0, e0), dmul(e1, e1)), dmul(e2, e2));
          if (isnan(d2)) nan = true;
          else if (d2 < mn) mn = d2;
        }
        while (m + 1 == bound) {                               // uniform: every thread walks the same ranks
          const bool hit = has && j >= nt - prm.levels[r] && !nan && mn < prm.tau_rep2;
          bits |= (unsigned)hit << r;
          if (++r == R) break;
          bound = min(prm.levels[r], ns);
        }
      }
    }
    for (int q = 0; q < R; ++q) {
      const int c = __popc(__ballot_sync(0xffffffffu, (bits >> q) & 1u));
      if ((threadIdx.x & 31) == 0 && c) atomicAdd(&hits[q], c);
    }
    __syncthreads();
    if (threadIdx.x < R && hits[threadIdx.x]) atomicAdd(n_repeated + (size_t)p * R + threadIdx.x, hits[threadIdx.x]);
    __syncthreads();                                           // qs and hits are reused by the next item
  }
}

__global__ void __launch_bounds__(kPoseThreads)
eval_pose_kernel(const int* __restrict__ pairs, const int* __restrict__ flags, const double* __restrict__ truth,
                 const double* __restrict__ info, int B, int P, const __grid_constant__ EvalParams prm, Outputs o) {
  const int e = blockIdx.x * kPoseThreads + threadIdx.x;
  if (e >= prm.S * P) return;
  const int s = e / P, p = e - s * P;
  double rte = NAN, rre = NAN, err = NAN;
  int bits = 0;
  int src, tgt;
  if (evaluated(pairs, flags, B, p, src, tgt)) {
    Pose G, T;
    load_pose(truth + (size_t)p * 16, G);
    load_pose(prm.pose[s] + (size_t)p * 16, T);
    const bool recall_pair = info != nullptr && (__ldg(flags + p) & 2);
    double c = NAN;
    if (finite_pose(G) && finite_pose(T)) {
      const double d0 = dsub(T.t[0], G.t[0]), d1 = dsub(T.t[1], G.t[1]), d2 = dsub(T.t[2], G.t[2]);
      rte = dsqrt(dadd(dadd(dmul(d0, d0), dmul(d1, d1)), dmul(d2, d2)));
      double col[3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
        col[i] = dadd(dadd(dmul(T.R[0][i], G.R[0][i]), dmul(T.R[1][i], G.R[1][i])), dmul(T.R[2][i], G.R[2][i]));
      c = ddiv(dsub(dadd(dadd(col[0], col[1]), col[2]), 1.0), 2.0);
      c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
      rre = dmul(acos(c), kRad2Deg);
      if (recall_pair) {
        // E = G inv(T), inv(T) = [R^T | -R^T t]; then dcm2quat and er^T info er / info_00
        double ti[3], E[3][3], er[6];
#pragma unroll
        for (int a = 0; a < 3; ++a)
          ti[a] = -dadd(dadd(dmul(T.R[0][a], T.t[0]), dmul(T.R[1][a], T.t[1])), dmul(T.R[2][a], T.t[2]));
#pragma unroll
        for (int a = 0; a < 3; ++a) {
#pragma unroll
          for (int b = 0; b < 3; ++b)
            E[a][b] = dadd(dadd(dmul(G.R[a][0], T.R[b][0]), dmul(G.R[a][1], T.R[b][1])), dmul(G.R[a][2], T.R[b][2]));
          er[a] = dadd(dadd(dadd(dmul(G.R[a][0], ti[0]), dmul(G.R[a][1], ti[1])), dmul(G.R[a][2], ti[2])), G.t[a]);
        }
        const double q0 = dmul(0.5, dsqrt(dadd(dadd(dadd(1.0, E[0][0]), E[1][1]), E[2][2])));
        const double d = dmul(4.0, q0);
        er[3] = -ddiv(-dsub(E[2][1], E[1][2]), d);
        er[4] = -ddiv(-dsub(E[0][2], E[2][0]), d);
        er[5] = -ddiv(-dsub(E[1][0], E[0][1]), d);
        const double* I = info + (size_t)p * 36;
        double num = 0.0;
        for (int jj = 0; jj < 6; ++jj) {
          double v = 0.0;
          for (int i = 0; i < 6; ++i) v = dadd(v, dmul(er[i], I[6 * i + jj]));
          num = dadd(num, dmul(v, er[jj]));
        }
        err = ddiv(num, I[0]);
      }
    }
    if (rte < prm.rte_max) bits |= kRteOk;
    if (c > prm.cos_max) bits |= kRreOk;
    if (recall_pair) bits |= kRecallPair;
    if (recall_pair && err <= prm.err2) bits |= kRecallHit;
  }
  const size_t i = (size_t)s * P + p;
  o.rte[i] = rte;
  o.rre_deg[i] = rre;
  o.rmse2[i] = err;
  o.success[i] = (bits & (kRteOk | kRreOk)) == (kRteOk | kRreOk);
  o.recall_hit[i] = (bits & kRecallHit) != 0;
  o.bits[i] = bits;
}

// Each CTA pass stages the contributions of kTotalsThreads consecutive pairs (0.0 where a pair does not count: every
// contribution is >= +0.0, so adding it leaves the sum's bits unchanged), then lane q of warp 0 adds total q's column
// in pair order.
__global__ void __launch_bounds__(kTotalsThreads)
eval_totals_kernel(int P, const __grid_constant__ EvalParams prm, Outputs o) {
  __shared__ double v[32][kTotalsThreads + 1];
  const int R = prm.R, S = prm.S, T = 4 + R + 7 * S, i = threadIdx.x;
  double acc = 0.0;
  for (int c0 = 0; c0 < P; c0 += kTotalsThreads) {
    const int p = c0 + i;
    if (p < P) {
      const bool ok = o.valid[p] != 0;
      v[0][i] = ok ? 1.0 : 0.0;
      v[1][i] = (double)o.fmr_hit[p];
      v[2][i] = o.inlier_ratio[p];
      v[3][i] = (double)o.n_match_inliers[p];
      for (int r = 0; r < R; ++r) {
        const double rep = ok ? ddiv((double)o.n_repeated[(size_t)p * R + r], (double)prm.levels[r]) : 0.0;
        o.repeatability[(size_t)p * R + r] = rep;
        v[4 + r][i] = rep;
      }
      for (int s = 0; s < S; ++s) {
        const size_t e = (size_t)s * P + p;
        const int b = o.bits[e];
        double* w = &v[4 + R + 7 * s][0];
        const int ld = kTotalsThreads + 1;
        w[0 * ld + i] = (b & (kRteOk | kRreOk)) == (kRteOk | kRreOk) ? 1.0 : 0.0;
        w[1 * ld + i] = (b & kRteOk) ? o.rte[e] : 0.0;
        w[2 * ld + i] = (b & kRteOk) ? 1.0 : 0.0;
        w[3 * ld + i] = (b & kRreOk) ? o.rre_deg[e] : 0.0;
        w[4 * ld + i] = (b & kRreOk) ? 1.0 : 0.0;
        w[5 * ld + i] = (b & kRecallHit) ? 1.0 : 0.0;
        w[6 * ld + i] = (b & kRecallPair) ? 1.0 : 0.0;
      }
    }
    __syncthreads();
    if (i < T) {
      const int n = min(kTotalsThreads, P - c0);
      for (int j = 0; j < n; ++j) acc = dadd(acc, v[i][j]);
    }
    __syncthreads();                     // v is refilled by the next pass
  }
  if (i < T) o.totals[i] = acc;
}

bool finite_positive(double x) { return std::isfinite(x) && x > 0.0; }

// one int per pair and pose set (at least one set)
size_t eval_layout(int P, int S, void* base, int** scratch) {
  if (P < 1 || S < 0 || S > kMaxPoseSets) return 0;
  Carver cv(base);
  int* s = cv.take<int>((size_t)(S > 0 ? S : 1) * P);
  if (scratch != nullptr) *scratch = s;
  return cv.off;
}

}  // namespace
}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_evaluate_pairs_workspace_bytes(int P, int S) { return eval_layout(P, S, nullptr, nullptr); }

extern "C" int d3f_evaluate_pairs(const float* points, const int* count, int B, int k, const int* matches,
                                  const int* n_matches, int L, const int* pairs, int P, const double* truth_pose,
                                  const double* truth_info, const int* truth_flags, const double* const* poses, int S,
                                  const int* levels, int R, double fmr_distance, double fmr_ratio,
                                  double repeat_distance, double err2, double rte_max, double rre_max_deg, int* valid,
                                  int* n_match_inliers, double* inlier_ratio, int* fmr_hit, int* n_repeated,
                                  double* repeatability, double* rte, double* rre_deg, double* rmse2, int* success,
                                  int* recall_hit, double* totals, void* workspace, size_t workspace_bytes,
                                  d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "evaluate_pairs: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(k >= 1 && L >= 1 && P >= 1, D3F_ERR_INVALID, "evaluate_pairs: bad shape k=%d L=%d P=%d", k, L, P);
  D3F_REQUIRE((long long)P * k <= INT32_MAX && (long long)P * L * 2 <= INT32_MAX && (long long)B * k * 3 <= INT32_MAX,
              D3F_ERR_INVALID, "evaluate_pairs: P*k, P*L*2 or B*k*3 exceeds int32 (B=%d k=%d L=%d P=%d)", B, k, L, P);
  D3F_REQUIRE(S >= 0 && S <= kMaxPoseSets, D3F_ERR_INVALID, "evaluate_pairs: S=%d pose sets must be in [0,%d]", S,
              kMaxPoseSets);
  D3F_REQUIRE(R >= 0 && R <= kMaxLevels, D3F_ERR_INVALID, "evaluate_pairs: R=%d levels must be in [0,%d]", R,
              kMaxLevels);
  D3F_REQUIRE(R == 0 || levels != nullptr, D3F_ERR_INVALID, "evaluate_pairs: null pointer (levels)");
  for (int r = 0; r < R; ++r)
    D3F_REQUIRE(levels[r] >= 1 && levels[r] <= k && (r == 0 || levels[r] > levels[r - 1]), D3F_ERR_INVALID,
                "evaluate_pairs: levels must ascend strictly within [1, k=%d] (levels[%d]=%d)", k, r, levels[r]);
  D3F_REQUIRE(finite_positive(fmr_distance) && finite_positive(repeat_distance), D3F_ERR_INVALID,
              "evaluate_pairs: fmr_distance=%g and repeat_distance=%g must be finite and > 0", fmr_distance,
              repeat_distance);
  D3F_REQUIRE(std::isfinite(fmr_ratio) && fmr_ratio >= 0.0 && fmr_ratio < 1.0, D3F_ERR_INVALID,
              "evaluate_pairs: fmr_ratio=%g must be in [0, 1)", fmr_ratio);
  D3F_REQUIRE(finite_positive(err2) && finite_positive(rte_max), D3F_ERR_INVALID,
              "evaluate_pairs: err2=%g and rte_max=%g must be finite and > 0", err2, rte_max);
  D3F_REQUIRE(std::isfinite(rre_max_deg) && rre_max_deg > 0.0 && rre_max_deg <= 180.0, D3F_ERR_INVALID,
              "evaluate_pairs: rre_max_deg=%g must be in (0, 180]", rre_max_deg);
  D3F_REQUIRE(points && count && matches && n_matches && pairs && truth_pose && truth_flags && valid &&
                  n_match_inliers && inlier_ratio && fmr_hit && totals && workspace &&
                  (R == 0 || (n_repeated && repeatability)) &&
                  (S == 0 || (poses && rte && rre_deg && rmse2 && success && recall_hit)),
              D3F_ERR_INVALID, "evaluate_pairs: null pointer");
  for (int s = 0; s < S; ++s)
    D3F_REQUIRE(poses[s] != nullptr, D3F_ERR_INVALID, "evaluate_pairs: null pointer (poses[%d])", s);
  int* scratch;
  const size_t need = eval_layout(P, S, workspace, &scratch);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE,
              "evaluate_pairs: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
  EvalParams prm = {};
  for (int r = 0; r < R; ++r) prm.levels[r] = levels[r];
  prm.R = R;
  prm.S = S;
  for (int s = 0; s < S; ++s) prm.pose[s] = poses[s];
  prm.tau_fmr2 = fmr_distance * fmr_distance;
  prm.fmr_ratio = fmr_ratio;
  prm.tau_rep2 = repeat_distance * repeat_distance;
  prm.err2 = err2;
  prm.rte_max = rte_max;
  prm.cos_max = std::cos(rre_max_deg * (3.141592653589793 / 180.0));   // the oracle's math.cos(deg * (pi / 180))
  Outputs o = {valid, n_match_inliers, inlier_ratio, fmr_hit, n_repeated, repeatability, rte, rre_deg, rmse2,
               success, recall_hit, totals, scratch};
  eval_match_kernel<<<ceil_div(P, kPairWarps), kPairWarps * 32, 0, stream>>>(
      points, count, B, k, matches, n_matches, L, pairs, truth_flags, truth_pose, P, R, prm.tau_fmr2, fmr_ratio, o);
  D3F_LAUNCH_CHECK("eval_match_kernel");
  if (R > 0) {
    const int tiles = ceil_div(levels[R - 1], kRepThreads);
    const int grid = (int)std::min<long long>((long long)P * tiles, (long long)kRepCtasPerSM * kNumSMs);
    eval_repeat_kernel<<<grid, kRepThreads, 0, stream>>>(points, count, B, k, pairs, truth_flags, truth_pose, P,
                                                          tiles, prm, n_repeated);
    D3F_LAUNCH_CHECK("eval_repeat_kernel");
  }
  if (S > 0) {
    eval_pose_kernel<<<ceil_div(S * P, kPoseThreads), kPoseThreads, 0, stream>>>(pairs, truth_flags, truth_pose,
                                                                                  truth_info, B, P, prm, o);
    D3F_LAUNCH_CHECK("eval_pose_kernel");
  }
  eval_totals_kernel<<<1, kTotalsThreads, 0, stream>>>(P, prm, o);
  D3F_LAUNCH_CHECK("eval_totals_kernel");
  return D3F_OK;
}

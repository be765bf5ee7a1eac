// RANSAC registration of cloud pairs from keypoint correspondences -- the host step every consumer of the matches runs:
//   geometric_registration/evaluate.py:84-99   3DMatch: ransac_n 3, distance 0.05, edge 0.9, (50000, 1000)
//   utils/tester.py:305-316                    KITTI: ransac_n 4, distance = voxel size, the same checkers
//   demo_registration.py:184-192               ransac_n 4, (4000000, 500)
// all Open3D's registration_ransac_based_on_correspondence / _feature_matching on the host, one pair at a time.
//
// The contract is oracle/register_np.py, exactly: every step is one correctly rounded fp64 operation (__dadd_rn,
// __dsub_rn, __dmul_rn, __ddiv_rn, __dsqrt_rn) in the order written there, so the multiply-adds are never contracted;
// sums run sequentially in ascending index. Hypothesis h of pair p samples idx_m = ((z >> 32) * n_c) >> 32 with
// z = splitmix64(seed + (((p << 32) | h) * 8 + m) * golden); a repeated index rejects it, then the edge-length
// checker, a Horn pose of the sample (cyclic Jacobi on the 4x4 quaternion matrix, kSweeps sweeps) and the distance
// checker. Only the first V validated hypotheses in ascending h are scored; the best has the most inliers
// (d^2 < tau^2), then the smaller sum of inlier d^2, then the smaller h, and its pose is refit over its inliers.
//
// reg_prepare_kernel     one warp per pair: validates the pair's clouds and real rows, resets the validated count.
// reg_hypothesis_kernel  one thread per hypothesis (many CTAs per pair), a round of h at a time; one validation bit
//                        per hypothesis (a warp ballot). Pairs that already hold V validated hypotheses skip the round.
// reg_select_kernel      one warp per pair: scans the round's bits in ascending h and lists validated hypotheses
//                        until V. Rounds double in length, so the early exit wastes at most one round's work.
// reg_score_kernel       one thread per listed hypothesis, sequentially over the pair's rows (staged in smem).
// reg_finalize_kernel    one CTA per pair: the best by a total order on (inliers, sum, h) -- independent of CTA and
//                        thread order -- and the refit (one thread sums, in row order, over smem tiles of flags).
// Launches are sized by (P, T, L); counts, pair ids and n_corr are read from the device: graph-capturable.
#include <algorithm>
#include <cmath>

#include "ops.cuh"
#include "rng.cuh"
#include "solver.cuh"

namespace d3f {

namespace {

constexpr int kHypThreads = 128;
constexpr int kScoreThreads = 128;
constexpr int kFinalizeThreads = 256;
constexpr int kWarpsPerCta = 8;          // prepare / select: one warp per pair
constexpr int kSelectWords = 8;          // validation words per lane and select iteration
constexpr int kFirstRound = 8192;        // hypotheses per pair in the first round; each later round is twice as long

// the source and target point of correspondence row r of pair p (the row was validated by reg_prepare_kernel)
struct Rows {
  const float* points;
  const int* corr;
  int k, L;
  template <typename F>
  __device__ __forceinline__ void load(int p, int src, int tgt, int r, F s[3], F t[3]) const {
    // two 4-byte loads: a caller's corr is only known to be int-aligned (a slice of a longer match buffer)
    const int* c = corr + 2 * ((size_t)p * L + r);
    const float* ps = points + ((size_t)src * k + __ldg(c)) * 3;
    const float* pt = points + ((size_t)tgt * k + __ldg(c + 1)) * 3;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      s[i] = __ldg(ps + i);
      t[i] = __ldg(pt + i);
    }
  }
};

__device__ __forceinline__ double length(const float a[3], const float b[3]) {
  const double dx = dsub(a[0], b[0]), dy = dsub(a[1], b[1]), dz = dsub(a[2], b[2]);
  return dsqrt(dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz)));
}

// Hypothesis h of pair p: sample, repeated-index rejection, edge checker, Horn pose, distance checker. Returns
// whether it is validated; `pose` is the sample pose whenever the sample reached the Horn solve.
template <int N>
__device__ bool hypothesis(const Rows& rows, int p, int src, int tgt, int h, int n_c, unsigned long long seed,
                           double ratio, double tau2, Pose& pose) {
  int idx[N];
#pragma unroll
  for (int m = 0; m < N; ++m) idx[m] = sample_index(p, h, m, n_c, seed);
#pragma unroll
  for (int a = 0; a < N; ++a)
#pragma unroll
    for (int b = a + 1; b < N; ++b)
      if (idx[a] == idx[b]) return false;
  float s[N][3], t[N][3];      // fp32 points; every use widens them to fp64 exactly
#pragma unroll
  for (int m = 0; m < N; ++m) rows.load(p, src, tgt, idx[m], s[m], t[m]);
#pragma unroll
  for (int a = 0; a < N; ++a)
#pragma unroll
    for (int b = a + 1; b < N; ++b) {
      const double ls = length(s[a], s[b]), lt = length(t[a], t[b]);
      if (ls < dmul(ratio, lt) || lt < dmul(ratio, ls)) return false;
    }
  double cs[3], ct[3], H[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double ss = 0.0, st = 0.0;
#pragma unroll
    for (int m = 0; m < N; ++m) {
      ss = dadd(ss, s[m][i]);
      st = dadd(st, t[m][i]);
    }
    cs[i] = ddiv(ss, (double)N);
    ct[i] = ddiv(st, (double)N);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double acc = 0.0;
#pragma unroll
      for (int m = 0; m < N; ++m) acc = dadd(acc, dmul(dsub(s[m][i], cs[i]), dsub(t[m][j], ct[j])));
      H[i][j] = acc;
    }
  pose_from_moments(cs, ct, H, pose);
  bool ok = true;
#pragma unroll
  for (int m = 0; m < N; ++m) ok = ok && residual2(pose, s[m], t[m]) <= tau2;
  return ok;
}

__device__ __forceinline__ bool cloud_ok(int b, int B) { return b >= 0 && b < B; }

// nc_eff[p] = n_c, or -1 for a pair that registers nothing (a cloud outside [0, B) or a real row naming a slot outside
// its cloud's count); n_val[p] = 0
__global__ void __launch_bounds__(kWarpsPerCta * 32)
reg_prepare_kernel(const int* __restrict__ count, int B, int k, const int* __restrict__ corr,
                   const int* __restrict__ n_corr, int L, const int* __restrict__ pairs, int P, int* __restrict__ nc_eff,
                   int* __restrict__ n_val) {
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  if (p >= P) return;
  const int src = __ldg(pairs + 2 * p), tgt = __ldg(pairs + 2 * p + 1);
  int nc = -1;
  if (cloud_ok(src, B) && cloud_ok(tgt, B)) {
    const int ns = min(max(__ldg(count + src), 0), k), nt = min(max(__ldg(count + tgt), 0), k);
    nc = min(max(__ldg(n_corr + p), 0), L);
    bool bad = false;
    for (int r = lane; r < nc; r += 32) {
      const int cs = __ldg(corr + 2 * ((size_t)p * L + r)), ct = __ldg(corr + 2 * ((size_t)p * L + r) + 1);
      bad = bad || cs < 0 || cs >= ns || ct < 0 || ct >= nt;
    }
    if (__any_sync(0xffffffffu, bad)) nc = -1;
  }
  if (lane == 0) {
    nc_eff[p] = nc;
    n_val[p] = 0;
  }
}

// hypotheses [h0, h0 + 32 * W) of every pair still short of V validated ones; bit (h & 31) of bits[p, h >> 5]
template <int N>
__global__ void __launch_bounds__(kHypThreads, 1)
reg_hypothesis_kernel(Rows rows, const int* __restrict__ pairs, int P, const int* __restrict__ nc_eff,
                      const int* __restrict__ n_val, int T, int V, int h0, int W, int WT, unsigned long long seed,
                      double ratio, double tau2, unsigned* __restrict__ bits) {
  const long long per_pair = 32ll * W;
  const long long total = per_pair * P;
  for (long long e = (long long)blockIdx.x * kHypThreads + threadIdx.x; e < total;
       e += (long long)gridDim.x * kHypThreads) {   // per_pair is a multiple of 32: a warp is one pair, uniform exit
    const int p = (int)(e / per_pair);
    const int h = h0 + (int)(e - (long long)p * per_pair);
    const int nc = __ldg(nc_eff + p);
    if (nc < N || __ldg(n_val + p) >= V) continue;
    bool ok = false;
    if (h < T) {
      Pose pose;
      ok = hypothesis<N>(rows, p, __ldg(pairs + 2 * p), __ldg(pairs + 2 * p + 1), h, nc, seed, ratio, tau2, pose);
    }
    const unsigned word = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0) bits[(size_t)p * WT + (h >> 5)] = word;
  }
}

// appends the validated hypotheses of [h0, h1) to list[p, :V] in ascending h
__global__ void __launch_bounds__(kWarpsPerCta * 32)
reg_select_kernel(int P, int N, const int* __restrict__ nc_eff, int* __restrict__ n_val, int V, int h0, int h1,
                  int WT, const unsigned* __restrict__ bits, int* __restrict__ list) {
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  if (p >= P || nc_eff[p] < N) return;
  int nv = n_val[p];
  const unsigned* pb = bits + (size_t)p * WT;
  const int w1 = (h1 + 31) >> 5;
  for (int w0 = h0 >> 5; w0 < w1 && nv < V; w0 += 32 * kSelectWords) {
    unsigned wd[kSelectWords];
    int c = 0;
#pragma unroll
    for (int i = 0; i < kSelectWords; ++i) {
      const int w = w0 + lane * kSelectWords + i;
      wd[i] = w < w1 ? pb[w] : 0u;
      c += __popc(wd[i]);
    }
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    int pos = nv + incl - c;
#pragma unroll
    for (int i = 0; i < kSelectWords; ++i) {
      for (unsigned b = wd[i]; b && pos < V; b &= b - 1, ++pos)
        list[(size_t)p * V + pos] = (w0 + lane * kSelectWords + i) * 32 + __ffs(b) - 1;
    }
    nv = min(V, nv + __shfl_sync(0xffffffffu, incl, 31));
  }
  if (lane == 0) n_val[p] = nv;
}

// inlier count and sequential sum of inlier d^2 of every listed hypothesis
template <int N>
__global__ void __launch_bounds__(kScoreThreads, 1)
reg_score_kernel(Rows rows, const int* __restrict__ pairs, int P, const int* __restrict__ nc_eff,
                 const int* __restrict__ n_val, const int* __restrict__ list, int V, unsigned long long seed,
                 double ratio, double tau2, int* __restrict__ inliers, double* __restrict__ sums) {
  __shared__ float tile[kScoreThreads][6];
  const int per_pair = ceil_div(V, kScoreThreads);
  const int p = blockIdx.x / per_pair;
  const int v = (blockIdx.x - p * per_pair) * kScoreThreads + threadIdx.x;
  const int nc = nc_eff[p];
  if (nc < N) return;
  const int nv = n_val[p];
  if ((blockIdx.x - p * per_pair) * kScoreThreads >= nv) return;     // uniform across the CTA
  const int src = __ldg(pairs + 2 * p), tgt = __ldg(pairs + 2 * p + 1);
  Pose pose;
  if (v < nv) hypothesis<N>(rows, p, src, tgt, list[(size_t)p * V + v], nc, seed, ratio, tau2, pose);
  int cnt = 0;
  double sum = 0.0;
  for (int r0 = 0; r0 < nc; r0 += kScoreThreads) {
    __syncthreads();
    if (r0 + threadIdx.x < nc) rows.load(p, src, tgt, r0 + threadIdx.x, &tile[threadIdx.x][0], &tile[threadIdx.x][3]);
    __syncthreads();
    if (v < nv) {
      const int nr = min(kScoreThreads, nc - r0);
      for (int r = 0; r < nr; ++r) {
        const double d2 = residual2(pose, &tile[r][0], &tile[r][3]);
        if (d2 < tau2) {
          ++cnt;
          sum = dadd(sum, d2);
        }
      }
    }
  }
  if (v < nv) {
    inliers[(size_t)p * V + v] = cnt;
    sums[(size_t)p * V + v] = sum;
  }
}

struct Best {
  int cnt;
  double sum;
  int v;     // list position: ascending v is ascending h
};

// the total order of the scores: more inliers, then the smaller sum, then the smaller h
__device__ __forceinline__ bool better(const Best& a, const Best& b) {
  if (a.cnt != b.cnt) return a.cnt > b.cnt;
  if (a.sum != b.sum) return a.sum < b.sum;
  return a.v < b.v;
}

// the best listed hypothesis of each pair, the refit over its inliers, and every output of the pair
template <int N>
__global__ void __launch_bounds__(kFinalizeThreads, 1)
reg_finalize_kernel(Rows rows, const int* __restrict__ pairs, int P, const int* __restrict__ nc_eff,
                    const int* __restrict__ n_val, const int* __restrict__ list, int V, unsigned long long seed,
                    double ratio, double tau2, const int* __restrict__ inliers, const double* __restrict__ sums,
                    double* __restrict__ pose_out, int* __restrict__ n_inliers, int* __restrict__ hypothesis_out,
                    int* __restrict__ n_validated) {
  __shared__ Best warp_best[kFinalizeThreads / 32];
  __shared__ Pose hyp;
  __shared__ float tile[kFinalizeThreads][6];
  __shared__ unsigned char use[kFinalizeThreads];
  __shared__ double centroid[6];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int p = blockIdx.x; p < P; p += gridDim.x) {
    const int nc = nc_eff[p], nv = n_val[p];
    double* out = pose_out + (size_t)p * 16;
    if (nc < N || nv == 0) {
      if (threadIdx.x < 16) out[threadIdx.x] = threadIdx.x % 5 == 0 ? 1.0 : 0.0;
      if (threadIdx.x == 0) {
        n_inliers[p] = 0;
        hypothesis_out[p] = -1;
        n_validated[p] = nv;
      }
      continue;
    }
    Best b{-1, 0.0, 0};
    for (int v = threadIdx.x; v < nv; v += kFinalizeThreads) {
      const Best c{inliers[(size_t)p * V + v], sums[(size_t)p * V + v], v};
      if (better(c, b)) b = c;
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      const Best c{__shfl_xor_sync(0xffffffffu, b.cnt, o), __shfl_xor_sync(0xffffffffu, b.sum, o),
                   __shfl_xor_sync(0xffffffffu, b.v, o)};
      if (better(c, b)) b = c;
    }
    if (lane == 0) warp_best[warp] = b;
    __syncthreads();
    const int src = __ldg(pairs + 2 * p), tgt = __ldg(pairs + 2 * p + 1);
    if (threadIdx.x == 0) {
      b = warp_best[0];
#pragma unroll
      for (int w = 1; w < kFinalizeThreads / 32; ++w)
        if (better(warp_best[w], b)) b = warp_best[w];
      warp_best[0] = b;
      Pose ph;
      hypothesis<N>(rows, p, src, tgt, list[(size_t)p * V + b.v], nc, seed, ratio, tau2, ph);
      hyp = ph;
    }
    __syncthreads();
    b = warp_best[0];
    const int h = list[(size_t)p * V + b.v];
    // refit over the inliers in ascending row order: pass 0 sums the centroids, pass 1 the cross-covariance
    double ss[3] = {0.0, 0.0, 0.0}, st[3] = {0.0, 0.0, 0.0}, H[3][3] = {};
    for (int pass = 0; pass < 2 && b.cnt > 0; ++pass) {
      for (int r0 = 0; r0 < nc; r0 += kFinalizeThreads) {
        const int r = r0 + threadIdx.x;
        if (r < nc) {
          float s[3], t[3];
          rows.load(p, src, tgt, r, s, t);
          use[threadIdx.x] = residual2(hyp, s, t) < tau2;
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            tile[threadIdx.x][i] = s[i];
            tile[threadIdx.x][3 + i] = t[i];
          }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
          const int nr = min(kFinalizeThreads, nc - r0);
          for (int j = 0; j < nr; ++j) {
            if (!use[j]) continue;
            const float* s = &tile[j][0];
            const float* t = &tile[j][3];
            if (pass == 0) {
#pragma unroll
              for (int i = 0; i < 3; ++i) {
                ss[i] = dadd(ss[i], s[i]);
                st[i] = dadd(st[i], t[i]);
              }
            } else {
              double ds[3], dt[3];
#pragma unroll
              for (int i = 0; i < 3; ++i) {
                ds[i] = dsub(s[i], centroid[i]);
                dt[i] = dsub(t[i], centroid[3 + i]);
              }
#pragma unroll
              for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j2 = 0; j2 < 3; ++j2) H[i][j2] = dadd(H[i][j2], dmul(ds[i], dt[j2]));
            }
          }
        }
        __syncthreads();
      }
      if (pass == 0 && threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          centroid[i] = ddiv(ss[i], (double)b.cnt);
          centroid[3 + i] = ddiv(st[i], (double)b.cnt);
        }
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      Pose res = hyp;                    // a best hypothesis without inliers keeps its own pose
      if (b.cnt > 0) pose_from_moments(&centroid[0], &centroid[3], H, res);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) out[i * 4 + j] = res.R[i][j];
        out[i * 4 + 3] = res.t[i];
        out[12 + i] = 0.0;
      }
      out[15] = 1.0;
      n_inliers[p] = b.cnt;
      hypothesis_out[p] = h;
      n_validated[p] = nv;
    }
    __syncthreads();                     // warp_best, hyp and the tiles are reused by the next pair
  }
}

struct Work {
  int* nc_eff;
  int* n_val;
  unsigned* bits;
  int* list;
  int* inliers;
  double* sums;
};

// the sizes the workspace depends on: L, P >= 1, T in [1, 2^24], V in [1, T], P * L * 2 and P * T within int32
bool sizes_ok(int L, int P, int T, int V) {
  if (L < 1 || P < 1 || T < 1 || T > (1 << 24) || V < 1 || V > T) return false;
  return (long long)P * L * 2 <= INT32_MAX && (long long)P * ceil_div(T, 32) * 32 <= INT32_MAX;
}

size_t work_layout(int L, int P, int T, int V, void* base, Work* w_out) {
  if (!sizes_ok(L, P, T, V)) return 0;
  Carver cv(base);
  Work w;
  w.nc_eff = cv.take<int>(P);
  w.n_val = cv.take<int>(P);
  w.bits = cv.take<unsigned>((size_t)P * ceil_div(T, 32));
  w.list = cv.take<int>((size_t)P * V);
  w.inliers = cv.take<int>((size_t)P * V);
  w.sums = cv.take<double>((size_t)P * V);
  if (w_out != nullptr) *w_out = w;
  return cv.off;
}

template <int N>
int run(const Rows& rows, const int* count, int B, const int* n_corr, const int* pairs, int P, int T, int V,
        double tau2, double ratio, unsigned long long seed, double* pose, int* n_inliers, int* hypothesis_out,
        int* n_validated, const Work& w, cudaStream_t stream) {
  const int WT = ceil_div(T, 32);
  const int warp_blocks = ceil_div(P, kWarpsPerCta);
  reg_prepare_kernel<<<warp_blocks, kWarpsPerCta * 32, 0, stream>>>(count, B, rows.k, rows.corr, n_corr, rows.L,
                                                                    pairs, P, w.nc_eff, w.n_val);
  D3F_LAUNCH_CHECK("reg_prepare_kernel");
  long long len = kFirstRound;
  for (int h0 = 0; h0 < T; h0 += (int)len, len *= 2) {
    const int h1 = (int)std::min<long long>(T, h0 + len);
    const int W = ceil_div(h1 - h0, 32);
    const long long lanes = 32ll * W * P;
    const int blocks = (int)std::min<long long>((lanes + kHypThreads - 1) / kHypThreads, 64ll * kNumSMs);
    reg_hypothesis_kernel<N><<<blocks, kHypThreads, 0, stream>>>(rows, pairs, P, w.nc_eff, w.n_val, T, V, h0, W, WT,
                                                                  seed, ratio, tau2, w.bits);
    D3F_LAUNCH_CHECK("reg_hypothesis_kernel");
    reg_select_kernel<<<warp_blocks, kWarpsPerCta * 32, 0, stream>>>(P, N, w.nc_eff, w.n_val, V, h0, h1, WT, w.bits,
                                                                     w.list);
    D3F_LAUNCH_CHECK("reg_select_kernel");
  }
  reg_score_kernel<N><<<P * ceil_div(V, kScoreThreads), kScoreThreads, 0, stream>>>(
      rows, pairs, P, w.nc_eff, w.n_val, w.list, V, seed, ratio, tau2, w.inliers, w.sums);
  D3F_LAUNCH_CHECK("reg_score_kernel");
  reg_finalize_kernel<N><<<std::min(P, 8 * kNumSMs), kFinalizeThreads, 0, stream>>>(
      rows, pairs, P, w.nc_eff, w.n_val, w.list, V, seed, ratio, tau2, w.inliers, w.sums, pose, n_inliers,
      hypothesis_out, n_validated);
  D3F_LAUNCH_CHECK("reg_finalize_kernel");
  return D3F_OK;
}

}  // namespace
}  // namespace d3f

using namespace d3f;

extern "C" size_t d3f_register_pairs_workspace_bytes(int L, int P, int max_iterations, int max_validation) {
  return work_layout(L, P, max_iterations, max_validation, nullptr, nullptr);
}

extern "C" int d3f_register_pairs(const float* points, const int* count, int B, int k, const int* corr,
                                  const int* n_corr, int L, const int* pairs, int P, int ransac_n, int max_iterations,
                                  int max_validation, double distance, double edge_ratio, unsigned long long seed,
                                  double* pose, int* n_inliers, int* hypothesis, int* n_validated, void* workspace,
                                  size_t workspace_bytes, d3f_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  D3F_REQUIRE(B >= 1 && B <= kMaxBatch, D3F_ERR_INVALID, "register_pairs: B=%d must be in [1,%d]", B, kMaxBatch);
  D3F_REQUIRE(k >= 1 && L >= 1 && P >= 1, D3F_ERR_INVALID, "register_pairs: bad shape k=%d L=%d P=%d", k, L, P);
  D3F_REQUIRE(ransac_n >= 3 && ransac_n <= 8, D3F_ERR_INVALID, "register_pairs: ransac_n=%d must be in [3,8]",
              ransac_n);
  D3F_REQUIRE(max_iterations >= 1 && max_iterations <= (1 << 24), D3F_ERR_INVALID,
              "register_pairs: max_iterations=%d must be in [1,2^24]", max_iterations);
  D3F_REQUIRE(max_validation >= 1 && max_validation <= max_iterations, D3F_ERR_INVALID,
              "register_pairs: max_validation=%d must be in [1,max_iterations]", max_validation);
  D3F_REQUIRE(std::isfinite(distance) && distance > 0.0, D3F_ERR_INVALID,
              "register_pairs: distance=%g must be finite and > 0", distance);
  D3F_REQUIRE(edge_ratio > 0.0 && edge_ratio <= 1.0, D3F_ERR_INVALID, "register_pairs: edge_ratio=%g must be in (0,1]",
              edge_ratio);
  D3F_REQUIRE((long long)B * k * 3 <= INT32_MAX && sizes_ok(L, P, max_iterations, max_validation), D3F_ERR_INVALID,
              "register_pairs: B*k*3, P*L*2 or P*max_iterations exceeds int32");
  D3F_REQUIRE(points && count && corr && n_corr && pairs && pose && n_inliers && hypothesis && n_validated &&
                  workspace,
              D3F_ERR_INVALID, "register_pairs: null pointer");
  Work w;
  const size_t need = work_layout(L, P, max_iterations, max_validation, workspace, &w);
  D3F_REQUIRE(need > 0 && workspace_bytes >= need, D3F_ERR_WORKSPACE,
              "register_pairs: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
  const Rows rows{points, corr, k, L};
  const double tau2 = distance * distance;
  const int T = max_iterations, V = max_validation;
  switch (ransac_n) {
    case 3: return run<3>(rows, count, B, n_corr, pairs, P, T, V, tau2, edge_ratio, seed, pose, n_inliers, hypothesis,
                          n_validated, w, stream);
    case 4: return run<4>(rows, count, B, n_corr, pairs, P, T, V, tau2, edge_ratio, seed, pose, n_inliers, hypothesis,
                          n_validated, w, stream);
    case 5: return run<5>(rows, count, B, n_corr, pairs, P, T, V, tau2, edge_ratio, seed, pose, n_inliers, hypothesis,
                          n_validated, w, stream);
    case 6: return run<6>(rows, count, B, n_corr, pairs, P, T, V, tau2, edge_ratio, seed, pose, n_inliers, hypothesis,
                          n_validated, w, stream);
    case 7: return run<7>(rows, count, B, n_corr, pairs, P, T, V, tau2, edge_ratio, seed, pose, n_inliers, hypothesis,
                          n_validated, w, stream);
    default: return run<8>(rows, count, B, n_corr, pairs, P, T, V, tau2, edge_ratio, seed, pose, n_inliers,
                           hypothesis, n_validated, w, stream);
  }
}

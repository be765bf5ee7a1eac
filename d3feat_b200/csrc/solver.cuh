// The fp64 rigid-pose solver shared by RANSAC (registration.cu) and ICP (icp.cu): every step is one correctly rounded
// operation (__dadd_rn, __dsub_rn, __dmul_rn, __ddiv_rn, __dsqrt_rn), so nvcc never contracts a multiply-add and the
// results equal the numpy restatement oracle/register_np.py bit for bit.
#pragma once
#include "common.cuh"

namespace d3f {

namespace {

constexpr int kSweeps = 6;               // cyclic Jacobi sweeps: the 4x4 matrix reaches fp64 precision in five

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double dsqrt(double a) { return __dsqrt_rn(a); }

struct Pose {
  double R[3][3];
  double t[3];
};

// d^2 = |R s + t - t'|^2: e_a = (((R_a0 s_0 + R_a1 s_1) + R_a2 s_2) + t_a) - t'_a, d^2 = (e_0^2 + e_1^2) + e_2^2
template <typename F>
__device__ __forceinline__ double residual2(const Pose& P, const F s[3], const F t[3]) {
  double e[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    e[i] = dsub(dadd(dadd(dadd(dmul(P.R[i][0], s[0]), dmul(P.R[i][1], s[1])), dmul(P.R[i][2], s[2])), P.t[i]), t[i]);
  return dadd(dadd(dmul(e[0], e[0]), dmul(e[1], e[1])), dmul(e[2], e[2]));
}

// Horn: N from the centred cross-covariance H, cyclic Jacobi, the quaternion of the largest eigenvalue, R and t
__device__ void pose_from_moments(const double cs[3], const double ct[3], const double H[3][3], Pose& out) {
  const double Sxx = H[0][0], Sxy = H[0][1], Sxz = H[0][2], Syx = H[1][0], Syy = H[1][1], Syz = H[1][2];
  const double Szx = H[2][0], Szy = H[2][1], Szz = H[2][2];
  double a[4][4], v[4][4];
  a[0][0] = dadd(dadd(Sxx, Syy), Szz);
  a[0][1] = dsub(Syz, Szy);
  a[0][2] = dsub(Szx, Sxz);
  a[0][3] = dsub(Sxy, Syx);
  a[1][1] = dsub(dsub(Sxx, Syy), Szz);
  a[1][2] = dadd(Sxy, Syx);
  a[1][3] = dadd(Szx, Sxz);
  a[2][2] = dsub(dsub(Syy, Sxx), Szz);
  a[2][3] = dadd(Syz, Szy);
  a[3][3] = dsub(dsub(Szz, Sxx), Syy);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int j = 0; j < i; ++j) a[i][j] = a[j][i];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[i][j] = i == j ? 1.0 : 0.0;
  }
#pragma unroll 1
  for (int sweep = 0; sweep < kSweeps; ++sweep) {
#pragma unroll
    for (int pv = 0; pv < 6; ++pv) {     // pivots (0,1) (0,2) (0,3) (1,2) (1,3) (2,3)
      const int p = pv < 3 ? 0 : (pv < 5 ? 1 : 2);
      const int q = pv < 3 ? pv + 1 : (pv < 5 ? pv - 1 : 3);
      const double apq = a[p][q];
      if (apq != 0.0) {                  // the exact-zero skip rule
        const double theta = ddiv(dsub(a[q][q], a[p][p]), dmul(2.0, apq));
        const double t = ddiv(theta >= 0.0 ? 1.0 : -1.0, dadd(fabs(theta), dsqrt(dadd(dmul(theta, theta), 1.0))));
        const double c = ddiv(1.0, dsqrt(dadd(dmul(t, t), 1.0)));
        const double s = dmul(t, c);
        const double tap = dmul(t, apq);
        a[p][p] = dsub(a[p][p], tap);
        a[q][q] = dadd(a[q][q], tap);
        a[p][q] = a[q][p] = 0.0;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          if (r == p || r == q) continue;
          const double arp = a[r][p], arq = a[r][q];
          a[r][p] = a[p][r] = dsub(dmul(c, arp), dmul(s, arq));
          a[r][q] = a[q][r] = dadd(dmul(s, arp), dmul(c, arq));
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const double vrp = v[r][p], vrq = v[r][q];
          v[r][p] = dsub(dmul(c, vrp), dmul(s, vrq));
          v[r][q] = dadd(dmul(s, vrp), dmul(c, vrq));
        }
      }
    }
  }
  double q[4], dbest = a[0][0];
#pragma unroll
  for (int r = 0; r < 4; ++r) q[r] = v[r][0];
#pragma unroll
  for (int i = 1; i < 4; ++i) {          // largest diagonal entry, ties to the lowest index
    if (a[i][i] > dbest) {
      dbest = a[i][i];
#pragma unroll
      for (int r = 0; r < 4; ++r) q[r] = v[r][i];
    }
  }
  const double nrm = dsqrt(dadd(dadd(dadd(dmul(q[0], q[0]), dmul(q[1], q[1])), dmul(q[2], q[2])), dmul(q[3], q[3])));
  const double w = ddiv(q[0], nrm), x = ddiv(q[1], nrm), y = ddiv(q[2], nrm), z = ddiv(q[3], nrm);
  const double ww = dmul(w, w), xx = dmul(x, x), yy = dmul(y, y), zz = dmul(z, z);
  const double xy = dmul(x, y), xz = dmul(x, z), yz = dmul(y, z), wx = dmul(w, x), wy = dmul(w, y), wz = dmul(w, z);
  out.R[0][0] = dsub(dsub(dadd(ww, xx), yy), zz);
  out.R[0][1] = dmul(2.0, dsub(xy, wz));
  out.R[0][2] = dmul(2.0, dadd(xz, wy));
  out.R[1][0] = dmul(2.0, dadd(xy, wz));
  out.R[1][1] = dsub(dadd(dsub(ww, xx), yy), zz);
  out.R[1][2] = dmul(2.0, dsub(yz, wx));
  out.R[2][0] = dmul(2.0, dsub(xz, wy));
  out.R[2][1] = dmul(2.0, dadd(yz, wx));
  out.R[2][2] = dadd(dsub(dsub(ww, xx), yy), zz);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    out.t[i] = dsub(ct[i], dadd(dadd(dmul(out.R[i][0], cs[0]), dmul(out.R[i][1], cs[1])), dmul(out.R[i][2], cs[2])));
}

}  // namespace

}  // namespace d3f

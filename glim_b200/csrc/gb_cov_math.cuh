// gb_cov_math.cuh -- covariance and normal of one point (CloudCovarianceEstimation::estimate with PLANE regularisation,
// cloud_covariance_estimation.cpp:80-102, :181-196), the arithmetic of k_covariances_planes.  Like
// gb_vgicp_math.cuh it holds nothing that only exists on the device, so the SAME TEXT compiles for the host:
// tests/cpp/cov_math_host.cpp builds it with g++ and tests/test_cov_degenerate.py checks it bit for bit against the oracle.
//
// Every fp64 multiply, add and subtract is written as an explicit round-to-nearest operation (__dmul_rn, __dadd_rn,
// __dsub_rn) in the oracle's association order, so nvcc cannot contract it into an FMA.  The oracle and the reference are
// built uncontracted, and on a neighbourhood whose smallest eigenvector is poorly defined (duplicated, collinear or isotropic
// points, a small spread far from the origin) the eigen solver scales the rounding noise of the covariance up to O(1): a
// contracted build then returns a different plane.  What remains between device and oracle are the ulps of atan2, cos and sin.
#pragma once
#ifdef __CUDACC__
#define GB_CHD __device__ __forceinline__
#else
#include <math.h>
#define GB_CHD static inline
struct double4 { double x, y, z, w; };
// the host build is compiled with -ffp-contract=off: a plain operator is one rounded operation
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
#endif

namespace {

GB_CHD void cross3(const double* a, const double* b, double* c) {
  c[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  c[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  c[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}
// (a0 a0 + a1 a1) + a2 a2
GB_CHD double dot3(const double* a, const double* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

// unit vector of the kernel of a symmetric rank <= 2 matrix m (row-major): cross products of the column with the largest
// diagonal magnitude (returned in rep) with the two others, the longer one normalised
GB_CHD void extract_kernel(const double* m, double* res, double* rep) {
  int i0 = 0;
  double best = fabs(m[0]);
  if (fabs(m[4]) > best) { best = fabs(m[4]); i0 = 1; }
  if (fabs(m[8]) > best) { best = fabs(m[8]); i0 = 2; }
  double c1v[3], c2v[3];
  const int i1 = (i0 + 1) % 3, i2 = (i0 + 2) % 3;
  for (int r = 0; r < 3; r++) { rep[r] = m[r * 3 + i0]; c1v[r] = m[r * 3 + i1]; c2v[r] = m[r * 3 + i2]; }
  double c0[3], c1[3];
  cross3(rep, c1v, c0);
  cross3(rep, c2v, c1);
  const double n0 = dot3(c0, c0);
  const double n1 = dot3(c1, c1);
  if (n0 > n1) { const double s = 1.0 / sqrt(n0); for (int k = 0; k < 3; k++) res[k] = __dmul_rn(c0[k], s); }
  else if (n1 > 0.0) { const double s = 1.0 / sqrt(n1); for (int k = 0; k < 3; k++) res[k] = __dmul_rn(c1[k], s); }
  else { res[0] = 1; res[1] = 0; res[2] = 0; }
}

// closed-form symmetric 3x3 eigen decomposition (the published algorithm of the oracle's go_eigen_sym3_direct / Eigen's
// computeDirect): shift by trace / 3, scale by the largest |entry|, trigonometric roots of the characteristic polynomial,
// eigenvectors from cross products of rows of (A - lambda I).  evals ascending, V[r*3+k] = k-th eigenvector.
GB_CHD void eigen_sym3_direct(const double* A, double* evals, double* V) {
  const double shift = __dadd_rn(__dadd_rn(A[0], A[4]), A[8]) / 3.0;
  double m[9];
  for (int k = 0; k < 9; k++) m[k] = A[k];
  m[0] = __dsub_rn(m[0], shift); m[4] = __dsub_rn(m[4], shift); m[8] = __dsub_rn(m[8], shift);
  double scale = 0.0;
  for (int k = 0; k < 9; k++) scale = fmax(scale, fabs(m[k]));
  if (scale > 0.0) for (int k = 0; k < 9; k++) m[k] /= scale;
  const double m00 = m[0], m11 = m[4], m22 = m[8], m10 = m[3], m20 = m[6], m21 = m[7];
  // c0 = m00 m11 m22 + 2 m10 m20 m21 - m00 m21 m21 - m11 m20 m20 - m22 m10 m10, left to right
  double c0 = __dadd_rn(__dmul_rn(__dmul_rn(m00, m11), m22), __dmul_rn(__dmul_rn(__dmul_rn(2.0, m10), m20), m21));
  c0 = __dsub_rn(c0, __dmul_rn(__dmul_rn(m00, m21), m21));
  c0 = __dsub_rn(c0, __dmul_rn(__dmul_rn(m11, m20), m20));
  c0 = __dsub_rn(c0, __dmul_rn(__dmul_rn(m22, m10), m10));
  // c1 = m00 m11 - m10 m10 + m00 m22 - m20 m20 + m11 m22 - m21 m21, left to right
  double c1 = __dsub_rn(__dmul_rn(m00, m11), __dmul_rn(m10, m10));
  c1 = __dadd_rn(c1, __dmul_rn(m00, m22));
  c1 = __dsub_rn(c1, __dmul_rn(m20, m20));
  c1 = __dadd_rn(c1, __dmul_rn(m11, m22));
  c1 = __dsub_rn(c1, __dmul_rn(m21, m21));
  const double c2 = __dadd_rn(__dadd_rn(m00, m11), m22);
  const double c2_3 = c2 / 3.0;
  double a_3 = __dsub_rn(__dmul_rn(c2, c2_3), c1) / 3.0;
  if (a_3 < 0.0) a_3 = 0.0;
  const double half_b = __dmul_rn(0.5, __dadd_rn(c0, __dmul_rn(c2_3, __dsub_rn(__dmul_rn(__dmul_rn(2.0, c2_3), c2_3), c1))));
  double qq = __dsub_rn(__dmul_rn(__dmul_rn(a_3, a_3), a_3), __dmul_rn(half_b, half_b));
  if (qq < 0.0) qq = 0.0;
  const double rho = sqrt(a_3);
  const double theta = atan2(sqrt(qq), half_b) / 3.0;
  const double ct = cos(theta), st = sin(theta);
  const double s3 = 1.7320508075688772935;
  double ev[3];
  ev[0] = __dsub_rn(c2_3, __dmul_rn(rho, __dadd_rn(ct, __dmul_rn(s3, st))));
  ev[1] = __dsub_rn(c2_3, __dmul_rn(rho, __dsub_rn(ct, __dmul_rn(s3, st))));
  ev[2] = __dadd_rn(c2_3, __dmul_rn(__dmul_rn(2.0, rho), ct));
  const double eps = 2.220446049250313e-16;
  if (__dsub_rn(ev[2], ev[0]) <= eps) {
    for (int k = 0; k < 9; k++) V[k] = 0.0;
    V[0] = V[4] = V[8] = 1.0;
  } else {
    double d0 = __dsub_rn(ev[2], ev[1]), d1 = __dsub_rn(ev[1], ev[0]);
    int k = 0, l = 2;
    if (d0 > d1) { const double t = d0; d0 = d1; d1 = t; k = 2; l = 0; }
    double tmp[9], vk[3], vl[3], rep[3];
    for (int e = 0; e < 9; e++) tmp[e] = m[e];
    tmp[0] = __dsub_rn(tmp[0], ev[k]); tmp[4] = __dsub_rn(tmp[4], ev[k]); tmp[8] = __dsub_rn(tmp[8], ev[k]);
    extract_kernel(tmp, vk, rep);
    if (d0 <= __dmul_rn(__dmul_rn(2.0, eps), d1)) {
      const double dp = dot3(vk, rep);
      for (int r = 0; r < 3; r++) vl[r] = __dsub_rn(rep[r], __dmul_rn(dp, vk[r]));
      const double nl = sqrt(dot3(vl, vl));
      if (nl > 0) for (int r = 0; r < 3; r++) vl[r] /= nl;
    } else {
      double dummy[3];
      for (int e = 0; e < 9; e++) tmp[e] = m[e];
      tmp[0] = __dsub_rn(tmp[0], ev[l]); tmp[4] = __dsub_rn(tmp[4], ev[l]); tmp[8] = __dsub_rn(tmp[8], ev[l]);
      extract_kernel(tmp, vl, dummy);
    }
    double v0[3], v1[3], v2[3];
    for (int r = 0; r < 3; r++) { v0[r] = (k == 0) ? vk[r] : vl[r]; v2[r] = (k == 0) ? vl[r] : vk[r]; }
    cross3(v2, v0, v1);
    const double n1 = sqrt(dot3(v1, v1));
    if (n1 > 0) for (int r = 0; r < 3; r++) v1[r] /= n1;
    for (int r = 0; r < 3; r++) { V[r * 3 + 0] = v0[r]; V[r * 3 + 1] = v1[r]; V[r * 3 + 2] = v2[r]; }
  }
  for (int k = 0; k < 3; k++) evals[k] = __dadd_rn(__dmul_rn(ev[k], scale), shift);
}

// calc_cov (cloud_covariance_estimation.cpp:80-102) of point i from the first k of its kc neighbours: the regularised
// covariance C (row-major 3x3) and the normal, flipped to face the origin; returns the point.
// The reference materialises pt_cross = p p^T per point (:58-63) and sums those; here the same rounded products are formed
// from the gathered neighbour points and summed in the same order.
GB_CHD double4 plane_covariance(int i, const double4* __restrict__ pts, const int* __restrict__ neighbors, int kc, int k, double (&C)[9], double (&nrm)[3]) {
  double S[3] = {0, 0, 0};
  double X[9];
  for (int e = 0; e < 9; e++) X[e] = 0.0;
  const size_t begin = (size_t)kc * (size_t)i;
  for (int j = 0; j < k; j++) {
    const double4 q = pts[neighbors[begin + j]];
    const double p[3] = {q.x, q.y, q.z};
    for (int r = 0; r < 3; r++) S[r] = __dadd_rn(S[r], p[r]);
    for (int c = 0; c < 3; c++)
      for (int r = 0; r < 3; r++) X[c * 3 + r] = __dadd_rn(X[c * 3 + r], __dmul_rn(p[r], p[c]));
  }
  double mean[3], A[9];
  for (int r = 0; r < 3; r++) mean[r] = S[r] / k;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) A[r * 3 + c] = __dsub_rn(X[c * 3 + r], __dmul_rn(mean[r], S[c])) / k;
  double evals[3], V[9];
  eigen_sym3_direct(A, evals, V);
  const double values[3] = {1e-3, 1.0, 1.0};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      double s = 0;
      for (int e = 0; e < 3; e++) s = __dadd_rn(s, __dmul_rn(__dmul_rn(V[r * 3 + e], values[e]), V[c * 3 + e]));
      C[r * 3 + c] = s;
    }
  const double4 p = pts[i];
  double nx = V[0], ny = V[3], nz = V[6];
  // p . n with the homogeneous term p.w * n.w (n.w = 0), as the reference evaluates it on Vector4d
  const double pn = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p.x, nx), __dmul_rn(p.y, ny)), __dmul_rn(p.z, nz)), __dmul_rn(p.w, 0.0));
  if (pn > 0.0) { nx = -nx; ny = -ny; nz = -nz; }
  nrm[0] = nx; nrm[1] = ny; nrm[2] = nz;
  return p;
}

// estimate_normals of one stored point (gb_cloud_estimate_normals, k_cloud_normals; the rule is written once in
// include/glim_b200.h): the unit eigenvector of the smallest eigenvalue of its fp32 covariance (c00 c01 c02 c11 c12 c22) widened
// to fp64, turned away from p when (px nx + py ny) + pz nz > 0, stored as fp32 in n.  Zero for a point whose position or
// covariance is not finite.
GB_CHD void covariance_normal(float px, float py, float pz, float c00, float c01, float c02, float c11, float c12, float c22, float (&n)[3]) {
  const double p[3] = {px, py, pz};
  const double A[9] = {c00, c01, c02, c01, c11, c12, c02, c12, c22};
  bool finite = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
  for (int k = 0; k < 9; k++) finite = finite && isfinite(A[k]);
  if (!finite) { n[0] = n[1] = n[2] = 0.f; return; }
  double evals[3], V[9];
  eigen_sym3_direct(A, evals, V);
  double v[3] = {V[0], V[3], V[6]};
  if (dot3(p, v) > 0.0) { v[0] = -v[0]; v[1] = -v[1]; v[2] = -v[2]; }
  n[0] = (float)v[0]; n[1] = (float)v[1]; n[2] = (float)v[2];
}

}  // namespace

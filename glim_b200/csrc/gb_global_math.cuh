// gb_global_math.cuh -- the per-pair and per-hypothesis arithmetic of global registration (gb_kernels_global.cu): FPFH pair
// features and their bins, the RANSAC sample draw, and the 6-DoF (Horn) and 4-DoF pose estimators.  Like gb_cov_math.cuh it
// holds nothing that only exists on the device, so the SAME TEXT compiles for the host: tests/cpp/global_math_host.cpp builds
// it with g++ -ffp-contract=off and tests/test_global_host.py checks it against the numpy restatement (tests/global_oracle.py).
// The rules are written once, in include/glim_b200.h (gb_cloud_estimate_fpfh, gb_ransac_align).
//
// Every fp64 multiply, add and subtract that could be contracted is an explicit round-to-nearest operation, so the device and
// the host build agree bit for bit; division and sqrt are correctly rounded on both.  What remains between them is atan2 (the
// pair feature f1 and the 4-DoF yaw), a few ulps apart: a bin can differ only for a feature within that distance of its edge.
#pragma once
#include "gb_grid_math.cuh"  // GB_HD, gb_coord, gb_lookup, rg_hash, PoseF, the fp32 intrinsics' host shims
#include "gb_cov_math.cuh"   // cross3, dot3, the fp64 intrinsics' host shims

namespace {

constexpr int kFpfhDim = 33;     // 3 features x 11 bins
constexpr int kFpfhBins = 11;
// A RANSAC sample is invalid when the doubled area |(x1 - x0) x (x2 - x0)| of its source or of its target triangle is below
// this (m^2), or not finite: three points that (nearly) coincide or lie on a line fix no pose.
constexpr double kRansacMinArea2 = 1e-3;

// The PCL / Open3D pair feature of point s (position ps, normal ns) and neighbour t: d = pt - ps; zero |d| gives (0, 0, 0).
// The roles swap when |ns . d| < |nt . d| (PCL's acos(|ns . d / |d||) > acos(|nt . d / |d||), compared on the cosines so that
// it is exact): then ns <-> nt, d -> -d.  f3 = ns . d / |d|, v = d x ns (zero |v| gives (0, 0, 0)), v /= |v|, w = ns x v,
// f2 = v . nt, f1 = atan2(w . nt, ns . nt).  Returns d . d (the squared distance of the pair, fp64).
GB_CHD double fpfh_pair(const double* ps, const double* ns_in, const double* pt, const double* nt_in, double* f) {
  double d[3] = {__dsub_rn(pt[0], ps[0]), __dsub_rn(pt[1], ps[1]), __dsub_rn(pt[2], ps[2])};
  const double dd = dot3(d, d);
  f[0] = 0.0; f[1] = 0.0; f[2] = 0.0;
  if (dd == 0.0) return dd;
  const double len = sqrt(dd);
  const double a1 = dot3(ns_in, d) / len, a2 = dot3(nt_in, d) / len;
  const double* ns = ns_in;
  const double* nt = nt_in;
  double f3 = a1;
  if (fabs(a1) < fabs(a2)) {
    ns = nt_in; nt = ns_in;
    d[0] = -d[0]; d[1] = -d[1]; d[2] = -d[2];
    f3 = -a2;
  }
  double v[3], w[3];
  cross3(d, ns, v);
  const double vv = dot3(v, v);
  if (vv == 0.0) return dd;
  const double vn = sqrt(vv);
  v[0] = v[0] / vn; v[1] = v[1] / vn; v[2] = v[2] / vn;
  cross3(ns, v, w);
  f[0] = atan2(dot3(w, nt), dot3(ns, nt));
  f[1] = dot3(v, nt);
  f[2] = f3;
  return dd;
}

// The bin of a scaled feature t in [0, 11): floor(t) clamped to [0, 10]; NaN goes to 0.
GB_CHD int fpfh_bin_of(double t) {
  if (!(t >= 1.0)) return 0;
  if (t >= 10.0) return 10;
  return (int)t;
}
// The three bins of a pair (Open3D's ComputeSPFHFeature): f1 over [-pi, pi], f2 and f3 over [-1, 1], 11 bins each; the
// returned indices are into the 33-bin histogram.
GB_CHD void fpfh_bins(const double* f, int* b) {
  const double two_pi = 6.283185307179586;
  b[0] = fpfh_bin_of(__dmul_rn(11.0, __dadd_rn(f[0], 3.141592653589793)) / two_pi);
  b[1] = kFpfhBins + fpfh_bin_of(__dmul_rn(__dmul_rn(11.0, __dadd_rn(f[1], 1.0)), 0.5));
  b[2] = 2 * kFpfhBins + fpfh_bin_of(__dmul_rn(__dmul_rn(11.0, __dadd_rn(f[2], 1.0)), 0.5));
}

// The source indices of hypothesis h: s_j = rg_hash(seed, 3 h + j) mod ns, j = 0, 1, 2.
GB_HD void ransac_sample(unsigned long long seed, int h, int ns, int* s) {
  for (int j = 0; j < 3; j++) s[j] = (int)(rg_hash(seed, 3u * (unsigned)h + (unsigned)j) % (unsigned long long)ns);
}

// the doubled area of triangle x (3 points, row-major)
GB_CHD double tri_area2(const double* x) {
  const double e1[3] = {__dsub_rn(x[3], x[0]), __dsub_rn(x[4], x[1]), __dsub_rn(x[5], x[2])};
  const double e2[3] = {__dsub_rn(x[6], x[0]), __dsub_rn(x[7], x[1]), __dsub_rn(x[8], x[2])};
  double c[3];
  cross3(e1, e2, c);
  return sqrt(dot3(c, c));
}

// centroids ((x0 + x1) + x2) / 3 and the centred points
GB_CHD void tri_centre(const double* x, double* c, double* xc) {
  for (int k = 0; k < 3; k++) c[k] = __dadd_rn(__dadd_rn(x[k], x[3 + k]), x[6 + k]) / 3.0;
  for (int i = 0; i < 3; i++)
    for (int k = 0; k < 3; k++) xc[3 * i + k] = __dsub_rn(x[3 * i + k], c[k]);
}

// one Jacobi rotation of the symmetric 4x4 A (row-major) in the plane (p, q), accumulated into V's columns
GB_CHD void jacobi_rotate(double* A, double* V, int p, int q) {
  const double apq = A[4 * p + q];
  if (apq == 0.0) return;
  const double theta = __dsub_rn(A[4 * q + q], A[4 * p + p]) / __dmul_rn(2.0, apq);
  const double t = (theta >= 0.0 ? 1.0 : -1.0) / __dadd_rn(fabs(theta), sqrt(__dadd_rn(__dmul_rn(theta, theta), 1.0)));
  const double c = 1.0 / sqrt(__dadd_rn(__dmul_rn(t, t), 1.0));
  const double s = __dmul_rn(t, c);
  for (int k = 0; k < 4; k++) {
    const double akp = A[4 * k + p], akq = A[4 * k + q];
    A[4 * k + p] = __dsub_rn(__dmul_rn(c, akp), __dmul_rn(s, akq));
    A[4 * k + q] = __dadd_rn(__dmul_rn(s, akp), __dmul_rn(c, akq));
  }
  for (int k = 0; k < 4; k++) {
    const double apk = A[4 * p + k], aqk = A[4 * q + k];
    A[4 * p + k] = __dsub_rn(__dmul_rn(c, apk), __dmul_rn(s, aqk));
    A[4 * q + k] = __dadd_rn(__dmul_rn(s, apk), __dmul_rn(c, aqk));
  }
  for (int k = 0; k < 4; k++) {
    const double vkp = V[4 * k + p], vkq = V[4 * k + q];
    V[4 * k + p] = __dsub_rn(__dmul_rn(c, vkp), __dmul_rn(s, vkq));
    V[4 * k + q] = __dadd_rn(__dmul_rn(s, vkp), __dmul_rn(c, vkq));
  }
}
constexpr int kJacobiSweeps = 8;  // fixed: a 4x4 converges to fp64 rounding in fewer

// T (16, column-major) with target ~ R source + t from three pairs (a: source, b: target; 3 x 3 row-major each).  dof 6:
// Horn's closed form -- the unit quaternion (w, x, y, z) is the eigenvector of the largest eigenvalue of Horn's 4x4 N built
// from S = sum_i a'_i b'_i^T (centred points), found by kJacobiSweeps cyclic Jacobi sweeps over the pairs (0,1) (0,2) (0,3)
// (1,2) (1,3) (2,3) (the largest diagonal entry after the sweeps, ties to the lower index).  dof 4: yaw = atan2(sum a'_x b'_y -
// a'_y b'_x, sum a'_x b'_x + a'_y b'_y), R = Rz(yaw).  Both: t = b_centroid - R a_centroid.  Returns false (T untouched) for an
// invalid sample (tri_area2 of either triangle below kRansacMinArea2 or not finite).
GB_CHD bool ransac_pose(const double* a, const double* b, int dof, double* T) {
  if (!(tri_area2(a) >= kRansacMinArea2) || !(tri_area2(b) >= kRansacMinArea2)) return false;
  double ca[3], cb[3], ac[9], bc[9], R[9];
  tri_centre(a, ca, ac);
  tri_centre(b, cb, bc);
  if (dof == 4) {
    double sn = 0.0, cs = 0.0;
    for (int i = 0; i < 3; i++) {
      const double* p = ac + 3 * i;
      const double* q = bc + 3 * i;
      sn = __dadd_rn(sn, __dsub_rn(__dmul_rn(p[0], q[1]), __dmul_rn(p[1], q[0])));
      cs = __dadd_rn(cs, __dadd_rn(__dmul_rn(p[0], q[0]), __dmul_rn(p[1], q[1])));
    }
    const double yaw = atan2(sn, cs), c = cos(yaw), s = sin(yaw);
    R[0] = c; R[1] = -s; R[2] = 0.0;
    R[3] = s; R[4] = c;  R[5] = 0.0;
    R[6] = 0.0; R[7] = 0.0; R[8] = 1.0;
  } else {
    double S[9];  // S[3 r + c] = sum_i a'_i[r] b'_i[c]
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++)
        S[3 * r + c] = __dadd_rn(__dadd_rn(__dmul_rn(ac[r], bc[c]), __dmul_rn(ac[3 + r], bc[3 + c])), __dmul_rn(ac[6 + r], bc[6 + c]));
    const double sxx = S[0], sxy = S[1], sxz = S[2], syx = S[3], syy = S[4], syz = S[5], szx = S[6], szy = S[7], szz = S[8];
    double N[16] = {
        __dadd_rn(__dadd_rn(sxx, syy), szz), __dsub_rn(syz, szy), __dsub_rn(szx, sxz), __dsub_rn(sxy, syx),
        __dsub_rn(syz, szy), __dsub_rn(__dsub_rn(sxx, syy), szz), __dadd_rn(sxy, syx), __dadd_rn(szx, sxz),
        __dsub_rn(szx, sxz), __dadd_rn(sxy, syx), __dsub_rn(__dsub_rn(syy, sxx), szz), __dadd_rn(syz, szy),
        __dsub_rn(sxy, syx), __dadd_rn(szx, sxz), __dadd_rn(syz, szy), __dsub_rn(__dsub_rn(szz, sxx), syy)};
    double V[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    for (int sweep = 0; sweep < kJacobiSweeps; sweep++)
      for (int p = 0; p < 3; p++)
        for (int q = p + 1; q < 4; q++) jacobi_rotate(N, V, p, q);
    int k = 0;
    for (int j = 1; j < 4; j++)
      if (N[5 * j] > N[5 * k]) k = j;
    double w = V[k], x = V[4 + k], y = V[8 + k], z = V[12 + k];
    const double qn = sqrt(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(w, w), __dmul_rn(x, x)), __dmul_rn(y, y)), __dmul_rn(z, z)));
    w = w / qn; x = x / qn; y = y / qn; z = z / qn;
    R[0] = __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(__dmul_rn(y, y), __dmul_rn(z, z))));
    R[1] = __dmul_rn(2.0, __dsub_rn(__dmul_rn(x, y), __dmul_rn(w, z)));
    R[2] = __dmul_rn(2.0, __dadd_rn(__dmul_rn(x, z), __dmul_rn(w, y)));
    R[3] = __dmul_rn(2.0, __dadd_rn(__dmul_rn(x, y), __dmul_rn(w, z)));
    R[4] = __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(__dmul_rn(x, x), __dmul_rn(z, z))));
    R[5] = __dmul_rn(2.0, __dsub_rn(__dmul_rn(y, z), __dmul_rn(w, x)));
    R[6] = __dmul_rn(2.0, __dsub_rn(__dmul_rn(x, z), __dmul_rn(w, y)));
    R[7] = __dmul_rn(2.0, __dadd_rn(__dmul_rn(y, z), __dmul_rn(w, x)));
    R[8] = __dsub_rn(1.0, __dmul_rn(2.0, __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y))));
  }
  for (int r = 0; r < 3; r++) {
    const double ra = __dadd_rn(__dadd_rn(__dmul_rn(R[3 * r], ca[0]), __dmul_rn(R[3 * r + 1], ca[1])), __dmul_rn(R[3 * r + 2], ca[2]));
    for (int c = 0; c < 3; c++) T[4 * c + r] = R[3 * r + c];
    T[12 + r] = __dsub_rn(cb[r], ra);
    T[3 + 4 * r] = 0.0;
  }
  T[15] = 1.0;
  return true;
}

// The RANSAC inlier test of source point (ax, ay, az) under P (the fp32 cast of the hypothesis): q = R a + t uncontracted,
// ((r0 ax + r1 ay) + r2 az) + t per row; an inlier iff q is finite and its cell (gb_coord at inv) holds a target point.
GB_HD bool ransac_inlier(const PoseF& P, float ax, float ay, float az, const int4* __restrict__ buckets, uint32_t mask, int max_scan, float inv) {
  const float qx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P.r00, ax), __fmul_rn(P.r01, ay)), __fmul_rn(P.r02, az)), P.tx);
  const float qy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P.r10, ax), __fmul_rn(P.r11, ay)), __fmul_rn(P.r12, az)), P.ty);
  const float qz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P.r20, ax), __fmul_rn(P.r21, ay)), __fmul_rn(P.r22, az)), P.tz);
  if (!(isfinite(qx) && isfinite(qy) && isfinite(qz))) return false;
  return gb_lookup(buckets, mask, max_scan, gb_coord(qx, inv), gb_coord(qy, inv), gb_coord(qz, inv)) >= 0;
}

}  // namespace

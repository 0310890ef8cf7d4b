// gb_editor_math.cuh -- the per-point rules of the map editor's selection tools (gb_select_gizmo, gb_kernels_plane.cu;
// gb_select_radius, gb_kernels_segment.cu), kept free of anything that only exists on the device so that the SAME TEXT also
// compiles for the host: tests/cpp/editor_math_host.cpp builds it with g++ -ffp-contract=off and tests/test_editor_host.py
// checks it against the numpy restatement of the rules (tests/editor_oracle.py).  The rules are written once, in
// include/glim_b200.h.
#pragma once
#include "gb_mincut_math.cuh"  // mc_d2, and through gb_segment_math.cuh GB_HD and the fp64 intrinsics' host shims

namespace {

// M = A B of two column-major 4x4 affine matrices whose bottom rows are (0, 0, 0, 1): M_rc = (A_r0 B_0c + A_r1 B_1c) + A_r2 B_2c
// for c < 3, and M_r3 = ((A_r0 B_03 + A_r1 B_13) + A_r2 B_23) + A_r3, each operation rounded (a host function: the library's
// host code is built for x86-64 without FMA, the host test with -ffp-contract=off); the bottom row is (0, 0, 0, 1).
inline void ed_compose(const double* A, const double* B, double* M) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 4; c++) {
      const double s = (A[r] * B[4 * c] + A[4 + r] * B[4 * c + 1]) + A[8 + r] * B[4 * c + 2];
      M[4 * c + r] = c < 3 ? s : s + A[12 + r];
    }
  }
  for (int c = 0; c < 4; c++) M[4 * c + 3] = c < 3 ? 0.0 : 1.0;
}

// The gizmo's box in its local frame: -0.5 < q_r < 0.5 on every axis, strict; a NaN is never inside.
GB_HD bool ed_in_box(const double* q) {
  for (int a = 0; a < 3; a++)
    if (!(q[a] > -0.5 && q[a] < 0.5)) return false;
  return true;
}

// The sphere about the origin: (q_x^2 + q_y^2) + q_z^2 < r2, each operation rounded; a NaN is never inside.  The gizmo's unit
// sphere is r2 = 1, the plane patch's sphere r2 = radius^2.
GB_HD bool ed_in_sphere(const double* q, double r2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])) < r2;
}

// The radius tools' flags of a stored point p about the picked point c: d2 = mc_d2 of p widened to fp64; bit 0 (inside):
// finite and d2 < inner2, bit 1 (participant): finite and d2 < outer2.
GB_HD int ed_radius_flags(float px, float py, float pz, const double* c, double inner2, double outer2) {
  if (!(isfinite(px) && isfinite(py) && isfinite(pz))) return 0;
  const double d2 = mc_d2(px, py, pz, c[0], c[1], c[2]);
  return (d2 < inner2 ? 1 : 0) | (d2 < outer2 ? 2 : 0);
}

// The outlier threshold over m participants from s = sum d and s2 = sum d^2: mean = s / m, var = s2 / m - mean^2 (population,
// clamped at 0), mean + stddev_thresh * sqrt(var), each operation rounded.
GB_HD double ed_outlier_threshold(double s, double s2, int m, double stddev_thresh) {
  const double mean = s / (double)m;
  const double var = __dsub_rn(s2 / (double)m, __dmul_rn(mean, mean));
  return __dadd_rn(mean, __dmul_rn(stddev_thresh, sqrt(var > 0.0 ? var : 0.0)));
}

// A participant is selected as an outlier iff it lies inside the radius and is not an inlier: !(d < thresh).
GB_HD bool ed_outlier_selected(bool inside, double d, double thresh) { return inside && !(d < thresh); }

}  // namespace

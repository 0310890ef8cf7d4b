// Host build of the map editor's selection rules (glim_b200/csrc/gb_editor_math.cuh, the text k_plane_flags, k_rs_flags and
// k_rs_outliers compile, and the composition gb_select_gizmo runs on the host).  tests/test_editor_host.py compiles this with
// g++ -ffp-contract=off and compares it with the numpy restatement (tests/editor_oracle.py).
#include "../../glim_b200/csrc/gb_editor_math.cuh"

extern "C" {

// M (n x 16) = ed_compose of A (16) and B_i (n x 16), column-major
void compose(int n, const double* A, const double* B, double* M) {
  for (int i = 0; i < n; i++) ed_compose(A, B + 16 * i, M + 16 * i);
}

// out[i] = ed_in_box (box) or ed_in_sphere(r2) of fp64 q_i
void inside(int n, const double* q, int box, double r2, int* out) {
  for (int i = 0; i < n; i++) out[i] = (box ? ed_in_box(q + 3 * i) : ed_in_sphere(q + 3 * i, r2)) ? 1 : 0;
}

// out[i] = ed_radius_flags of fp32 point i about c
void radius_flags(int n, const float* xyz, const double* c, double inner2, double outer2, int* out) {
  for (int i = 0; i < n; i++) out[i] = ed_radius_flags(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], c, inner2, outer2);
}

// *th = ed_outlier_threshold(S, S2, m, stddev_thresh); out[i] = ed_outlier_selected(inside_i, d_i, *th)
void outliers(int n, double S, double S2, int m, double stddev_thresh, const double* d, const int* in, double* th, int* out) {
  *th = ed_outlier_threshold(S, S2, m, stddev_thresh);
  for (int i = 0; i < n; i++) out[i] = ed_outlier_selected(in[i] != 0, d[i], *th) ? 1 : 0;
}
}

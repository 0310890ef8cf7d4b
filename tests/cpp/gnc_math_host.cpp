// Host build of GNC's arithmetic (glim_b200/csrc/gb_global_math.cuh, the text k_gnc_solve compiles): the schedule of
// include/glim_b200.h run sequentially through the same functions the kernel calls.  tests/test_gnc_host.py compiles this with
// g++ -ffp-contract=off and compares it with the numpy restatement (tests/gnc_oracle.py).
#include "../../glim_b200/csrc/gb_global_math.cuh"

extern "C" {

// the schedule on K pairs (a source, b target; K x 3 each, fp64 of fp32 positions): T (16, column-major), the last iteration's
// weights (K), the iteration count; returns the status (0 found, 1 degenerate: K < 3, T = I, weights 0)
int gnc_solve(int K, const double* a, const double* b, int dof, double* T, double* weights, int* iterations) {
  *iterations = 0;
  if (K < 3) {
    for (int k = 0; k < 16; k++) T[k] = k % 5 == 0 ? 1.0 : 0.0;
    for (int k = 0; k < K; k++) weights[k] = 0.0;
    return 1;
  }
  double shift[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < K; k++)
    for (int r = 0; r < 3; r++) {
      shift[r] = __dadd_rn(shift[r], a[3 * k + r]);
      shift[3 + r] = __dadd_rn(shift[3 + r], b[3 * k + r]);
    }
  for (int r = 0; r < 6; r++) shift[r] = shift[r] / (double)K;
  const auto pose = [&](bool unit, double mu, bool last) {
    double s[kGncSums] = {};
    double Tn[16];
    for (int k = 0; k < K; k++) {
      double w = 1.0;
      if (!unit) {
        w = gnc_weight(mu, gnc_residual2(T, a + 3 * k, b + 3 * k));
        if (last) weights[k] = w;
      }
      double ac[3], bc[3];
      for (int r = 0; r < 3; r++) {
        ac[r] = __dsub_rn(a[3 * k + r], shift[r]);
        bc[r] = __dsub_rn(b[3 * k + r], shift[3 + r]);
      }
      gnc_accumulate(s, w, ac, bc);
    }
    gnc_pose(s, shift, shift + 3, dof, Tn);
    for (int e = 0; e < 16; e++) T[e] = Tn[e];
  };
  pose(true, 0.0, false);
  double max_r2 = 0.0;
  for (int k = 0; k < K; k++) max_r2 = fmax(max_r2, gnc_residual2(T, a + 3 * k, b + 3 * k));
  double mu = gnc_initial_scale(max_r2);
  for (;;) {
    const bool last = mu == kGncMinScale;
    pose(false, mu, last);
    ++*iterations;
    if (last) break;
    mu = gnc_next_scale(mu);
  }
  return 0;
}

// the weighted closed form of K pairs at weights w (about the means of a and b, as gnc_solve shifts them)
void gnc_pose_weighted(int K, const double* a, const double* b, const double* w, int dof, double* T) {
  double shift[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < K; k++)
    for (int r = 0; r < 3; r++) {
      shift[r] = __dadd_rn(shift[r], a[3 * k + r]);
      shift[3 + r] = __dadd_rn(shift[3 + r], b[3 * k + r]);
    }
  for (int r = 0; r < 6; r++) shift[r] = shift[r] / (double)K;
  double s[kGncSums] = {};
  for (int k = 0; k < K; k++) {
    double ac[3], bc[3];
    for (int r = 0; r < 3; r++) {
      ac[r] = __dsub_rn(a[3 * k + r], shift[r]);
      bc[r] = __dsub_rn(b[3 * k + r], shift[3 + r]);
    }
    gnc_accumulate(s, w[k], ac, bc);
  }
  gnc_pose(s, shift, shift + 3, dof, T);
}

// RANSAC's estimator on three pairs (3 x 3 each); returns 0 for an invalid sample
int ransac_pose3(const double* a, const double* b, int dof, double* T) { return ransac_pose(a, b, dof, T) ? 1 : 0; }

}  // extern "C"

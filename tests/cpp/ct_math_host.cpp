// Host build of the CT factor's per-problem arithmetic (glim_b200/csrc/gb_ct_math.cuh -- the SAME text k_ct_sweep, ct_reduce,
// k_ct_step and k_ct_accept compile) and of gb_ct_gicp_align's round structure for one problem.
// TEST INFRASTRUCTURE: built by tests/test_ct_host.py with g++ and compared with tests/ct_oracle.py on the CPU-only box;
// nothing in the product links it.
#include <string.h>

#include "../../glim_b200/csrc/gb_ct_math.cuh"

extern "C" int cm_time_table(const double* times, int n, int* starts, double* tau) { return ct_time_table(times, n, starts, tau); }
extern "C" void cm_exp(const double* xi, double* T) { ct_exp(xi, T); }
extern "C" void cm_log(const double* T, double* xi) { ct_log(T, xi); }
extern "C" void cm_jr(const double* xi, int inverse, double* J) { ct_se3_jr(xi, inverse != 0, J); }
extern "C" void cm_adjoint(const double* T, double* A) { ct_adjoint(T, A); }
extern "C" void cm_entry_pose(const double* X, const double* Y, double tau, double* T) {
  double xi[6];
  ct_motion(X, Y, xi);
  ct_entry_pose(X, xi, tau, T);
}
extern "C" void cm_entry_blocks(const double* X, const double* Y, double tau, double* D0, double* D1) {
  double xi[6], Jinv[36], AdYX[36];
  ct_problem_blocks(X, Y, xi, Jinv, AdYX);
  ct_entry_blocks(xi, Jinv, AdYX, tau, D0, D1);
}
extern "C" double cm_small_terms(const double* X, const double* Y, const double* Xp, double wl, double wc, double* H, double* b) {
  return ct_small_terms(X, Y, Xp, wl, wc, H, b);
}
extern "C" int cm_solve12(const double* H, const double* b, double lambda, double* delta) { return ct_solve12(H, b, lambda, delta) ? 1 : 0; }

// One problem driven through the device's round structure.  lin(X, Y, sys) writes the CT factor's 12x12 system at (X, Y)
// (H row-major 144 | b 12 | error | num_inliers); err(X_lin, Y_lin, X_eval, Y_eval) returns its error at the eval poses with
// the correspondences of the lin poses.
typedef void (*lin_fn)(const double* X, const double* Y, double* sys);
typedef double (*err_fn)(const double* Xl, const double* Yl, const double* Xe, const double* Ye);
extern "C" int cm_align(const gb_align_params* P, double wl, double wc, const double* X0, const double* Y0, const double* Xp, lin_fn lin, err_fn err,
                        double* X, double* Y, double* stats /* error num_inliers lambda iterations trials */) {
  CtState s;
  ct_init(s, X0, Y0, Xp, P->lambda_initial);
  double sys[158];
  while (s.a.status == GB_ALIGN_ACTIVE) {
    if (s.a.need_lin) {  // k_ct_step
      lin(s.a.T, s.Y, sys);
      memcpy(s.H, sys, sizeof(double) * 144);
      memcpy(s.b, sys + 144, sizeof(double) * 12);
      s.a.e = sys[156] + ct_small_terms(s.a.T, s.Y, s.Xp, wl, wc, s.H, s.b);
      s.a.n = sys[157];
      align_linearized(s.a);
      if (s.a.status != GB_ALIGN_ACTIVE) break;
    }
    ct_trial(s);
    const double e_new = err(s.a.T, s.Y, s.a.Tn, s.Yn) + ct_small_terms(s.a.Tn, s.Yn, s.Xp, wl, wc, nullptr, nullptr);  // k_ct_accept
    ct_conclude(s, *P, e_new);
  }
  memcpy(X, s.a.T, sizeof(double) * 16);
  memcpy(Y, s.Y, sizeof(double) * 16);
  stats[0] = s.a.e; stats[1] = s.a.n; stats[2] = s.a.lambda; stats[3] = s.a.iterations; stats[4] = s.a.trials;
  return s.a.status;
}

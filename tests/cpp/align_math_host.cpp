// Host build of gb_vgicp_align's per-problem arithmetic (glim_b200/csrc/gb_align_math.cuh -- the SAME text k_align_step /
// k_align_accept compile) and of its round structure for one problem: linearize -> gather -> trial -> error -> conclude.
// TEST INFRASTRUCTURE: built by tests/test_align_math_host.py with g++ and compared with numpy, synth.se3_exp and
// tests/lm_oracle.py (through tests/align_oracle.py's align_gpumap) on the CPU-only box; nothing in the product links it.
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../glim_b200/csrc/gb_align_math.cuh"

extern "C" int am_solve(const double* H, const double* b, double lambda, double* delta) { return align_solve(H, b, lambda, delta) ? 1 : 0; }
extern "C" void am_exp(const double* xi, double* E) { align_exp(xi, E); }
extern "C" void am_compose(const double* A, const double* B, double* C) { align_compose(A, B, C); }
extern "C" void am_step_norms(const double* xi, double* dt, double* dr) {
  double E[16];
  align_exp(xi, E);
  align_step_norms(E, xi, dt, dr);
}

// rule steps 4-5 on a state with the given fields; returns the status (-1 = still active)
extern "C" int am_conclude(const gb_align_params* P, int solved, double e, double e_new, double dt, double dr, int iterations, double lambda,
                           double* lambda_out, int* need_lin_out, double* e_out) {
  AlignState s;
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  align_init(s, I, lambda);
  s.solved = solved; s.e = e; s.dt = dt; s.dr = dr; s.iterations = iterations; s.need_lin = 0;
  align_conclude(s, *P, e_new);
  *lambda_out = s.lambda;
  *need_lin_out = s.need_lin;
  *e_out = s.e;
  return s.status;
}

// One problem of F factors driven through the device's round structure.  lin(T, records F x 122) linearizes every factor at T;
// err(T_lin, T_eval, records) writes each factor's error at T_eval with the inliers of T_lin into records[f * 122 + 120].
typedef void (*lin_fn)(const double* T, double* records);
typedef void (*err_fn)(const double* T_lin, const double* T_eval, double* records);
extern "C" int am_align(const gb_align_params* P, int F, const double* T_init, lin_fn lin, err_fn err, gb_align_result* r) {
  std::vector<double> out((size_t)F * 122, 0.0);
  AlignState s;
  align_init(s, T_init, P->lambda_initial);
  while (s.status == GB_ALIGN_ACTIVE) {
    if (s.need_lin) {
      lin(s.T, out.data());
      for (int k = 0; k < GB_ALIGN_STATE_ENTRIES; k++) align_set_entry(s, k, align_record_entry(out.data(), 0, F, k));
      align_linearized(s);
      if (s.status != GB_ALIGN_ACTIVE) break;
    }
    align_trial(s);
    err(s.T, s.Tn, out.data());
    align_conclude(s, *P, align_record_entry(out.data(), 0, F, 42));
  }
  memcpy(r->T_target_source, s.T, sizeof(double) * 16);
  align_result(s, *r);
  return 0;
}

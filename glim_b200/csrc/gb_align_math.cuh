// gb_align_math.cuh -- the per-problem Levenberg-Marquardt arithmetic of gb_vgicp_align (gb_align.cu) and gb_ct_gicp_align
// (gb_kernels_ct.cu): record sum, the N x N Cholesky solve, 3x3 helpers, the SE(3) Exp tail, compose, step norms, the accept /
// terminate rule of include/glim_b200.h, the round's status word and the result fields.  Like gb_vgicp_math.cuh it holds
// nothing that only exists on the device (the status-word helpers excepted), so the SAME TEXT compiles for the host:
// tests/cpp/align_math_host.cpp builds it with g++ and tests/test_align_math_host.py checks it against numpy, synth.se3_exp
// and the rule's restatement in tests/lm_oracle.py.
// All poses are 4x4 column-major doubles; tangent order [rot; trans] (GTSAM Pose3, SURVEY A.3); square matrices are ROW-major.
#pragma once
#ifdef __CUDACC__
#define GB_AHD __host__ __device__ inline
#else
#include <math.h>
#define GB_AHD static inline
#endif

#include "../../include/glim_b200.h"

#define GB_ALIGN_ACTIVE (-1)       // status of a problem that is still iterating
#define GB_ALIGN_STATE_ENTRIES 44  // H_ss (36, column-major in the record) | b (6) | error | num_inliers

namespace {

// Everything the rule keeps for one problem between rounds.
struct AlignState {
  double T[16];      // current pose
  double Tn[16];     // trial pose T * Exp(delta)
  double H[36];      // sum of H_ss of the last linearization (row-major)
  double b[6];       // sum of b_s
  double e;          // error: of the last linearization, then of the accepted trial pose
  double n;          // inliers of the last linearization
  double lambda;
  double dt, dr;     // step of the last trial: translation norm (m), rotation angle (rad)
  int iterations;    // linearizations
  int trials;        // solves
  int status;        // GB_ALIGN_ACTIVE or a final GB_ALIGN_* status
  int need_lin;      // the next round linearizes at T
  int solved;        // the last trial's factorization succeeded
  int pad;
};

// entry k of the state vector (H_ss column-major | b | error | num_inliers) summed over the records [f0, f1) of a
// F x GB_OUT_DOUBLES (122) record array, in record order
GB_AHD double align_record_entry(const double* out, int f0, int f1, int k) {
  const int r = k < 36 ? 36 + k : (k < 42 ? 114 + (k - 36) : 120 + (k - 42));  // H_ss | b_s | error | num_inliers
  double s = 0.0;
  for (int f = f0; f < f1; f++) s += out[(size_t)f * 122 + r];
  return s;
}
// entry k of the state vector into the state (H_ss transposed into the row-major H)
GB_AHD void align_set_entry(AlignState& s, int k, double v) {
  if (k < 36) s.H[(k % 6) * 6 + k / 6] = v;
  else if (k < 42) s.b[k - 36] = v;
  else if (k == 42) s.e = v;
  else s.n = v;
}

// (H + lambda I) delta = -b for an N x N row-major H by Cholesky (lower, row by row; only H(i, j <= i) is read).  N is 6
// for a pose problem (the default) and 12 for a CT problem (ct_solve12).  false: not positive definite (or not finite).
template <int N = 6>
GB_AHD bool align_solve(const double* H, const double* b, double lambda, double* delta) {
  double L[N * N];
  for (int i = 0; i < N; i++) {
    for (int j = 0; j <= i; j++) {
      double s = H[i * N + j] + (i == j ? lambda : 0.0);
      for (int k = 0; k < j; k++) s -= L[i * N + k] * L[j * N + k];
      if (i == j) {
        if (!(s > 0.0) || !(s < INFINITY)) return false;
        L[i * N + i] = sqrt(s);
      } else {
        L[i * N + j] = s / L[j * N + j];
      }
    }
  }
  double y[N];
  for (int i = 0; i < N; i++) {
    double s = -b[i];
    for (int k = 0; k < i; k++) s -= L[i * N + k] * y[k];
    y[i] = s / L[i * N + i];
  }
  for (int i = N - 1; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < N; k++) s -= L[k * N + i] * delta[k];
    delta[i] = s / L[i * N + i];
  }
  return true;
}

// ---- 3x3 helpers (row-major) ----
GB_AHD void mat3_hat(const double* w, double* K) {
  K[0] = 0.0; K[1] = -w[2]; K[2] = w[1];
  K[3] = w[2]; K[4] = 0.0; K[5] = -w[0];
  K[6] = -w[1]; K[7] = w[0]; K[8] = 0.0;
}
GB_AHD void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
}

// Pose3::Expmap([w; v]) as a column-major 4x4 from its coefficients: R = I + a K + bb K^2, V = I + bb K + c K^2, t = V v
// (K = hat(w)).  align_exp and ct_exp choose a, bb, c by their own rules.
GB_AHD void se3_exp_coeffs(const double* xi, double a, double bb, double c, double* E) {
  double K[9], K2[9];
  mat3_hat(xi, K);
  mat3_mul(K, K, K2);
  double V[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      const double I = i == j ? 1.0 : 0.0;
      E[j * 4 + i] = I + a * K[i * 3 + j] + bb * K2[i * 3 + j];
      V[i * 3 + j] = I + bb * K[i * 3 + j] + c * K2[i * 3 + j];
    }
  for (int i = 0; i < 3; i++) {
    E[12 + i] = V[i * 3 + 0] * xi[3] + V[i * 3 + 1] * xi[4] + V[i * 3 + 2] * xi[5];
    E[i * 4 + 3] = 0.0;
  }
  E[15] = 1.0;
}

// Pose3::Expmap([w; v]) as a column-major 4x4 (the formulas of synth.se3_exp; second-order series below 1e-10 rad)
GB_AHD void align_exp(const double* xi, double* E) {
  const double th2 = xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2], th = sqrt(th2);
  double a, bb, c;
  if (th < 1e-10) {
    a = 1.0; bb = 0.5; c = 0.0;
  } else {
    a = sin(th) / th; bb = (1.0 - cos(th)) / th2; c = (th - sin(th)) / (th2 * th);
  }
  se3_exp_coeffs(xi, a, bb, c, E);
}

// C = A B (column-major 4x4 rigid transforms)
GB_AHD void align_compose(const double* A, const double* B, double* C) {
  for (int j = 0; j < 4; j++)
    for (int i = 0; i < 4; i++) {
      double s = 0.0;
      for (int k = 0; k < 4; k++) s += A[k * 4 + i] * B[j * 4 + k];
      C[j * 4 + i] = s;
    }
}

// size of the step Exp(delta): translation norm and rotation angle |w| (what GLIM's termination_criteria measures on
// last_estimate^-1 * current_pose, odometry_estimation_cpu.cpp:121-135)
GB_AHD void align_step_norms(const double* E, const double* xi, double* dt, double* dr) {
  *dt = sqrt(E[12] * E[12] + E[13] * E[13] + E[14] * E[14]);
  *dr = sqrt(xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]);
}

GB_AHD void align_init(AlignState& s, const double* T_init, double lambda) {
  for (int k = 0; k < 16; k++) { s.T[k] = T_init[k]; s.Tn[k] = T_init[k]; }
  for (int k = 0; k < 36; k++) s.H[k] = 0.0;
  for (int k = 0; k < 6; k++) s.b[k] = 0.0;
  s.e = 0.0; s.n = 0.0; s.lambda = lambda; s.dt = 0.0; s.dr = 0.0;
  s.iterations = 0; s.trials = 0; s.status = GB_ALIGN_ACTIVE; s.need_lin = 1; s.solved = 0; s.pad = 0;
}

// rule step 1, after H, b, e, n have been summed from a linearization at T
GB_AHD void align_linearized(AlignState& s) {
  s.iterations += 1;
  s.need_lin = 0;
  if (s.n == 0.0 && s.iterations == 1) s.status = GB_ALIGN_DEGENERATE;  // T is still T_init
}

// rule step 2: solve and form the trial pose (a failed factorization leaves Tn = T and is rejected by align_conclude)
GB_AHD void align_trial(AlignState& s) {
  double d[6], E[16];
  s.trials += 1;
  s.solved = align_solve(s.H, s.b, s.lambda, d) ? 1 : 0;
  if (!s.solved) {
    for (int k = 0; k < 16; k++) s.Tn[k] = s.T[k];
    s.dt = 0.0; s.dr = 0.0;
    return;
  }
  align_exp(d, E);
  align_compose(s.T, E, s.Tn);
  align_step_norms(E, d, &s.dt, &s.dr);
}

// rule steps 4-5, given the error e_new of the trial pose with the inliers of T
GB_AHD void align_conclude(AlignState& s, const gb_align_params& P, double e_new) {
  if (s.solved && e_new < s.e) {  // accept
    for (int k = 0; k < 16; k++) s.T[k] = s.Tn[k];
    s.lambda /= P.lambda_factor;
    s.need_lin = 1;
    const double de = s.e - e_new;
    const bool tiny = s.dt < 1e-10 && s.dr < 1e-10;  // "maybe failed to solve the linear system" (odometry_estimation_cpu.cpp:129-131)
    if (!tiny && s.dt < P.step_translation_tol && s.dr < P.step_rotation_tol) s.status = GB_ALIGN_CONVERGED;
    else if (de <= P.absolute_error_tol || de / s.e <= P.relative_error_tol) s.status = GB_ALIGN_CONVERGED;
    else if (s.iterations >= P.max_iterations) s.status = GB_ALIGN_MAX_ITERATIONS;
    s.e = e_new;
  } else {  // reject
    s.lambda *= P.lambda_factor;
    s.need_lin = 0;
    if (s.lambda > P.lambda_upper_bound) s.status = GB_ALIGN_LAMBDA_EXCEEDED;
  }
}

// the result fields every solve reports (gb_align_result, gb_ct_result) from a concluded state
template <class Result>
GB_AHD void align_result(const AlignState& s, Result& r) {
  r.error = s.e;
  r.num_inliers = s.n;
  r.lambda = s.lambda;
  r.iterations = s.iterations;
  r.trials = s.trials;
  r.status = s.status;
}

#ifdef __CUDACC__
// The status word of a round: [0] the active problems, [1] those of them that need a linearization.  Block 0 of the step
// kernel clears it; the accept kernel tallies every problem it concludes and gets its flags back (1: need_lin, 2: active).
__device__ __forceinline__ void align_status_clear(unsigned* ctr) {
  if (blockIdx.x == 0 && threadIdx.x < 2) ctr[threadIdx.x] = 0u;
}
__device__ __forceinline__ int align_status_tally(const AlignState& s, unsigned* ctr) {
  const int flags = (s.need_lin ? 1 : 0) | (s.status == GB_ALIGN_ACTIVE ? 2 : 0);
  if (flags & 2) atomicAdd(&ctr[0], 1u);
  if (flags == 3) atomicAdd(&ctr[1], 1u);
  return flags;
}
#endif

}  // namespace

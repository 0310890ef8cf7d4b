// gb_ct_math.cuh -- the arithmetic of the continuous-time GICP factor and its solve (gb_kernels_ct.cu): the time table of
// gb_cloud_add_times, SE(3) Exp / Log / right Jacobian / its inverse / adjoint, the entry poses and their chain-rule blocks
// D0 / D1, the prior and between terms of gb_ct_gicp_align, and its trial step (ct_solve12 is align_solve at 12 dof).  Like
// gb_align_math.cuh it holds nothing that only exists on the device, so the SAME TEXT compiles for the host:
// tests/cpp/ct_math_host.cpp builds it with g++ and tests/test_ct_host.py checks it against tests/ct_oracle.py.
// The rule is written once, in include/glim_b200.h.  Poses are 4x4 column-major doubles, tangent order [rot; trans] with
// perturbations on the right (GTSAM Pose3, Expmap chart); 6x6 and 12x12 matrices here are ROW-major.
#pragma once
#include "gb_align_math.cuh"  // GB_AHD, AlignState, align_solve, mat3_*, se3_exp_coeffs, align_compose, align_step_norms, align_linearized, align_conclude

#define GB_CT_TIME_EPS 1e-3  // s: a point opens a new time-table entry iff it is later than the entry's time by more than this

namespace {

// The time table of n ascending times: entry starts (starts[0] = 0, starts[B] = n) and normalized times tau[b].  starts and
// tau hold n + 1 and n entries.  Returns B (0 for n == 0).
GB_AHD int ct_time_table(const double* times, int n, int* starts, double* tau) {
  if (n <= 0) { starts[0] = 0; return 0; }
  int B = 0;
  double cur = times[0];
  starts[B++] = 0;
  for (int i = 1; i < n; i++) {
    if (times[i] - cur > GB_CT_TIME_EPS) {
      starts[B++] = i;
      cur = times[i];
    }
  }
  starts[B] = n;
  const double t0 = times[0], span = cur - t0;
  for (int b = 0; b < B; b++) tau[b] = B == 1 ? 0.0 : (times[starts[b]] - t0) / span;
  return B;
}

// SO(3) left Jacobian J_l(w) = I + a K + c K^2 and its inverse I - K / 2 + d K^2 (series below 1e-2 rad)
GB_AHD void ct_so3_jl(const double* w, bool inverse, double* J) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double K[9], K2[9];
  mat3_hat(w, K);
  mat3_mul(K, K, K2);
  double a, c;
  if (inverse) {
    a = -0.5;
    c = th < 1e-2 ? 1.0 / 12.0 + th2 / 720.0 + th2 * th2 / 30240.0 : 1.0 / th2 - (1.0 + cos(th)) / (2.0 * th * sin(th));
  } else if (th < 1e-2) {
    a = 0.5 - th2 / 24.0 + th2 * th2 / 720.0;
    c = 1.0 / 6.0 - th2 / 120.0 + th2 * th2 / 5040.0;
  } else {
    a = (1.0 - cos(th)) / th2;
    c = (th - sin(th)) / (th2 * th);
  }
  for (int e = 0; e < 9; e++) J[e] = (e % 4 == 0 ? 1.0 : 0.0) + a * K[e] + c * K2[e];
}

// SE(3) left Jacobian of xi = [w; v]: [[J, 0], [Q, J]] (row-major 6x6), or its inverse [[J^-1, 0], [-J^-1 Q J^-1, J^-1]].
// Q(w, v) as Barfoot, "State Estimation for Robotics", eq. 7.86 (translation and rotation blocks swapped); series below 0.1 rad.
GB_AHD void ct_se3_jl(const double* xi, bool inverse, double* J6) {
  const double* w = xi;
  const double* v = xi + 3;
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double c1, c2, c3;
  if (th < 0.1) {
    const double t4 = th2 * th2, t6 = t4 * th2;
    c1 = 1.0 / 6.0 - th2 / 120.0 + t4 / 5040.0 - t6 / 362880.0;
    c2 = 1.0 / 24.0 - th2 / 720.0 + t4 / 40320.0 - t6 / 3628800.0;
    c3 = 1.0 / 120.0 - th2 / 2520.0 + t4 / 120960.0 - t6 / 9979200.0;
  } else {
    const double s = sin(th), c = cos(th);
    c1 = (th - s) / (th2 * th);
    c2 = (th2 + 2.0 * c - 2.0) / (2.0 * th2 * th2);
    c3 = (2.0 * th - 3.0 * s + th * c) / (2.0 * th2 * th2 * th);
  }
  double P[9], R[9], PR[9], RP[9], PRP[9], PP[9], PPR[9], RPP[9], PRPP[9], PPRP[9], Q[9];
  mat3_hat(w, P);
  mat3_hat(v, R);
  mat3_mul(P, R, PR);
  mat3_mul(R, P, RP);
  mat3_mul(PR, P, PRP);
  mat3_mul(P, P, PP);
  mat3_mul(PP, R, PPR);
  mat3_mul(RP, P, RPP);
  mat3_mul(PRP, P, PRPP);
  mat3_mul(P, PRP, PPRP);
  for (int e = 0; e < 9; e++)
    Q[e] = 0.5 * R[e] + c1 * (PR[e] + RP[e] + PRP[e]) + c2 * (PPR[e] + RPP[e] - 3.0 * PRP[e]) + c3 * (PRPP[e] + PPRP[e]);
  double J[9];
  ct_so3_jl(w, inverse, J);
  double B[9];
  if (inverse) {
    double T[9];
    mat3_mul(J, Q, T);
    mat3_mul(T, J, B);
    for (int e = 0; e < 9; e++) B[e] = -B[e];
  } else {
    for (int e = 0; e < 9; e++) B[e] = Q[e];
  }
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) {
      const int r = i % 3, c = j % 3;
      J6[i * 6 + j] = (i < 3) == (j < 3) ? J[r * 3 + c] : (i >= 3 ? B[r * 3 + c] : 0.0);
    }
}

// SE(3) right Jacobian J_r(xi) = J_l(-xi), or its inverse
GB_AHD void ct_se3_jr(const double* xi, bool inverse, double* J6) {
  const double m[6] = {-xi[0], -xi[1], -xi[2], -xi[3], -xi[4], -xi[5]};
  ct_se3_jl(m, inverse, J6);
}

// Pose3::Expmap and Pose3::Logmap of a column-major rigid transform.  ct_exp is se3_exp_coeffs with series coefficients below
// 1e-2 rad (align_exp's closed form loses the K^2 coefficient of V at tiny angles, which the entry poses of a slow scan reach);
// Exp(0) is exactly the identity.
GB_AHD void ct_exp(const double* xi, double* E) {
  const double th2 = xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2], th = sqrt(th2);
  double a, bb, c;
  if (th < 1e-2) {
    a = 1.0 - th2 / 6.0 + th2 * th2 / 120.0;
    bb = 0.5 - th2 / 24.0 + th2 * th2 / 720.0;
    c = 1.0 / 6.0 - th2 / 120.0 + th2 * th2 / 5040.0;
  } else {
    a = sin(th) / th; bb = (1.0 - cos(th)) / th2; c = (th - sin(th)) / (th2 * th);
  }
  se3_exp_coeffs(xi, a, bb, c, E);
}
GB_AHD void ct_log(const double* T, double* xi) {
  // R(i, j) = T[j * 4 + i]
  const double tr = T[0] + T[5] + T[10];
  const double vx = T[6] - T[9], vy = T[8] - T[2], vz = T[1] - T[4];  // R - R^T = 2 sin(th) hat(axis)
  const double s2 = sqrt(vx * vx + vy * vy + vz * vz);               // 2 sin(th)
  double cth = 0.5 * (tr - 1.0);
  cth = cth > 1.0 ? 1.0 : (cth < -1.0 ? -1.0 : cth);
  const double th = atan2(0.5 * s2, cth);
  double w[3];
  if (cth > -0.99) {
    const double f = th < 1e-4 ? 0.5 + th * th / 12.0 : th / s2;  // th / (2 sin th)
    w[0] = f * vx; w[1] = f * vy; w[2] = f * vz;
  } else {  // near pi: the axis from the largest diagonal of (R + I) / 2 = a a^T (1 - cos) / 2 + cos-part; sign from R - R^T
    const double d0 = T[0], d1 = T[5], d2 = T[10];
    const double oc = 1.0 - cth;
    double a[3];
    if (d0 >= d1 && d0 >= d2) {
      a[0] = sqrt((d0 - cth) / oc);
      a[1] = (T[4] + T[1]) / (2.0 * oc * a[0]);
      a[2] = (T[8] + T[2]) / (2.0 * oc * a[0]);
    } else if (d1 >= d2) {
      a[1] = sqrt((d1 - cth) / oc);
      a[0] = (T[4] + T[1]) / (2.0 * oc * a[1]);
      a[2] = (T[9] + T[6]) / (2.0 * oc * a[1]);
    } else {
      a[2] = sqrt((d2 - cth) / oc);
      a[0] = (T[8] + T[2]) / (2.0 * oc * a[2]);
      a[1] = (T[9] + T[6]) / (2.0 * oc * a[2]);
    }
    if (a[0] * vx + a[1] * vy + a[2] * vz < 0.0) { a[0] = -a[0]; a[1] = -a[1]; a[2] = -a[2]; }
    const double an = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    for (int k = 0; k < 3; k++) w[k] = th * a[k] / an;
  }
  double Ji[9];
  ct_so3_jl(w, true, Ji);
  xi[0] = w[0]; xi[1] = w[1]; xi[2] = w[2];
  for (int i = 0; i < 3; i++) xi[3 + i] = Ji[i * 3 + 0] * T[12] + Ji[i * 3 + 1] * T[13] + Ji[i * 3 + 2] * T[14];
}

// inverse of a column-major rigid transform
GB_AHD void ct_inverse(const double* T, double* Ti) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) Ti[j * 4 + i] = T[i * 4 + j];
  for (int i = 0; i < 3; i++) Ti[12 + i] = -(T[i * 4 + 0] * T[12] + T[i * 4 + 1] * T[13] + T[i * 4 + 2] * T[14]);
  Ti[3] = Ti[7] = Ti[11] = 0.0;
  Ti[15] = 1.0;
}

// Ad(T) = [[R, 0], [hat(t) R, R]] (row-major 6x6)
GB_AHD void ct_adjoint(const double* T, double* A) {
  double R[9], K[9], KR[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[i * 3 + j] = T[j * 4 + i];
  mat3_hat(T + 12, K);
  mat3_mul(K, R, KR);
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) {
      const int r = i % 3, c = j % 3;
      A[i * 6 + j] = (i < 3) == (j < 3) ? R[r * 3 + c] : (i >= 3 ? KR[r * 3 + c] : 0.0);
    }
}

GB_AHD void ct_mul6(const double* A, const double* B, double* C) {
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) {
      double s = 0.0;
      for (int k = 0; k < 6; k++) s += A[i * 6 + k] * B[k * 6 + j];
      C[i * 6 + j] = s;
    }
}

// xi = Log(X^-1 Y): the motion of a scan from its first to its last time-table entry
GB_AHD void ct_motion(const double* X, const double* Y, double* xi) {
  double Xi[16], D[16];
  ct_inverse(X, Xi);
  align_compose(Xi, Y, D);
  ct_log(D, xi);
}

// the pose of an entry with normalized time tau: T = X Exp(tau xi)
GB_AHD void ct_entry_pose(const double* X, const double* xi, double tau, double* T) {
  const double s[6] = {tau * xi[0], tau * xi[1], tau * xi[2], tau * xi[3], tau * xi[4], tau * xi[5]};
  double E[16];
  ct_exp(s, E);
  align_compose(X, E, T);
}

// The chain-rule blocks of an entry pose T = X Exp(tau xi), xi = Log(X^-1 Y), for right perturbations of X and Y:
//   D0 = Ad(Exp(-tau xi)) - tau J_r(tau xi) J_r^-1(xi) Ad(Y^-1 X),   D1 = tau J_r(tau xi) J_r^-1(xi)   (row-major 6x6).
// Jinv_xi = J_r^-1(xi) and Ad_YX = Ad(Y^-1 X) are the same for every entry of a problem (ct_problem_blocks).
GB_AHD void ct_problem_blocks(const double* X, const double* Y, double* xi, double* Jinv_xi, double* Ad_YX) {
  ct_motion(X, Y, xi);
  ct_se3_jr(xi, true, Jinv_xi);
  double Yi[16], YX[16];
  ct_inverse(Y, Yi);
  align_compose(Yi, X, YX);
  ct_adjoint(YX, Ad_YX);
}
GB_AHD void ct_entry_blocks(const double* xi, const double* Jinv_xi, const double* Ad_YX, double tau, double* D0, double* D1) {
  const double s[6] = {tau * xi[0], tau * xi[1], tau * xi[2], tau * xi[3], tau * xi[4], tau * xi[5]};
  const double m[6] = {-s[0], -s[1], -s[2], -s[3], -s[4], -s[5]};
  double Jt[36], E[16], AdE[36], T[36];
  ct_se3_jr(s, false, Jt);
  ct_exp(m, E);
  ct_adjoint(E, AdE);
  ct_mul6(Jt, Jinv_xi, T);
  for (int e = 0; e < 36; e++) D1[e] = tau * T[e];
  ct_mul6(D1, Ad_YX, T);
  for (int e = 0; e < 36; e++) D0[e] = AdE[e] - T[e];
}

// The two small terms of the objective at (X, Y): w_prior |Log(Xp^-1 X)|^2 + w_between |Log(X^-1 Y)|^2, added to the 12x12
// system (row-major H, b over [X; Y]) when H and b are given.  Jacobians: J_r^-1(r) for X in the prior; -J_r^-1(r) Ad(Y^-1 X)
// for X and J_r^-1(r) for Y in the between term.  No 1/2, as the CT error: e += w r^T r, H += w J^T J, b += w J^T r.
GB_AHD double ct_small_terms(const double* X, const double* Y, const double* Xp, double w_prior, double w_between, double* H, double* b) {
  double Xpi[16], D[16], r[6], J[36];
  ct_inverse(Xp, Xpi);
  align_compose(Xpi, X, D);
  ct_log(D, r);
  double e = 0.0;
  for (int k = 0; k < 6; k++) e += w_prior * r[k] * r[k];
  if (H) {
    ct_se3_jr(r, true, J);
    for (int i = 0; i < 6; i++) {
      for (int j = 0; j < 6; j++) {
        double s = 0.0;
        for (int k = 0; k < 6; k++) s += J[k * 6 + i] * J[k * 6 + j];
        H[i * 12 + j] += w_prior * s;
      }
      double s = 0.0;
      for (int k = 0; k < 6; k++) s += J[k * 6 + i] * r[k];
      b[i] += w_prior * s;
    }
  }
  double xi[6], Jinv[36], AdYX[36];
  ct_problem_blocks(X, Y, xi, Jinv, AdYX);
  for (int k = 0; k < 6; k++) e += w_between * xi[k] * xi[k];
  if (H) {
    double Jx[36], Jb[72];  // Jb: 6 x 12 = [-Jinv Ad_YX, Jinv]
    ct_mul6(Jinv, AdYX, Jx);
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) { Jb[i * 12 + j] = -Jx[i * 6 + j]; Jb[i * 12 + 6 + j] = Jinv[i * 6 + j]; }
    for (int i = 0; i < 12; i++) {
      for (int j = 0; j < 12; j++) {
        double s = 0.0;
        for (int k = 0; k < 6; k++) s += Jb[k * 12 + i] * Jb[k * 12 + j];
        H[i * 12 + j] += w_between * s;
      }
      double s = 0.0;
      for (int k = 0; k < 6; k++) s += Jb[k * 12 + i] * xi[k];
      b[i] += w_between * s;
    }
  }
  return e;
}

// the 12x12 solve of a CT problem over [X; Y] (row-major H): align_solve at 12 dof
GB_AHD bool ct_solve12(const double* H, const double* b, double lambda, double* delta) { return align_solve<12>(H, b, lambda, delta); }

// Everything gb_ct_gicp_align keeps for one problem.  The accept / terminate rule is gb_vgicp_align's (align_conclude on
// `a`): a.T / a.Tn hold X and its trial, Y / Yn the scan-end pose and its trial; a.H and a.b are unused.
struct CtState {
  AlignState a;
  double Y[16], Yn[16];
  double Xp[16];     // the prior's pose (last_T_world_lidar_end)
  double H[144];     // 12x12 of the last linearization, row-major over [X; Y]
  double b[12];
};

GB_AHD void ct_init(CtState& s, const double* X, const double* Y, const double* Xp, double lambda) {
  align_init(s.a, X, lambda);
  for (int k = 0; k < 16; k++) { s.Y[k] = Y[k]; s.Yn[k] = Y[k]; s.Xp[k] = Xp[k]; }
  for (int k = 0; k < 144; k++) s.H[k] = 0.0;
  for (int k = 0; k < 12; k++) s.b[k] = 0.0;
}

// rule step 2 at 12 dof: solve, X' = X Exp(d_X), Y' = Y Exp(d_Y).  The step size that the step tests read is the larger of the
// two poses' steps (translation norm and rotation angle).
GB_AHD void ct_trial(CtState& s) {
  double d[12], E[16], dt, dr;
  s.a.trials += 1;
  s.a.solved = ct_solve12(s.H, s.b, s.a.lambda, d) ? 1 : 0;
  if (!s.a.solved) {
    for (int k = 0; k < 16; k++) { s.a.Tn[k] = s.a.T[k]; s.Yn[k] = s.Y[k]; }
    s.a.dt = 0.0; s.a.dr = 0.0;
    return;
  }
  ct_exp(d, E);
  align_compose(s.a.T, E, s.a.Tn);
  align_step_norms(E, d, &s.a.dt, &s.a.dr);
  ct_exp(d + 6, E);
  align_compose(s.Y, E, s.Yn);
  align_step_norms(E, d + 6, &dt, &dr);
  s.a.dt = s.a.dt > dt ? s.a.dt : dt;
  s.a.dr = s.a.dr > dr ? s.a.dr : dr;
}

// rule steps 4-5 (align_conclude), given the objective at the trial poses; an accepted trial moves Y too
GB_AHD void ct_conclude(CtState& s, const gb_align_params& P, double e_new) {
  align_conclude(s.a, P, e_new);
  if (s.a.need_lin)
    for (int k = 0; k < 16; k++) s.Y[k] = s.Yn[k];
}

}  // namespace

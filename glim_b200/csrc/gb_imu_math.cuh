// gb_imu_math.cuh -- the arithmetic of gb_imu_preintegrate (gb_imu.cu) and of the navigation terms of gb_nav_graph_optimize
// (gb_pose_graph.cu): one preintegration step with its Jacobians A, B, C, the window of IMUIntegration::integrate_imu, the IMU
// term (ImuFactor's residual and its Jacobian in the solver's charts) and the vector terms.  The rules are stated in
// include/glim_b200.h.  Like gb_ct_math.cuh it holds nothing that only exists on the device, so the SAME TEXT compiles for the
// host: tests/cpp/imu_math_host.cpp builds it with g++ and tests/test_imu_host.py checks it against tests/imu_oracle.py.
// Poses are 4x4 column-major doubles; 3x3 and 9xM matrices here are ROW-major.  The preintegrated vector is [theta; p; v].
#pragma once
#include "gb_ct_math.cuh"  // ct_so3_jl, ct_log; through gb_align_math.cuh: GB_AHD, mat3_hat, mat3_mul

#define IMU_TERM_COLS 30  // an IMU term's Jacobian: pose_i | vel_i (3 live) | pose_j | vel_j (3 live) | bias_i [acc; gyro]

namespace {

// R = Exp(w) (row-major 3x3)
GB_AHD void imu_so3_exp(const double* w, double* R) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], th = sqrt(th2);
  double a, b;
  if (th < 1e-2) {
    a = 1.0 - th2 / 6.0 + th2 * th2 / 120.0;
    b = 0.5 - th2 / 24.0 + th2 * th2 / 720.0;
  } else {
    a = sin(th) / th;
    b = (1.0 - cos(th)) / th2;
  }
  double K[9], K2[9];
  mat3_hat(w, K);
  mat3_mul(K, K, K2);
  for (int e = 0; e < 9; e++) R[e] = (e % 4 == 0 ? 1.0 : 0.0) + a * K[e] + b * K2[e];
}

// Log(R) of a row-major rotation (ct_log on its rigid transform)
GB_AHD void imu_so3_log(const double* R, double* w) {
  double T[16] = {0.0}, xi[6];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) T[j * 4 + i] = R[i * 3 + j];
  T[15] = 1.0;
  ct_log(T, xi);
  w[0] = xi[0]; w[1] = xi[1]; w[2] = xi[2];
}

// J_r(w) and J_r(w)^-1 (J_r(w) = J_l(-w))
GB_AHD void imu_so3_jr(const double* w, bool inverse, double* J) {
  const double m[3] = {-w[0], -w[1], -w[2]};
  ct_so3_jl(m, inverse, J);
}

GB_AHD void mat3_transpose(const double* A, double* At) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) At[j * 3 + i] = A[i * 3 + j];
}
GB_AHD void mat3_vec(const double* A, const double* x, double* y) {
  for (int i = 0; i < 3; i++) y[i] = A[i * 3 + 0] * x[0] + A[i * 3 + 1] * x[1] + A[i * 3 + 2] * x[2];
}

// D = d(J_r(th)^-1 w) / d th, exactly: J_r^-1 w = w + th x w / 2 + c(t) th x (th x w) with t = |th| and
// c = 1 / t^2 - (1 + cos t) / (2 t sin t), so D = -[w]x / 2 + c ((th.w) I + th w^T - 2 w th^T) + (c'(t) / t) (th x (th x w)) th^T
// (series of c and c' / t below 0.1 rad)
GB_AHD void imu_dinvjr(const double* th, const double* w, double* D) {
  const double t2 = th[0] * th[0] + th[1] * th[1] + th[2] * th[2], t = sqrt(t2);
  double c, cpt;
  if (t < 0.1) {
    c = 1.0 / 12.0 + t2 / 720.0 + t2 * t2 / 30240.0;
    cpt = 1.0 / 360.0 + t2 / 7560.0 + t2 * t2 / 201600.0;
  } else {
    const double s = sin(t), ct = cos(t), cot = (1.0 + ct) / s, csc2 = 1.0 / ((1.0 - ct) * 0.5);  // cot(t/2), csc^2(t/2)
    c = 1.0 / t2 - cot / (2.0 * t);
    cpt = (-2.0 / (t2 * t) + csc2 / (4.0 * t) + cot / (2.0 * t2)) / t;
  }
  const double tw = th[0] * w[0] + th[1] * w[1] + th[2] * w[2];
  double u[3];  // th x (th x w) = th (th.w) - w t^2
  for (int i = 0; i < 3; i++) u[i] = th[i] * tw - w[i] * t2;
  double W[9];
  mat3_hat(w, W);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      D[i * 3 + j] = -0.5 * W[i * 3 + j] + c * ((i == j ? tw : 0.0) + th[i] * w[j] - 2.0 * w[i] * th[j]) + cpt * u[i] * th[j];
}

// One step of the tangent preintegration at x = [theta; p; v] with bias-corrected a, w: xn and (when given) A (9x9), B, C (9x3)
GB_AHD void imu_step_jacobians(const double* x, const double* a, const double* w, double dt, double* xn, double* A, double* B, double* C) {
  const double* th = x;
  double R[9], Ji[9], Jr[9], wt[3], an[3];
  imu_so3_exp(th, R);
  imu_so3_jr(th, true, Ji);
  mat3_vec(Ji, w, wt);
  mat3_vec(R, a, an);
  const double dt22 = 0.5 * dt * dt;
  for (int i = 0; i < 3; i++) {
    xn[i] = th[i] + wt[i] * dt;
    xn[3 + i] = x[3 + i] + x[6 + i] * dt + an[i] * dt22;
    xn[6 + i] = x[6 + i] + an[i] * dt;
  }
  if (!A) return;
  double D[9], na[3] = {-a[0], -a[1], -a[2]}, Ka[9], RK[9], RKJ[9];
  imu_dinvjr(th, w, D);
  imu_so3_jr(th, false, Jr);
  mat3_hat(na, Ka);
  mat3_mul(R, Ka, RK);
  mat3_mul(RK, Jr, RKJ);  // d(R a) / d theta
  for (int e = 0; e < 81; e++) A[e] = e % 10 == 0 ? 1.0 : 0.0;
  for (int e = 0; e < 27; e++) B[e] = C[e] = 0.0;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      A[i * 9 + j] += D[i * 3 + j] * dt;
      A[(3 + i) * 9 + j] = RKJ[i * 3 + j] * dt22;
      A[(3 + i) * 9 + 6 + j] = i == j ? dt : 0.0;
      A[(6 + i) * 9 + j] = RKJ[i * 3 + j] * dt;
      B[(3 + i) * 3 + j] = R[i * 3 + j] * dt22;
      B[(6 + i) * 3 + j] = R[i * 3 + j] * dt;
      C[i * 3 + j] = Ji[i * 3 + j] * dt;
    }
}

// A record reset to bias b_hat: zero state, Jacobians and covariance
GB_AHD void imu_reset(gb_imu_preintegrated& p, const double* bias, const gb_imu_params& prm) {
  p.delta_t = 0.0;
  for (int e = 0; e < 9; e++) p.preintegrated[e] = 0.0;
  for (int e = 0; e < 27; e++) p.H_bias_acc[e] = p.H_bias_omega[e] = 0.0;
  for (int e = 0; e < 81; e++) p.covariance[e] = 0.0;
  for (int e = 0; e < 6; e++) p.bias_hat[e] = bias[e];
  for (int e = 0; e < 3; e++) p.gravity[e] = prm.gravity[e];
  p.num_integrated = 0;
  p.pad = 0;
}

// PreintegratedImuMeasurements::integrateMeasurement(acc, omega, dt) on the record
GB_AHD void imu_integrate(gb_imu_preintegrated& p, const double* acc, const double* omega, double dt, const gb_imu_params& prm) {
  const double a[3] = {acc[0] - p.bias_hat[0], acc[1] - p.bias_hat[1], acc[2] - p.bias_hat[2]};
  const double w[3] = {omega[0] - p.bias_hat[3], omega[1] - p.bias_hat[4], omega[2] - p.bias_hat[5]};
  double xn[9], A[81], B[27], C[27];
  imu_step_jacobians(p.preintegrated, a, w, dt, xn, A, B, C);
  p.delta_t += dt;
  for (int e = 0; e < 9; e++) p.preintegrated[e] = xn[e];
  double Ha[27], Hw[27];
  for (int i = 0; i < 9; i++)
    for (int j = 0; j < 3; j++) {
      double sa = 0.0, sw = 0.0;
      for (int k = 0; k < 9; k++) {
        sa += A[i * 9 + k] * p.H_bias_acc[k * 3 + j];
        sw += A[i * 9 + k] * p.H_bias_omega[k * 3 + j];
      }
      Ha[i * 3 + j] = sa - B[i * 3 + j];
      Hw[i * 3 + j] = sw - C[i * 3 + j];
    }
  for (int e = 0; e < 27; e++) {
    p.H_bias_acc[e] = Ha[e];
    p.H_bias_omega[e] = Hw[e];
  }
  double AS[81];
  for (int i = 0; i < 9; i++)
    for (int j = 0; j < 9; j++) {
      double s = 0.0;
      for (int k = 0; k < 9; k++) s += A[i * 9 + k] * p.covariance[k * 9 + j];
      AS[i * 9 + j] = s;
    }
  const double qa = prm.acc_noise * prm.acc_noise / dt, qg = prm.gyro_noise * prm.gyro_noise / dt, qi = prm.int_noise * prm.int_noise * dt;
  for (int i = 0; i < 9; i++)
    for (int j = 0; j <= i; j++) {
      double s = 0.0, sb = 0.0, sc = 0.0;
      for (int k = 0; k < 9; k++) s += AS[i * 9 + k] * A[j * 9 + k];
      for (int k = 0; k < 3; k++) {
        sb += B[i * 3 + k] * B[j * 3 + k];
        sc += C[i * 3 + k] * C[j * 3 + k];
      }
      double v = s + qa * sb + qg * sc;
      if (i == j && i >= 3 && i < 6) v += qi;
      p.covariance[i * 9 + j] = v;
    }
  for (int i = 0; i < 9; i++)
    for (int j = i + 1; j < 9; j++) p.covariance[i * 9 + j] = p.covariance[j * 9 + i];
}

// The window of IMUIntegration::integrate_imu over S samples (rows t, a, w; non-decreasing t) for [start, end] at bias b_hat
GB_AHD void imu_preintegrate_interval(const double* samples, int S, double start, double end, const double* bias, const gb_imu_params& prm,
                                      gb_imu_preintegrated& p) {
  imu_reset(p, bias, prm);
  if (S <= 0) return;
  int lo = 0, hi = S;  // the first sample later than start: every earlier one has dt <= 0
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (samples[7 * (size_t)mid] > start) hi = mid;
    else lo = mid + 1;
  }
  double last = start;
  int i = lo;
  for (; i < S; i++) {
    const double* s = samples + 7 * (size_t)i;
    if (s[0] > end) break;
    const double dt = s[0] - last;
    if (dt <= 0.0) continue;
    imu_integrate(p, s + 1, s + 4, dt, prm);
    last = s[0];
    p.num_integrated++;
  }
  const double dt = end - last;
  if (dt > 0.0) {
    const double* s = samples + 7 * (size_t)(i < S ? i : S - 1);
    imu_integrate(p, s + 1, s + 4, dt, prm);
  }
}

// In place: the lower Cholesky factor of an n x n row-major symmetric matrix (upper triangle zeroed); false when a pivot is not
// positive or not finite
GB_AHD bool imu_cholesky(double* L, int n) {
  for (int j = 0; j < n; j++) {
    for (int i = j; i < n; i++) {
      double s = L[i * n + j];
      for (int k = 0; k < j; k++) s -= L[i * n + k] * L[j * n + k];
      if (i == j) {
        if (!(s > 0.0) || !(s < INFINITY)) return false;
        L[j * n + j] = sqrt(s);
      } else {
        L[i * n + j] = s / L[j * n + j];
      }
    }
    for (int i = 0; i < j; i++) L[i * n + j] = 0.0;
  }
  return true;
}

// The IMU term's residual r (9) and, when J is given, its Jacobian (9 x IMU_TERM_COLS, row-major) at pose_i Ti, velocity vi,
// pose_j Tj, velocity vj, bias bi [acc; gyro]
GB_AHD void imu_residual(const double* Ti, const double* vi, const double* Tj, const double* vj, const double* bi, const gb_imu_preintegrated& p,
                         double* r, double* J) {
  double d[9];
  for (int k = 0; k < 9; k++) {
    double s = p.preintegrated[k];
    for (int c = 0; c < 3; c++) s += p.H_bias_acc[k * 3 + c] * (bi[c] - p.bias_hat[c]) + p.H_bias_omega[k * 3 + c] * (bi[3 + c] - p.bias_hat[3 + c]);
    d[k] = s;
  }
  double Ri[9], Rjt[9], Ed[9];
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      Ri[a * 3 + b] = Ti[b * 4 + a];
      Rjt[b * 3 + a] = Tj[b * 4 + a];
    }
  imu_so3_exp(d, Ed);
  double RiE[9], E[9], RjRi[9];
  mat3_mul(Ri, Ed, RiE);
  mat3_mul(Rjt, RiE, E);
  mat3_mul(Rjt, Ri, RjRi);
  imu_so3_log(E, r);
  const double dt = p.delta_t, *g = p.gravity;
  double Rdp[3], Rdv[3], up[3], uv[3];
  mat3_vec(Ri, d + 3, Rdp);
  mat3_vec(Ri, d + 6, Rdv);
  for (int k = 0; k < 3; k++) {
    up[k] = Ti[12 + k] + vi[k] * dt + 0.5 * g[k] * dt * dt + Rdp[k] - Tj[12 + k];
    uv[k] = vi[k] + g[k] * dt + Rdv[k] - vj[k];
  }
  mat3_vec(Rjt, up, r + 3);
  mat3_vec(Rjt, uv, r + 6);
  if (!J) return;
  for (int e = 0; e < 9 * IMU_TERM_COLS; e++) J[e] = 0.0;
  double Jri[9], Jrd[9], Edt[9], Et[9], A0[9], A1[9], A2[9];
  imu_so3_jr(r, true, Jri);
  imu_so3_jr(d, false, Jrd);
  mat3_transpose(Ed, Edt);
  mat3_transpose(E, Et);
  mat3_mul(Jri, Edt, A0);  // d r_theta / d phi_i
  mat3_mul(Jri, Et, A1);   // -d r_theta / d phi_j
  mat3_mul(Jri, Jrd, A2);  // d r_theta / d delta_theta
  double Kp[9], Kv[9], Mp[9], Mv[9], Krp[9], Krv[9];
  mat3_hat(d + 3, Kp);
  mat3_hat(d + 6, Kv);
  mat3_mul(RjRi, Kp, Mp);
  mat3_mul(RjRi, Kv, Mv);
  mat3_hat(r + 3, Krp);
  mat3_hat(r + 6, Krv);
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) {
      double* Jt = J + a * IMU_TERM_COLS;
      double* Jp = J + (3 + a) * IMU_TERM_COLS;
      double* Jv = J + (6 + a) * IMU_TERM_COLS;
      Jt[b] = A0[a * 3 + b];
      Jt[12 + b] = -A1[a * 3 + b];
      Jp[b] = -Mp[a * 3 + b];
      Jp[3 + b] = RjRi[a * 3 + b];
      Jp[6 + b] = Rjt[a * 3 + b] * dt;
      Jp[12 + b] = Krp[a * 3 + b];
      Jp[15 + b] = a == b ? -1.0 : 0.0;
      Jv[b] = -Mv[a * 3 + b];
      Jv[6 + b] = Rjt[a * 3 + b];
      Jv[12 + b] = Krv[a * 3 + b];
      Jv[18 + b] = -Rjt[a * 3 + b];
    }
  for (int c = 0; c < 6; c++) {  // bias: d r / d delta times [H_bias_acc | H_bias_omega]
    const double* H = c < 3 ? p.H_bias_acc : p.H_bias_omega;
    const int cc = c % 3;
    for (int a = 0; a < 3; a++) {
      double st = 0.0, sp = 0.0, sv = 0.0;
      for (int k = 0; k < 3; k++) {
        st += A2[a * 3 + k] * H[k * 3 + cc];
        sp += RjRi[a * 3 + k] * H[(3 + k) * 3 + cc];
        sv += RjRi[a * 3 + k] * H[(6 + k) * 3 + cc];
      }
      J[a * IMU_TERM_COLS + 24 + c] = st;
      J[(3 + a) * IMU_TERM_COLS + 24 + c] = sp;
      J[(6 + a) * IMU_TERM_COLS + 24 + c] = sv;
    }
  }
}

// The vector term's residual (3 or 6 entries; returns the count) and, when J is given, its Jacobian (rows x 12, row-major,
// columns: the slot of key_a | the slot of key_b) at the states xa, xb (a pose as 4x4 column-major, a velocity 3, a bias 6)
GB_AHD int vector_residual(const gb_vector_term& m, const double* xa, const double* xb, double* r, double* J) {
  const int d = (m.kind == GB_VECTOR_BIAS_PRIOR || m.kind == GB_VECTOR_BIAS_BETWEEN) ? 6 : 3;
  if (J)
    for (int e = 0; e < 6 * 12; e++) J[e] = 0.0;
  if (m.kind == GB_VECTOR_ROTATE_VELOCITY) {
    double R[9], K[9], RK[9];
    for (int a = 0; a < 3; a++)
      for (int b = 0; b < 3; b++) R[a * 3 + b] = xa[b * 4 + a];
    mat3_vec(R, m.z, r);
    for (int k = 0; k < 3; k++) r[k] -= xb[k];
    if (J) {
      mat3_hat(m.z, K);
      mat3_mul(R, K, RK);
      for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++) J[a * 12 + b] = -RK[a * 3 + b];
        J[a * 12 + 6 + a] = -1.0;
      }
    }
    return 3;
  }
  const bool between = m.kind == GB_VECTOR_VELOCITY_BETWEEN || m.kind == GB_VECTOR_BIAS_BETWEEN;
  for (int k = 0; k < d; k++) {
    r[k] = (between ? xb[k] - xa[k] : xa[k]) - m.z[k];
    if (J) {
      J[k * 12 + k] = between ? -1.0 : 1.0;
      if (between) J[k * 12 + 6 + k] = 1.0;
    }
  }
  return d;
}

}  // namespace

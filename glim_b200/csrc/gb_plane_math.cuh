// gb_plane_math.cuh -- the arithmetic of the plane patch and of PlaneEVMFactor (gb_kernels_plane.cu), the rules of
// include/glim_b200.h ("plane bundle adjustment").  Like gb_cov_math.cuh it holds nothing that only exists on the device, so
// the same text compiles for the host: tests/cpp/plane_math_host.cpp builds it with g++ and tests/test_plane_ba_host.py checks
// it against the per-point restatement of tests/plane_ba_oracle.py.
//
// A key's moments are GB_PLANE_MOMENTS doubles {N, m (3), S (6: xx xy xz yy yz zz)}: its point count, the mean of its local
// points and their scatter about that mean.  Poses are 16 doubles, column-major: R(r, c) = X[4 c + r], t_r = X[12 + r].
#pragma once
#include "gb_cov_math.cuh"

#define GB_PLANE_MOMENTS 10
// per key, what the Hessian's blocks are made of (plane_evm_key): A (6), Y_1 (6), Y_2 (6), D (36, row-major)
#define GB_PLANE_KEY_TERMS 54

namespace {

// index of entry (r, c) of a symmetric 3x3 in the 6-vector xx xy xz yy yz zz
GB_CHD int sym6(int r, int c) {
  const int lo = r < c ? r : c, hi = r < c ? c : r;
  return lo == 0 ? hi : (lo == 1 ? 2 + hi : 5);
}

// The patch statistics of calc_eigenvalues from n points with s = sum q and S = sum q q^T (6): mean = s / n,
// Cov(r, c) = (S(r, c) - mean_r s_c) / n for r <= c, mirrored; eigenvalues ascending by eigen_sym3_direct.  n == 0 gives NaN.
GB_CHD void plane_stats(double n, const double* s, const double* S, double* ev) {
  if (!(n > 0.0)) {
    ev[0] = ev[1] = ev[2] = NAN;
    return;
  }
  double mean[3], A[9], V[9];
  for (int r = 0; r < 3; r++) mean[r] = s[r] / n;
  for (int r = 0; r < 3; r++)
    for (int c = r; c < 3; c++) A[3 * r + c] = A[3 * c + r] = __dsub_rn(S[sym6(r, c)], __dmul_rn(mean[r], s[c])) / n;
  eigen_sym3_direct(A, ev, V);
}

// q = R m + t - o of a key at pose X: row r as ((R_r0 m_0 + R_r1 m_1) + R_r2 m_2) + (t_r - o_r)
GB_CHD void plane_key_center(const double* X, const double* m, const double* o, double* q) {
  for (int r = 0; r < 3; r++) q[r] = ((X[r] * m[0] + X[4 + r] * m[1]) + X[8 + r] * m[2]) + (X[12 + r] - o[r]);
}

// C = (1/N) sum_k [R_k S_k R_k^T + N_k (q_k - pbar)(q_k - pbar)^T] (row-major) of K keys at poses X (K x 16), with
// pbar = (1/N) sum_k N_k q_k and N = sum_k N_k; the sums in key order.
GB_CHD void plane_evm_cov(int K, const double* mom, const double* X, const double* o, double* C, double* pbar, double* N_out) {
  double N = 0.0, sq[3] = {0.0, 0.0, 0.0};
  for (int k = 0; k < K; k++) {
    const double* M = mom + GB_PLANE_MOMENTS * k;
    double q[3];
    plane_key_center(X + 16 * k, M + 1, o, q);
    N += M[0];
    for (int r = 0; r < 3; r++) sq[r] += M[0] * q[r];
  }
  for (int r = 0; r < 3; r++) pbar[r] = sq[r] / N;
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < K; k++) {
    const double* M = mom + GB_PLANE_MOMENTS * k;
    const double* R = X + 16 * k;
    double q[3], d[3], RS[9];
    plane_key_center(R, M + 1, o, q);
    for (int r = 0; r < 3; r++) d[r] = q[r] - pbar[r];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) RS[3 * r + c] = (R[r] * M[4 + sym6(0, c)] + R[4 + r] * M[4 + sym6(1, c)]) + R[8 + r] * M[4 + sym6(2, c)];
    for (int r = 0; r < 3; r++)
      for (int c = r; c < 3; c++) {
        const double rsr = (RS[3 * r] * R[c] + RS[3 * r + 1] * R[4 + c]) + RS[3 * r + 2] * R[8 + c];
        acc[sym6(r, c)] += rsr + M[0] * d[r] * d[c];
      }
  }
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) C[3 * r + c] = acc[sym6(r, c)] / N;
  *N_out = N;
}

GB_CHD void plane_cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// S v for the 6-vector S
GB_CHD void plane_sym_mul(const double* S, const double* v, double* out) {
  for (int r = 0; r < 3; r++) out[r] = (S[sym6(r, 0)] * v[0] + S[sym6(r, 1)] * v[1]) + S[sym6(r, 2)] * v[2];
}

// The terms of key k (moments M, pose X) given the factor's pbar, N and eigenvectors U (U[3 r + j] = u_j), with
// v_j = R^T u_j and gamma_j = u_j . (q - pbar):
//   A = N_k [m x v_0; v_0]
//   Y_j = [m x c_j + (S v_0) x v_j + (S v_j) x v_0; c_j], c_j = N_k (gamma_0 v_j + gamma_j v_0)   (j = 1, 2)
//   D = (2/N) (N_k [m x v_0; v_0][m x v_0; v_0]^T + [[-hat(v_0) S hat(v_0), 0], [0, 0]])
//       + [[(1/N)(v_0 w^T + w v_0^T) - (2/N)(v_0 . w) I, -(N_k gamma_0 / N) hat(v_0)], [(N_k gamma_0 / N) hat(v_0), 0]],
//       w = N_k gamma_0 m + S v_0 (the last bracket is the second-order term of Exp)
//   g = de/dxi_k = (2/N) [N_k gamma_0 m x v_0 + (S v_0) x v_0; N_k gamma_0 v_0]
// written to T (GB_PLANE_KEY_TERMS) and g (6).  The Hessian of e is then, block (k, l),
//   delta_kl D_k - (2/N^2) A_k A_l^T + (2/N^2) sum_j Y_jk Y_jl^T / (lambda_0 - lambda_j).
GB_CHD void plane_evm_key(const double* M, const double* X, const double* o, const double* pbar, double N, const double* U, double* T, double* g) {
  const double Nk = M[0];
  const double* m = M + 1;
  const double* S = M + 4;
  double q[3], d[3], v[3][3], gam[3];
  plane_key_center(X, m, o, q);
  for (int r = 0; r < 3; r++) d[r] = q[r] - pbar[r];
  for (int j = 0; j < 3; j++) {
    for (int c = 0; c < 3; c++) v[j][c] = (X[4 * c] * U[j] + X[4 * c + 1] * U[3 + j]) + X[4 * c + 2] * U[6 + j];
    gam[j] = (U[j] * d[0] + U[3 + j] * d[1]) + U[6 + j] * d[2];
  }
  const double* v0 = v[0];
  double mxv[3], Sv0[3], Sv0xv0[3];
  plane_cross(m, v0, mxv);
  plane_sym_mul(S, v0, Sv0);
  plane_cross(Sv0, v0, Sv0xv0);
  for (int r = 0; r < 3; r++) {
    T[r] = Nk * mxv[r];
    T[3 + r] = Nk * v0[r];
  }
  for (int j = 1; j < 3; j++) {
    double c[3], mxc[3], a[3], Svj[3], b[3];
    for (int r = 0; r < 3; r++) c[r] = Nk * (gam[0] * v[j][r] + gam[j] * v0[r]);
    plane_cross(m, c, mxc);
    plane_cross(Sv0, v[j], a);
    plane_sym_mul(S, v[j], Svj);
    plane_cross(Svj, v0, b);
    double* Y = T + 6 * j;
    for (int r = 0; r < 3; r++) {
      Y[r] = (mxc[r] + a[r]) + b[r];
      Y[3 + r] = c[r];
    }
  }
  const double z[6] = {mxv[0], mxv[1], mxv[2], v0[0], v0[1], v0[2]};
  double* D = T + 18;
  for (int r = 0; r < 6; r++)
    for (int c = 0; c < 6; c++) D[6 * r + c] = 2.0 / N * Nk * z[r] * z[c];
  // -hat(v) S hat(v): column c of hat(v) is e_c x v ... written as (e_r x v)^T S (e_c x v)
  double hv[3][3];  // hv[c] = hat(v0) e_c = v0 x e_c
  for (int c = 0; c < 3; c++) {
    const double e[3] = {c == 0 ? 1.0 : 0.0, c == 1 ? 1.0 : 0.0, c == 2 ? 1.0 : 0.0};
    plane_cross(v0, e, hv[c]);
  }
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      double Sh[3];
      plane_sym_mul(S, hv[c], Sh);
      D[6 * r + c] += 2.0 / N * ((hv[r][0] * Sh[0] + hv[r][1] * Sh[1]) + hv[r][2] * Sh[2]);
    }
  const double ng = Nk * gam[0];
  double w[3];
  for (int r = 0; r < 3; r++) w[r] = ng * m[r] + Sv0[r];
  const double vw = (v0[0] * w[0] + v0[1] * w[1]) + v0[2] * w[2];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) D[6 * r + c] += (v0[r] * w[c] + w[r] * v0[c]) / N - (r == c ? 2.0 / N * vw : 0.0);
  // hat(v0)(r, c) = (v0 x e_c)_r
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      D[6 * r + 3 + c] -= ng / N * hv[c][r];
      D[6 * (3 + r) + c] += ng / N * hv[c][r];
    }
  for (int r = 0; r < 3; r++) {
    g[r] = 2.0 / N * (ng * mxv[r] + Sv0xv0[r]);
    g[3 + r] = 2.0 / N * ng * v0[r];
  }
}

// entry (i, j) of H = (1/2) d2e/dxi2 (both in 0 .. 6K) from the keys' terms (K x GB_PLANE_KEY_TERMS)
GB_CHD double plane_evm_entry(int i, int j, const double* terms, double N, const double* ev) {
  const int k = i / 6, a = i % 6, l = j / 6, b = j % 6;
  const double* Tk = terms + GB_PLANE_KEY_TERMS * k;
  const double* Tl = terms + GB_PLANE_KEY_TERMS * l;
  const double s = 2.0 / (N * N);
  double h = s * (Tk[6 + a] * Tl[6 + b] / (ev[0] - ev[1]) + Tk[12 + a] * Tl[12 + b] / (ev[0] - ev[2])) - s * Tk[a] * Tl[b];
  if (k == l) h += Tk[18 + 6 * a + b];
  return 0.5 * h;
}

// the status rule: degenerate iff !(lambda_1 - lambda_0 > 0)
GB_CHD bool plane_evm_degenerate(const double* ev) { return !(ev[1] - ev[0] > 0.0); }

}  // namespace

// Host build of gb_imu_preintegrate's and gb_nav_graph_optimize's arithmetic (glim_b200/csrc/gb_imu_math.cuh and
// gb_pose_graph_math.cuh -- the SAME text k_imu_preintegrate and k_pose_graph_step / k_pose_graph_accept compile, here with one
// thread, no barrier and scalar tile products): one preintegration step, the window, the IMU and vector terms, and a
// navigation graph's assembly and round structure (terms, assembly, damped copy, tiled Cholesky, retraction, conclude).
// TEST INFRASTRUCTURE: built by tests/test_imu_host.py with g++ and compared with numpy and tests/imu_oracle.py /
// tests/nav_graph_oracle.py on the CPU-only box; nothing in the product links it.
#include <string.h>

#include <vector>

#include "../../glim_b200/csrc/gb_pose_graph_math.cuh"

namespace {
struct NoSync {
  void operator()() const {}
};

struct HostTiles {
  double* A;
  double* x;
  int N;
  bool potrf(int kt) {
    int flag = 0;
    return pg_potrf_tile(A + (size_t)kt * PG_TILE * (N + 1), N, 0, 1, NoSync{}, &flag);
  }
  void panel(int kt) {
    for (int R = (kt + 1) * PG_TILE; R < N; R++) pg_trsm_row(A + (size_t)R * N + kt * PG_TILE, A + (size_t)kt * PG_TILE * (N + 1), N);
  }
  void trailing(int kt) {
    const int m = N / PG_TILE - 1 - kt;
    for (long long t = 0; t < (long long)m * (m + 1) / 2; t++) {
      int i, j;
      pg_tri(t, &i, &j);
      pg_tile_update(A, N, kt + 1 + i, kt + 1 + j, kt);
    }
  }
  void trsv(int kt, bool backward) { pg_trsv_tile(A + (size_t)kt * PG_TILE * (N + 1), N, x + kt * PG_TILE, backward, 0, 1, NoSync{}); }
  void rows(int kt, bool backward) {
    for (int R = pg_rows_begin(kt, backward); R < pg_rows_end(kt, N, backward); R++) pg_substitute_row(A, N, kt, x, R, backward);
  }
  void sync() {}
};

// Everything one navigation graph without factors holds, as the device carves it.  X: K slots x 16 (poses, velocities, biases).
struct Host {
  PoseGraphCall c{};
  std::vector<int> keys, cptr, qptr, qidx;
  std::vector<GraphContrib> contrib;
  std::vector<double> brec, prec, bterm, pterm, nrec, nterm, nchol, Tn, H, b, A, x, steps;
  AlignState st;
  int ok = 0;
  Host(int KX, int KV, int KB, int B, const gb_between_term* bt, int Q, const int* pkeys, const double* pposes, const double* pw, int NI, const gb_imu_term* it,
       int NV, const gb_vector_term* vt, const int* nslots, double* X) {
    const int K = KX + KV + KB, n = 6 * K, N = pg_padded(n);
    keys.assign(2 * (size_t)B, 0);
    for (int m = 0; m < B; m++) {
      keys[2 * m] = bt[m].key_i;
      keys[2 * m + 1] = bt[m].key_j;
    }
    cptr.resize(graph_num_blocks(K) + 1);
    contrib.resize(5 * (size_t)B + 20 * (size_t)(NI + NV));
    graph_contributions(K, B, keys.data(), 0, cptr.data(), contrib.data(), NI + NV, nslots);
    qptr.resize(K + 1);
    qidx.resize(Q);
    pg_prior_index(K, Q, pkeys, qptr.data(), qidx.data());
    brec.assign(122 * (size_t)B, 0.0);
    prec.assign(PG_PRIOR_DOUBLES * (size_t)Q, 0.0);
    bterm.assign(B, 0.0);
    pterm.assign(Q, 0.0);
    nrec.assign(PG_NAV_DOUBLES * (size_t)(NI + NV), 0.0);
    nterm.assign(NI + NV, 0.0);
    nchol.assign(81 * (size_t)NI, 0.0);
    for (int m = 0; m < NI; m++) {
      for (int e = 0; e < 81; e++) nchol[81 * (size_t)m + e] = it[m].pim.covariance[e];
      imu_cholesky(nchol.data() + 81 * (size_t)m, 9);
    }
    Tn.assign(X, X + 16 * K);
    H.assign((size_t)n * n, 0.0);
    b.assign(n, 0.0);
    A.assign((size_t)N * N, 0.0);
    x.assign(N, 0.0);
    steps.assign(2 * K, 0.0);
    c.K = K; c.n = n; c.N = N; c.F = 0; c.B = B; c.Q = Q;
    c.cptr = cptr.data(); c.contrib = contrib.data(); c.qptr = qptr.data(); c.qidx = qidx.data(); c.fkeys = keys.data();
    c.bt = bt; c.pkeys = pkeys; c.pposes = pposes; c.pw = pw;
    c.brec = brec.data(); c.prec = prec.data(); c.bterm = bterm.data(); c.pterm = pterm.data();
    c.T = X; c.Tn = Tn.data(); c.H = H.data(); c.b = b.data(); c.A = A.data(); c.x = x.data(); c.steps = steps.data();
    c.ok = &ok; c.st = &st;
    c.KV = KV; c.KB = KB; c.NI = NI; c.NV = NV; c.it = it; c.vt = vt; c.nslots = nslots; c.nrec = nrec.data(); c.nterm = nterm.data();
    c.nchol = nchol.data();
  }
  bool solve(double lambda) {
    pg_damped_copy(c, lambda, 0, 1);
    HostTiles g{c.A, c.x, c.N};
    return pg_cholesky_solve(g, c.N);
  }
};
}  // namespace

// one step of the tangent preintegration at x with bias-corrected a, w: xn (9), A (9x9), B, C (9x3), row-major
extern "C" void imh_step(const double* x, const double* a, const double* w, double dt, double* xn, double* A, double* B, double* C) {
  imu_step_jacobians(x, a, w, dt, xn, A, B, C);
}

// the window of one interval
extern "C" void imh_preintegrate(const double* samples, int S, double start, double end, const double* bias, const gb_imu_params* prm, gb_imu_preintegrated* out) {
  imu_preintegrate_interval(samples, S, start, end, bias, *prm, *out);
}

// the IMU term's residual (9) and Jacobian (9 x 30); poses column-major
extern "C" void imh_imu_residual(const double* Ti, const double* vi, const double* Tj, const double* vj, const double* b, const gb_imu_preintegrated* p, double* r,
                                 double* J) {
  imu_residual(Ti, vi, Tj, vj, b, *p, r, J);
}

// a vector term's residual (returns its length) and Jacobian (rows x 12)
extern "C" int imh_vector_residual(const gb_vector_term* m, const double* xa, const double* xb, double* r, double* J) { return vector_residual(*m, xa, xb, r, J); }

// the system of a navigation graph without factors at the slot states X (K x 16): H (n x n, lower blocks), b (n), the terms'
// records nrec ((NI + NV) x PG_NAV_DOUBLES) and the damped padded copy A (N x N) and x (N) at lambda
extern "C" void imh_nav_assemble(int KX, int KV, int KB, int B, const gb_between_term* bt, int Q, const int* pkeys, const double* pposes, const double* pw, int NI,
                                 const gb_imu_term* it, int NV, const gb_vector_term* vt, const int* nslots, double* X, double lambda, double* H, double* b,
                                 double* nrec, double* A, double* x, double* e) {
  Host h(KX, KV, KB, B, bt, Q, pkeys, pposes, pw, NI, it, NV, vt, nslots, X);
  align_init(h.st, X, 1e-5);
  pg_terms_at(h.c, 0, 1);
  pg_assemble(h.c, 0, 1);
  pg_linearized(h.c);
  pg_damped_copy(h.c, lambda, 0, 1);
  memcpy(H, h.H.data(), sizeof(double) * h.H.size());
  memcpy(b, h.b.data(), sizeof(double) * h.b.size());
  memcpy(nrec, h.nrec.data(), sizeof(double) * h.nrec.size());
  memcpy(A, h.A.data(), sizeof(double) * h.A.size());
  memcpy(x, h.x.data(), sizeof(double) * h.x.size());
  *e = h.st.e;
}

// One navigation graph without factors driven through the device's round structure.  X (K x 16) in: the initial slot states,
// out: the result.
extern "C" int imh_nav_optimize(const gb_align_params* prm, int KX, int KV, int KB, int B, const gb_between_term* bt, int Q, const int* pkeys, const double* pposes,
                                const double* pw, int NI, const gb_imu_term* it, int NV, const gb_vector_term* vt, const int* nslots, double* X, gb_graph_result* r) {
  Host h(KX, KV, KB, B, bt, Q, pkeys, pposes, pw, NI, it, NV, vt, nslots, X);
  align_init(h.st, X, prm->lambda_initial);
  while (h.st.status == GB_ALIGN_ACTIVE) {
    if (h.st.need_lin) {
      pg_terms_at(h.c, 0, 1);
      pg_assemble(h.c, 0, 1);
      pg_linearized(h.c);
      if (h.st.status != GB_ALIGN_ACTIVE) break;
    }
    const bool solved = h.solve(h.st.lambda);
    pg_retract(h.c, solved, 0, 1, NoSync{});
    if (pg_conclude(h.c, *prm)) pg_accept_rows(h.c, 0, 1, NoSync{});
  }
  align_result(h.st, *r);
  return 0;
}

// Host build of gb_pose_graph_optimize's arithmetic (glim_b200/csrc/gb_pose_graph_math.cuh -- the SAME text k_pose_graph_step /
// k_pose_graph_accept compile, here with one thread, no barrier and scalar tile products) and of its round structure:
// linearize -> terms, assembly, damped copy, tiled Cholesky, retraction -> error -> conclude / accept rows.
// TEST INFRASTRUCTURE: built by tests/test_pose_graph_host.py with g++ and compared with numpy and tests/pose_graph_oracle.py on
// the CPU-only box; nothing in the product links it.
#include <string.h>

#include <vector>

#include "../../glim_b200/csrc/gb_pose_graph_math.cuh"

namespace {
struct NoSync {
  void operator()() const {}
};

// The tile steps on one host thread: the diagonal tile and the panels in place, scalar tile products
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

// Everything one call holds, as the device carves it
struct Host {
  PoseGraphCall c{};
  std::vector<int> keys, cptr, qptr, qidx;
  std::vector<GraphContrib> contrib;
  std::vector<double> brec, prec, bterm, pterm, Tn, H, b, A, x, steps, poses, poses_eval;
  AlignState st;
  int ok = 0;
  Host(int K, int F, const int* fkeys, int B, const gb_between_term* bt, int Q, const int* pkeys, const double* pposes, const double* pw, double* T, const double* out) {
    const int n = 6 * K, N = pg_padded(n);
    keys.assign(2 * (size_t)(F + B), 0);
    for (int f = 0; f < 2 * F; f++) keys[f] = fkeys[f];
    for (int m = 0; m < B; m++) {
      keys[2 * (F + m)] = bt[m].key_i;
      keys[2 * (F + m) + 1] = bt[m].key_j;
    }
    cptr.resize(graph_num_blocks(K) + 1);
    contrib.resize(5 * (size_t)(F + B));
    graph_contributions(K, F + B, keys.data(), 0, cptr.data(), contrib.data());
    qptr.resize(K + 1);
    qidx.resize(Q);
    pg_prior_index(K, Q, pkeys, qptr.data(), qidx.data());
    brec.assign(122 * (size_t)B, 0.0);
    prec.assign(PG_PRIOR_DOUBLES * (size_t)Q, 0.0);
    bterm.assign(B, 0.0);
    pterm.assign(Q, 0.0);
    Tn.assign(T, T + 16 * K);
    H.assign((size_t)n * n, 0.0);
    b.assign(n, 0.0);
    A.assign((size_t)N * N, 0.0);
    x.assign(N, 0.0);
    steps.assign(2 * K, 0.0);
    poses.assign(16 * (size_t)F, 0.0);
    poses_eval.assign(16 * (size_t)F, 0.0);
    c = PoseGraphCall{K, n, N, F, B, Q, cptr.data(), contrib.data(), qptr.data(), qidx.data(), keys.data(), bt, pkeys, pposes, pw,
                      brec.data(), prec.data(), bterm.data(), pterm.data(), T, Tn.data(), H.data(), b.data(), A.data(), x.data(), steps.data(),
                      &ok, &st, poses.data(), poses_eval.data(), out};
  }
  bool solve(double lambda) {
    pg_damped_copy(c, lambda, 0, 1);
    HostTiles g{c.A, c.x, c.N};
    return pg_cholesky_solve(g, c.N);
  }
};
}  // namespace

// the between term's error and (when rec is not null) its 122-double record
extern "C" double pgm_between(const double* Ti, const double* Tj, const gb_between_term* m, double* rec) { return pg_between_term(Ti, Tj, *m, rec); }

// (H + lambda I) d = -b for an n x n row-major H (lower triangle read) through the padded tiled schedule; 1 on success
extern "C" int pgm_solve(int n, const double* H, const double* b, double lambda, double* d) {
  const int K = (n + 5) / 6;
  std::vector<double> T(16 * (size_t)K, 0.0);
  Host h(K, 0, nullptr, 0, nullptr, 0, nullptr, nullptr, nullptr, T.data(), nullptr);
  h.c.n = n;  // any n: the solve reads only n, N, H, b, A and x
  h.c.N = pg_padded(n);
  h.A.assign((size_t)h.c.N * h.c.N, 0.0);
  h.x.assign(h.c.N, 0.0);
  h.c.A = h.A.data();
  h.c.x = h.x.data();
  h.c.H = const_cast<double*>(H);
  h.c.b = const_cast<double*>(b);
  if (!h.solve(lambda)) return 0;
  for (int i = 0; i < n; i++) d[i] = h.x[i];
  return 1;
}

// the system at poses T (K x 16) of F records (F x 122, local keys F x 2), B between terms and Q priors; brec (B x 122) and prec
// (Q x 43) receive the terms' records, H (n x n, lower blocks) and b (n) the sums
extern "C" void pgm_assemble(int K, int F, const int* fkeys, const double* records, int B, const gb_between_term* bt, int Q, const int* pkeys,
                             const double* pposes, const double* pw, double* T, double* H, double* b, double* brec, double* prec) {
  Host h(K, F, fkeys, B, bt, Q, pkeys, pposes, pw, T, records);
  pg_terms_at(h.c, 0, 1);
  pg_assemble(h.c, 0, 1);
  memcpy(H, h.H.data(), sizeof(double) * h.H.size());
  memcpy(b, h.b.data(), sizeof(double) * h.b.size());
  memcpy(brec, h.brec.data(), sizeof(double) * h.brec.size());
  memcpy(prec, h.prec.data(), sizeof(double) * h.prec.size());
}

// One graph driven through the device's round structure (lin / err as tests/cpp/graph_math_host.cpp's).  T (K x 16) in:
// T_init, out: the result.  dt, dr: the last trial's step.
typedef void (*lin_fn)(const double* rows, double* records);
typedef void (*err_fn)(const double* rows_lin, const double* rows_eval, double* records);
extern "C" int pgm_optimize(const gb_align_params* prm, int K, int F, const int* fkeys, int B, const gb_between_term* bt, int Q, const int* pkeys,
                            const double* pposes, const double* pw, double* T, lin_fn lin, err_fn err, gb_graph_result* r, double* dt, double* dr) {
  std::vector<double> out(122 * (size_t)F, 0.0);
  Host h(K, F, fkeys, B, bt, Q, pkeys, pposes, pw, T, out.data());
  align_init(h.st, T, prm->lambda_initial);
  for (int f = 0; f < F; f++) graph_row(T, fkeys[2 * f], fkeys[2 * f + 1], h.poses.data() + 16 * f);
  while (h.st.status == GB_ALIGN_ACTIVE) {
    if (h.st.need_lin) {
      if (F > 0) lin(h.poses.data(), out.data());
      pg_terms_at(h.c, 0, 1);
      pg_assemble(h.c, 0, 1);
      pg_linearized(h.c);
      if (h.st.status != GB_ALIGN_ACTIVE) break;
    }
    const bool solved = h.solve(h.st.lambda);
    pg_retract(h.c, solved, 0, 1, NoSync{});
    if (F > 0) err(h.poses.data(), h.poses_eval.data(), out.data());
    if (pg_conclude(h.c, *prm)) pg_accept_rows(h.c, 0, 1, NoSync{});
  }
  align_result(h.st, *r);
  *dt = h.st.dt;
  *dr = h.st.dr;
  return 0;
}

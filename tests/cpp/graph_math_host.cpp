// Host build of gb_graph_optimize's per-problem arithmetic (glim_b200/csrc/gb_graph_math.cuh -- the SAME text k_graph_step /
// k_graph_accept compile, here with one thread and no barrier) and of its round structure for one problem:
// linearize -> graph_step -> error -> graph_conclude / graph_accept_rows.
// TEST INFRASTRUCTURE: built by tests/test_graph_host.py with g++ and compared with numpy and tests/graph_oracle.py on the
// CPU-only box; nothing in the product links it.
#include <string.h>

#include <vector>

#include "../../glim_b200/csrc/gb_graph_math.cuh"

namespace {
struct NoSync {
  void operator()() const {}
};
}  // namespace

// (H + lambda I) d = -b for an n x n row-major H through the packed solve; 1 on success
extern "C" int gm_solve(int n, const double* H, const double* b, double lambda, double* d) {
  std::vector<double> A(graph_packed_size(n));
  for (int i = 0; i < n; i++) {
    for (int j = 0; j <= i; j++) A[i * (i + 1) / 2 + j] = H[i * n + j] + (i == j ? lambda : 0.0);
    d[i] = -b[i];
  }
  int flag = 0;
  return graph_cholesky_solve(A.data(), d, n, 0, 1, NoSync{}, &flag) ? 1 : 0;
}

// the system (H n x n with its lower blocks and diagonal blocks written, b n) of F records (F x 122) at local keys (F x 2)
extern "C" void gm_assemble(int K, int F, const int* keys, const double* records, double* H, double* b) {
  std::vector<int> cptr(graph_num_blocks(K) + 1);
  std::vector<GraphContrib> contrib(5 * (size_t)F);
  graph_contributions(K, F, keys, 0, cptr.data(), contrib.data());
  graph_assemble(records, cptr.data(), contrib.data(), K, H, b, 0, 1, NoSync{});
}

// se3_prior_term with its 6x6 block (row-major) and 6-vector, both added to
extern "C" double gm_prior(const double* T, const double* Z, double w, double* H, double* b) { return se3_prior_term(T, Z, w, H, 6, b); }

// One problem driven through the device's round structure.  lin(rows F x 16, records F x 122) linearizes every factor at its
// row T_t^-1 T_s; err(rows_lin, rows_eval, records) writes each factor's error at rows_eval with the inliers of rows_lin into
// records[f * 122 + 120].  T (K x 16) in: T_init, out: the result.  dt, dr: the last trial's step.
typedef void (*lin_fn)(const double* rows, double* records);
typedef void (*err_fn)(const double* rows_lin, const double* rows_eval, double* records);
extern "C" int gm_optimize(const gb_align_params* prm, int K, int F, const int* keys, int Q, const int* pkeys, const double* pposes, const double* pw,
                           double* T, lin_fn lin, err_fn err, gb_graph_result* r, double* dt, double* dr) {
  const int n = 6 * K;
  GraphProblem g{K, n, 0, 0, F, 0, Q, 0, 0, 0};
  std::vector<int> cptr(graph_num_blocks(K) + 1);
  std::vector<GraphContrib> contrib(5 * (size_t)F);
  graph_contributions(K, F, keys, 0, cptr.data(), contrib.data());
  std::vector<double> Tn(T, T + 16 * K), sys((size_t)n * n + n), pterm(Q), poses(16 * (size_t)F), poses_eval(16 * (size_t)F), out(122 * (size_t)F, 0.0);
  std::vector<double> smem(graph_smem_doubles(n));
  GraphState st;
  align_init(st.a, T, prm->lambda_initial);
  GraphCall c{&g, &st, cptr.data(), contrib.data(), keys, pkeys, pposes, pw, pterm.data(), T, Tn.data(), sys.data(), poses.data(), poses_eval.data(), out.data()};
  for (int f = 0; f < F; f++) graph_row(T, keys[2 * f], keys[2 * f + 1], poses.data() + 16 * f);
  int flag = 0;
  while (st.a.status == GB_ALIGN_ACTIVE) {
    if (st.a.need_lin) lin(poses.data(), out.data());
    graph_step(c, 0, smem.data(), 0, 1, NoSync{}, &flag);
    if (st.a.status != GB_ALIGN_ACTIVE) break;
    err(poses.data(), poses_eval.data(), out.data());
    if (graph_conclude(c, 0, *prm)) graph_accept_rows(c, 0, 0, 1, NoSync{});
  }
  align_result(st.a, *r);
  *dt = st.a.dt;
  *dr = st.a.dr;
  return 0;
}

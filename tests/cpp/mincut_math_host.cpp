// Host build of the min-cut segmentation's per-node arithmetic (glim_b200/csrc/gb_mincut_math.cuh, the text k_mc_nodes,
// k_mc_graph and k_mc_solve compile) and a sequential driver of k_mc_solve's synchronous rounds: the same initialisation,
// global relabels (exact distances to the seed, here by a queue) and push / relabel steps, in node order.
// tests/test_mincut_host.py compiles this with g++ -ffp-contract=off and compares it with scipy (tests/mincut_oracle.py).
#include "../../glim_b200/csrc/gb_mincut_math.cuh"

#include <deque>
#include <vector>

extern "C" {

// out[i] = mc_edge_capacity of rows i of the fp32 positions / normals (n x 3 each)
void edge_capacity(int n, const float* pa, const float* na, const float* pb, const float* nb, double s2d, double s2a, int* out) {
  for (int i = 0; i < n; i++) {
    const float *a = pa + 3 * i, *an = na + 3 * i, *b = pb + 3 * i, *bn = nb + 3 * i;
    out[i] = mc_edge_capacity(a[0], a[1], a[2], an[0], an[1], an[2], b[0], b[1], b[2], bn[0], bn[1], bn[2], s2d, s2a);
  }
}

// out[i] = mc_role of fp32 point i (n x 3) against the fp64 picked point c
void roles(int n, const float* xyz, const double* c, double fg2, double bg2, int* out) {
  for (int i = 0; i < n; i++) out[i] = mc_role(mc_d2(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], c[0], c[1], c[2]), fg2, bg2);
}

// The solve of k_mc_solve on m nodes (row: m + 1 CSR offsets; head, rev, cap per arc; role per node, one MC_SEED), run
// sequentially with at most max_rounds rounds.  sel[u] = 1 for the selected nodes; *cut = the flow; *rounds; returns
// GB_MINCUT_FOUND (0) or GB_MINCUT_NOT_CONVERGED (2).
int solve(int m, const int* row, const int* head, const int* rev, const int* cap, const int* role, int fg_cap, int max_rounds, int* sel, long long* cut,
          int* rounds_out) {
  const int A = row[m], H = m + 2;
  int seed = -1;
  for (int u = 0; u < m; u++)
    if (role[u] == MC_SEED) seed = u;
  std::vector<int> res(A > 0 ? A : 1), fg_res(m), h(m), hn(m);
  std::vector<long long> e(m, 0), incoming(m, 0);
  for (int u = 0; u < m; u++) {
    fg_res[u] = role[u] == MC_FOREGROUND ? fg_cap : 0;
    for (int a = row[u]; a < row[u + 1]; a++) {
      res[a] = mc_initial_residual(role[u], role[head[a]], cap[a]);
      if (role[u] == MC_BACKGROUND && role[head[a]] != MC_BACKGROUND) e[head[a]] += cap[a];
    }
  }
  const auto inner = [&](int u) { return role[u] == MC_FREE || role[u] == MC_FOREGROUND; };
  const auto global_relabel = [&]() {
    for (int u = 0; u < m; u++) h[u] = u == seed ? 0 : H;
    std::deque<int> q{seed};
    while (!q.empty()) {
      const int v = q.front();
      q.pop_front();
      if (v == seed)
        for (int u = 0; u < m; u++)
          if (role[u] == MC_FOREGROUND && fg_res[u] > 0 && h[u] == H) {
            h[u] = 1;
            q.push_back(u);
          }
      for (int a = row[v]; a < row[v + 1]; a++) {
        const int u = head[a];
        if (h[u] == H && role[u] != MC_BACKGROUND && res[rev[a]] > 0) {
          h[u] = h[v] + 1;
          q.push_back(u);
        }
      }
    }
  };
  const auto active = [&]() {
    int x = 0;
    for (int u = 0; u < m; u++) x += inner(u) && h[u] < H && e[u] > 0;
    return x;
  };
  int rounds = 0;
  global_relabel();
  int act = active();
  while (act > 0 && rounds < max_rounds) {
    rounds++;
    for (int u = 0; u < m; u++)
      if (inner(u) && h[u] < H && e[u] > 0) e[u] = mc_push_node(u, e[u], row, head, rev, res.data(), fg_res.data(), h.data(), incoming.data(), seed);
    act = 0;
    for (int u = 0; u < m; u++) {
      int hu = h[u];
      if (inner(u) && hu < H && e[u] > 0) hu = mc_relabel_node(u, role[u], row, head, res.data(), fg_res.data(), h.data(), H);
      hn[u] = hu;
      e[u] += incoming[u];
      incoming[u] = 0;
      act += inner(u) && hu < H && e[u] > 0;
    }
    h.swap(hn);
    if (act > 0 && rounds % kMcRelabelPeriod == 0) {
      global_relabel();
      act = active();
    }
  }
  *rounds_out = rounds;
  for (int u = 0; u < m; u++) sel[u] = 0;
  *cut = 0;
  if (act > 0) return 2;
  global_relabel();
  for (int u = 0; u < m; u++) sel[u] = h[u] < H && role[u] != MC_BACKGROUND ? 1 : 0;
  *cut = e[seed];
  return 0;
}

int max_rounds() { return kMcMaxRounds; }

}  // extern "C"

// gb_mincut_math.cuh -- the per-node arithmetic of the map editor's min-cut segmentation (gb_min_cut, gb_kernels_segment.cu),
// kept free of anything that only exists on the device so that the SAME TEXT also compiles for the host:
// tests/cpp/mincut_math_host.cpp builds it with g++ -ffp-contract=off, drives the same synchronous rounds sequentially and
// tests/test_mincut_host.py checks it against scipy's maximum flow (tests/mincut_oracle.py).  The rule is written once, in
// include/glim_b200.h.
//
// The solve is push-relabel with the roles swapped: the background participants are the (contracted) source, at height
// H = m + 2, the seed is the sink, at height 0, and every other node is free or foreground.  A foreground node's arc
// to the seed is kept beside the CSR as fg_res[i] (its residual).  Each round is a push step (every active node pushes along
// its admissible arcs in CSR order, the foreground arc first; received excess goes to `incoming`) and, after a barrier, a
// relabel step (incoming folded in; a node that was active and still holds excess takes min over its residual arcs of the
// old height + 1).  A push only ever goes downhill, so the two arcs of an edge have one writer per step, and the integer
// additions into `incoming` commute: the rounds are the same in any order the nodes are visited.
#pragma once
#include "gb_segment_math.cuh"  // GB_HD, seg_seed_key, the fp64 intrinsics' host shims

namespace {

enum { MC_FREE = 0, MC_FOREGROUND = 1, MC_BACKGROUND = 2, MC_SEED = 3 };
constexpr int kMcMaxRounds = 65536;    // the round cap of the solve: NOT_CONVERGED beyond it
constexpr int kMcRelabelPeriod = 16;   // a global relabel (exact distances to the seed) after every this many rounds
constexpr double kMcScale = 65536.0;   // capacities are floor(w * 2^16)

// fp64 (dx^2 + dy^2) + dz^2 of two points, each operation rounded
GB_HD double mc_d2(double ax, double ay, double az, double bx, double by, double bz) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// The role of a participant other than the seed from its fp64 d2 to the picked point: foreground inside the foreground
// radius (fg2 = r_f^2), background beyond the background radius (bg2 = r_b^2), free between.
GB_HD int mc_role(double d2, double fg2, double bg2) { return d2 < fg2 ? MC_FOREGROUND : (d2 > bg2 ? MC_BACKGROUND : MC_FREE); }

// The capacity of edge {i, j}: floor(2^16 exp(-d2 / s2d) exp(-theta^2 / s2a)) with s2d = 2 sigma_d^2, s2a = 2 sigma_a^2,
// d2 the fp64 d2 of the fp32 positions and theta = acos(min(|n_i . n_j|, 1)), the dot (x + y) + z in fp64 from the fp32
// normals.  0 for a NaN dot or a zero normal.  The same in both directions, bit for bit.
GB_HD int mc_edge_capacity(float ax, float ay, float az, float anx, float any, float anz, float bx, float by, float bz, float bnx, float bny, float bnz,
                           double s2d, double s2a) {
  if ((anx == 0.f && any == 0.f && anz == 0.f) || (bnx == 0.f && bny == 0.f && bnz == 0.f)) return 0;
  const double dot = __dadd_rn(__dadd_rn(__dmul_rn((double)anx, (double)bnx), __dmul_rn((double)any, (double)bny)), __dmul_rn((double)anz, (double)bnz));
  if (isnan(dot)) return 0;
  const double c = fmin(fabs(dot), 1.0);
  const double th = acos(c);
  const double d2 = mc_d2(ax, ay, az, bx, by, bz);
  const double w = __dmul_rn(exp(-(d2 / s2d)), exp(-(__dmul_rn(th, th) / s2a)));
  return (int)floor(__dmul_rn(w, kMcScale));
}

GB_HD void mc_add(long long* a, long long v) {
#ifdef __CUDACC__
  atomicAdd((unsigned long long*)a, (unsigned long long)v);
#else
  *a += v;
#endif
}

// The push step of active node u (free or foreground, excess ex > 0, height h[u] below the source's): along the foreground
// arc (admissible at h[u] == 1) and then along every arc a of row u in CSR order that is admissible (res[a] > 0 and
// h[u] == h[head[a]] + 1), min(excess left, res[a]) each.  Receivers get their share in incoming[] (the seed's is the flow);
// returns the excess left.  Only u writes its arcs' residuals and their reverses in a step: no other node can push along
// them, since it would have to stand one above u while u stands one above it.
GB_HD long long mc_push_node(int u, long long ex, const int* row, const int* head, const int* rev, int* res, int* fg_res, const int* h, long long* incoming, int seed) {
  const int hu = h[u];
  if (hu == 1 && fg_res[u] > 0) {
    const int d = ex < fg_res[u] ? (int)ex : fg_res[u];
    fg_res[u] -= d;
    mc_add(&incoming[seed], d);
    ex -= d;
  }
  for (int a = row[u]; a < row[u + 1] && ex > 0; a++) {
    const int v = head[a];
    if (hu != h[v] + 1) continue;  // the height first: an uphill arc's residual may be written by v in this step
    const int r = res[a];
    if (r <= 0) continue;
    const int d = ex < r ? (int)ex : r;
    res[a] = r - d;
    res[rev[a]] += d;
    mc_add(&incoming[v], d);
    ex -= d;
  }
  return ex;
}

// The relabel of a node that was active and still holds excess after the push step: min over its residual arcs of the
// old height of the head + 1 (the foreground arc's head is the seed, at 0), capped at H (no residual arc: H).
GB_HD int mc_relabel_node(int u, int role_u, const int* row, const int* head, const int* res, const int* fg_res, const int* h_old, int H) {
  int best = H;
  if (role_u == MC_FOREGROUND && fg_res[u] > 0) best = 1;
  for (int a = row[u]; a < row[u + 1]; a++)
    if (res[a] > 0 && h_old[head[a]] + 1 < best) best = h_old[head[a]] + 1;
  return best;
}

// The initial residual of arc (u, v) of capacity q: every arc out of a background node into the rest is saturated (its
// reverse holds 2q), arcs between two background nodes and between two other nodes keep q.
GB_HD int mc_initial_residual(int role_u, int role_v, int q) {
  const bool bu = role_u == MC_BACKGROUND, bv = role_v == MC_BACKGROUND;
  return bu == bv ? q : (bu ? 0 : 2 * q);
}

}  // namespace

// gb_graph_math.cuh -- the per-problem arithmetic of gb_graph_optimize (gb_graph.cu): the assembly of the 6K x 6K system from
// the factors' records, the priors, the packed Cholesky solve, the retraction of every key, and the two halves of a round
// (graph_step, graph_accept) around the error sweep.  The accept / terminate rule is gb_vgicp_align's (align_conclude), the
// prior term gb_ct_gicp_align's (se3_prior_term).  Like gb_align_math.cuh it holds nothing that only exists on the device: the
// loops that a CTA shares are strided over (tid, nthreads) with a barrier hook, so the SAME TEXT compiles for the host with
// (0, 1, no-op): tests/cpp/graph_math_host.cpp builds it with g++ and tests/test_graph_host.py checks it against numpy and the
// rule's restatement in tests/graph_oracle.py.
// Poses are 4x4 column-major doubles, tangent order [rot; trans]; the system is ROW-major, keys in problem order.
#pragma once
#include "gb_ct_math.cuh"  // se3_prior_term, ct_inverse; through gb_align_math.cuh: AlignState, align_exp, align_compose, align_step_norms, align_conclude

namespace {

// Everything the host derives once per call for one problem.  Its keys are rows [key0, key0 + K) of the pose arrays, its
// factors records [f0, f1), its priors [q0, q1); its system is n * n + n doubles of scratch at sys (H row-major, then b).
struct GraphProblem {
  int K, n;
  int key0;
  int f0, f1;
  int q0, q1;
  int cp0;         // its block CSR: cptr[cp0 .. cp0 + graph_num_blocks(K)]
  int pad;
  long long sys;
};

// One contribution of a record to the system: factor (global record index) and role (GB_GRAPH_H_TT ... GB_GRAPH_B_S).
struct GraphContrib {
  int factor, role;
};
enum { GB_GRAPH_H_TT = 0, GB_GRAPH_H_SS, GB_GRAPH_H_TS, GB_GRAPH_H_ST, GB_GRAPH_B_T, GB_GRAPH_B_S, GB_GRAPH_NAV_H, GB_GRAPH_NAV_B = GB_GRAPH_NAV_H + 25 };

// What the rule keeps for one problem between rounds: the scalars of gb_vgicp_align's state (a.T, a.Tn, a.H and a.b unused;
// the poses live in the call's T / Tn arrays).
struct GraphState {
  AlignState a;
};

// The blocks of a K-key system: the lower-triangle 6x6 blocks (i >= j) at i (i + 1) / 2 + j, then the 6-vector of key i at
// K (K + 1) / 2 + i.
GB_AHD int graph_num_blocks(int K) { return K * (K + 1) / 2 + K; }
GB_AHD int graph_block(int i, int j) { return i * (i + 1) / 2 + j; }
GB_AHD int graph_packed_size(int n) { return n * (n + 1) / 2; }

// The contributions of F factors (problem-local keys[2f] = target, keys[2f + 1] = source, target != source) to the blocks of a
// K-key system, grouped by block and in record order within each: block k gathers contrib[cptr[k] .. cptr[k + 1]).  Each
// factor adds H_tt to (t, t), H_ss to (s, s), H_ts to (t, s) -- stored as its transpose in the lower block (s, t) when t < s
// -- and b_t, b_s to t, s: five contributions.  f_base is the record index of the first factor.  The R records that follow
// (record index f_base + F + m) touch up to five distinct keys each, rslots[5 m ..] (-1 past the last): slot pair (a, b) adds
// its block to the lower block of its keys (role GB_GRAPH_NAV_H + 5 a + b, key of a >= key of b) and slot a its vector
// (GB_GRAPH_NAV_B + a).  A counting sort: cptr must hold graph_num_blocks(K) + 1 entries, contrib 5 F + 20 R.
GB_AHD void graph_contributions(int K, int F, const int* keys, int f_base, int* cptr, GraphContrib* contrib, int R = 0, const int* rslots = nullptr) {
  const int nb = graph_num_blocks(K), tri = K * (K + 1) / 2;
  for (int k = 0; k <= nb; k++) cptr[k] = 0;
  for (int pass = 0; pass < 2; pass++) {
    for (int f = 0; f < F; f++) {
      const int t = keys[2 * f], s = keys[2 * f + 1];
      const int blk[5] = {graph_block(t, t), graph_block(s, s), t > s ? graph_block(t, s) : graph_block(s, t), tri + t, tri + s};
      const int role[5] = {GB_GRAPH_H_TT, GB_GRAPH_H_SS, t > s ? GB_GRAPH_H_TS : GB_GRAPH_H_ST, GB_GRAPH_B_T, GB_GRAPH_B_S};
      for (int c = 0; c < 5; c++) {
        if (pass == 0) cptr[blk[c] + 1]++;
        else contrib[cptr[blk[c]]++] = GraphContrib{f_base + f, role[c]};
      }
    }
    for (int m = 0; m < R; m++) {
      const int* sl = rslots + 5 * (size_t)m;
      for (int a = 0; a < 5 && sl[a] >= 0; a++)
        for (int b = 0; b <= 5; b++) {
          if (b < 5 && (sl[b] < 0 || sl[b] > sl[a])) continue;
          const int blk = b < 5 ? graph_block(sl[a], sl[b]) : tri + sl[a];
          if (pass == 0) cptr[blk + 1]++;
          else contrib[cptr[blk]++] = GraphContrib{f_base + F + m, b < 5 ? GB_GRAPH_NAV_H + 5 * a + b : GB_GRAPH_NAV_B + a};
        }
    }
    if (pass == 0)
      for (int k = 0; k < nb; k++) cptr[k + 1] += cptr[k];
  }
  for (int k = nb; k > 0; k--) cptr[k] = cptr[k - 1];  // the fill advanced every start to the next block's
  cptr[0] = 0;
}

// entry (r, c) of a contribution, from the F x 122 records (gb_linearized6: H_tt | H_ss | H_ts column-major, b_t, b_s)
GB_AHD double graph_entry(const double* out, GraphContrib x, int r, int c) {
  const double* rec = out + (size_t)x.factor * 122;
  switch (x.role) {
    case GB_GRAPH_H_TT: return rec[c * 6 + r];
    case GB_GRAPH_H_SS: return rec[36 + c * 6 + r];
    case GB_GRAPH_H_TS: return rec[72 + c * 6 + r];
    case GB_GRAPH_H_ST: return rec[72 + r * 6 + c];
    case GB_GRAPH_B_T: return rec[108 + r];
    default: return rec[114 + r];
  }
}

// H (n x n row-major, its lower-triangle blocks and full diagonal blocks written) and b (n) of a K-key system: every entry the
// sum of its contributions in record order, from 0.0.  Ends with a barrier.
template <class Sync>
GB_AHD void graph_assemble(const double* out, const int* cptr, const GraphContrib* contrib, int K, double* H, double* b, int tid, int nt, Sync sync) {
  const int n = 6 * K, tri = K * (K + 1) / 2, nb = graph_num_blocks(K);
  for (int x = tid; x < nb * 36; x += nt) {
    const int k = x / 36, r = (x % 36) / 6, c = x % 6;
    if (k >= tri && c != 0) continue;
    double s = 0.0;
    for (int m = cptr[k]; m < cptr[k + 1]; m++) s += graph_entry(out, contrib[m], r, c);
    if (k >= tri) {
      b[6 * (k - tri) + r] = s;
    } else {
      int i = 0;
      while ((i + 1) * (i + 2) / 2 <= k) i++;
      const int j = k - i * (i + 1) / 2;
      H[(size_t)(6 * i + r) * n + 6 * j + c] = s;
    }
  }
  sync();
}

// e plus each prior's w |Log(Z_q^-1 T_k)|^2 in prior order, at the poses T (K x 16); when H is given each prior's Jacobian terms
// go into its key's diagonal block of the n x n system (H, b).
GB_AHD double graph_priors(const double* T, const int* pkeys, const double* pposes, const double* pw, int q0, int q1, int n, double e, double* H, double* b) {
  for (int q = q0; q < q1; q++) {
    const int k = pkeys[q];
    e += se3_prior_term(T + 16 * k, pposes + 16 * q, pw[q], H ? H + (size_t)(6 * k) * n + 6 * k : nullptr, n, H ? b + 6 * k : nullptr);
  }
  return e;
}

// In place: A holds the packed lower triangle (row i at i (i + 1) / 2) of an n x n symmetric matrix, x holds -b.  Left-looking
// Cholesky A = L L^T column by column (each column's dot products in ascending k, as align_solve), then L y = x and L^T d = y;
// x holds d on success.  Every thread returns the same value: false when a pivot is not positive (or not finite).  *flag is
// shared by the threads (a __shared__ int on the device).
template <class Sync>
GB_AHD bool graph_cholesky_solve(double* A, double* x, int n, int tid, int nt, Sync sync, int* flag) {
  for (int j = 0; j < n; j++) {
    double* Lj = A + j * (j + 1) / 2;
    if (tid == 0) {
      double s = Lj[j];
      for (int k = 0; k < j; k++) s -= Lj[k] * Lj[k];
      *flag = (s > 0.0) && (s < INFINITY);
      Lj[j] = *flag ? sqrt(s) : 0.0;
    }
    sync();
    if (!*flag) return false;
    for (int i = j + 1 + tid; i < n; i += nt) {
      double* Li = A + i * (i + 1) / 2;
      double s = Li[j];
      for (int k = 0; k < j; k++) s -= Li[k] * Lj[k];
      Li[j] = s / Lj[j];
    }
    sync();
  }
  for (int j = 0; j < n; j++) {  // forward: x_i = (x_i - sum_{k < i} L_ik x_k) / L_ii, subtracted in ascending k
    if (tid == 0) x[j] /= A[j * (j + 1) / 2 + j];
    sync();
    for (int i = j + 1 + tid; i < n; i += nt) x[i] -= A[i * (i + 1) / 2 + j] * x[j];
    sync();
  }
  for (int i = n - 1; i >= 0; i--) {  // backward, with L^T's column i = L's row i
    const double* Li = A + i * (i + 1) / 2;
    if (tid == 0) x[i] /= Li[i];
    sync();
    for (int m = tid; m < i; m += nt) x[m] -= Li[m] * x[i];
    sync();
  }
  return true;
}

// the sweep's pose row of a factor: T_t^-1 T_s
GB_AHD void graph_row(const double* T, int t, int s, double* row) {
  double Ti[16];
  ct_inverse(T + 16 * t, Ti);
  align_compose(Ti, T + 16 * s, row);
}

// Device pointers (or host arrays) of one call.
struct GraphCall {
  const GraphProblem* prob;
  GraphState* st;
  const int* cptr;
  const GraphContrib* contrib;  // 5 per factor: problem p's from 5 f0 on, its block CSR relative to there
  const int* fkeys;      // F x 2, problem-local (target, source)
  const int* pkeys;      // Q, problem-local
  const double* pposes;  // Q x 16
  const double* pw;      // Q
  double* pterm;         // Q: each prior's term at the trial poses
  double* T;             // sum K x 16: the current poses
  double* Tn;            // sum K x 16: the trial poses
  double* sys;           // the problems' systems
  double* poses;         // F x 16: the sweep's linearization rows, T_t^-1 T_s
  double* poses_eval;    // F x 16: the sweep's evaluation rows
  const double* out;     // F x 122: the sweep's records
};

// The shared memory of graph_step for n unknowns: the packed factor, the right-hand side and the per-key steps.
GB_AHD size_t graph_smem_doubles(int n) { return (size_t)graph_packed_size(n) + n + 2 * GB_GRAPH_MAX_KEYS; }

// Rule steps 1-2 and the priors of step 3 for problem p, by nt threads sharing smem (graph_smem_doubles) and *flag: on a fresh
// linearization the system into the problem's scratch (the error sweep that follows overwrites the records) with the priors
// at T; then (H + lambda I) d = -b, T'_k = T_k Exp(d_k), each prior's term at T', and each factor's evaluation row.
template <class Sync>
GB_AHD void graph_step(const GraphCall& c, int p, double* smem, int tid, int nt, Sync sync, int* flag) {
  const GraphProblem& g = c.prob[p];
  AlignState& s = c.st[p].a;
  if (s.status != GB_ALIGN_ACTIVE) return;
  const int n = g.n, K = g.K;
  double* H = c.sys + g.sys;
  double* b = H + (size_t)n * n;
  const double* T = c.T + 16 * (size_t)g.key0;
  double* Tn = c.Tn + 16 * (size_t)g.key0;
  if (s.need_lin) {
    graph_assemble(c.out, c.cptr + g.cp0, c.contrib + 5 * (size_t)g.f0, K, H, b, tid, nt, sync);
    if (tid == 0) {
      double e = 0.0, m = 0.0;
      for (int f = g.f0; f < g.f1; f++) {
        e += c.out[(size_t)f * 122 + 120];
        m += c.out[(size_t)f * 122 + 121];
      }
      s.e = graph_priors(T, c.pkeys, c.pposes, c.pw, g.q0, g.q1, n, e, H, b);
      s.n = m;
      align_linearized(s);
    }
    sync();
    if (s.status != GB_ALIGN_ACTIVE) return;
  }
  double* A = smem;
  double* x = A + graph_packed_size(n);
  double* dt = x + n;
  double* dr = dt + GB_GRAPH_MAX_KEYS;
  const double lambda = s.lambda;
  for (int k = tid; k < n * n; k += nt) {
    const int i = k / n, j = k % n;
    if (j <= i) A[i * (i + 1) / 2 + j] = H[k] + (i == j ? lambda : 0.0);
  }
  for (int i = tid; i < n; i += nt) x[i] = -b[i];
  sync();
  const bool solved = graph_cholesky_solve(A, x, n, tid, nt, sync, flag);
  for (int k = tid; k < K; k += nt) {
    if (solved) {
      double E[16];
      align_exp(x + 6 * k, E);
      align_compose(T + 16 * k, E, Tn + 16 * k);
      align_step_norms(E, x + 6 * k, dt + k, dr + k);
    } else {
      for (int e = 0; e < 16; e++) Tn[16 * k + e] = T[16 * k + e];
    }
  }
  sync();
  if (tid == 0) {
    s.trials += 1;
    s.solved = solved ? 1 : 0;
    s.dt = 0.0;
    s.dr = 0.0;
    if (solved)
      for (int k = 0; k < K; k++) {
        s.dt = dt[k] > s.dt ? dt[k] : s.dt;
        s.dr = dr[k] > s.dr ? dr[k] : s.dr;
      }
  }
  for (int q = g.q0 + tid; q < g.q1; q += nt) c.pterm[q] = se3_prior_term(Tn + 16 * c.pkeys[q], c.pposes + 16 * q, c.pw[q], nullptr, 0, nullptr);
  for (int f = g.f0 + tid; f < g.f1; f += nt) graph_row(Tn, c.fkeys[2 * f], c.fkeys[2 * f + 1], c.poses_eval + 16 * (size_t)f);
}

// Rule steps 3-5 for problem p (one thread): e' = the factors' errors at T' in record order, then each prior's term in prior
// order; align_conclude.  Returns whether the trial was accepted (graph_accept_rows follows).
GB_AHD bool graph_conclude(const GraphCall& c, int p, const gb_align_params& prm) {
  const GraphProblem& g = c.prob[p];
  AlignState& s = c.st[p].a;
  double e = 0.0;
  for (int f = g.f0; f < g.f1; f++) e += c.out[(size_t)f * 122 + 120];
  for (int q = g.q0; q < g.q1; q++) e += c.pterm[q];
  align_conclude(s, prm, e);
  return s.need_lin != 0;
}

// An accepted trial: T = T' and every factor's linearization row at the new poses, by nt threads.  Ends with a barrier.
template <class Sync>
GB_AHD void graph_accept_rows(const GraphCall& c, int p, int tid, int nt, Sync sync) {
  const GraphProblem& g = c.prob[p];
  double* T = c.T + 16 * (size_t)g.key0;
  const double* Tn = c.Tn + 16 * (size_t)g.key0;
  for (int k = tid; k < 16 * g.K; k += nt) T[k] = Tn[k];
  sync();
  for (int f = g.f0 + tid; f < g.f1; f += nt) graph_row(T, c.fkeys[2 * f], c.fkeys[2 * f + 1], c.poses + 16 * (size_t)f);
  sync();
}

}  // namespace

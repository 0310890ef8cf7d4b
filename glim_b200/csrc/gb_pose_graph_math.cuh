// gb_pose_graph_math.cuh -- the arithmetic of gb_pose_graph_optimize (gb_pose_graph.cu): the between term, the assembly of the
// 6K x 6K system from the factors' records, the between terms and the priors, the damped padded copy, the tiled Cholesky's
// per-tile steps and its schedule, the blocked substitution, and the two halves of a round around the error sweep; with
// gb_nav_graph_optimize's velocity and bias slots, IMU and vector terms (gb_imu_math.cuh) in the same code.  The accept
// / terminate rule is gb_vgicp_align's (align_conclude), the prior term gb_ct_gicp_align's (se3_prior_term), the block CSR and
// the pose rows gb_graph_optimize's (graph_contributions, graph_row).  Like gb_graph_math.cuh it holds nothing that only exists
// on the device: the loops a grid or a CTA shares are strided over (tid, nthreads) with a barrier hook, and the tile schedule
// takes its tile steps from a policy, so the SAME TEXT compiles for the host with (0, 1, no-op) and scalar tile products:
// tests/cpp/pose_graph_math_host.cpp builds it with g++ and tests/test_pose_graph_host.py checks it against numpy and the rule's
// restatement in tests/pose_graph_oracle.py.
// Poses are 4x4 column-major doubles, tangent order [rot; trans]; H is ROW-major n x n (its lower 6x6 blocks written), the
// factor A ROW-major N x N with N = n rounded up to PG_TILE (its lower tiles used).
#pragma once
#include "gb_graph_math.cuh"  // GraphContrib, graph_contributions, graph_num_blocks, graph_row; through gb_ct_math.cuh: se3_prior_term, ct_*
#include "gb_imu_math.cuh"    // imu_residual, imu_cholesky, vector_residual

#define PG_TILE 64
#define PG_PRIOR_DOUBLES 43  // a prior's record: its 6x6 block (row-major) | its 6-vector | its error
#define PG_NAV_DOUBLES 931   // an IMU or vector term's record over its (up to 5) slots: H 30 x 30 row-major | b 30 | its error
// a loop the device compiler keeps rolled: the between term's 6x6 products, fully unrolled, hold more doubles than a thread has
// registers
#ifdef __CUDA_ARCH__
#define PG_ROLLED _Pragma("unroll 1")
#else
#define PG_ROLLED
#endif
// a function the device calls out of line: an IMU term's 9 x 30 Jacobian inlined into the step kernel would spill its registers
#ifdef __CUDACC__
#define PG_OUT_OF_LINE __host__ __device__ __noinline__
#else
#define PG_OUT_OF_LINE static inline
#endif

namespace {

// i, j (j <= i) of entry k of a row-major packed lower triangle: k = i (i + 1) / 2 + j, without a search
GB_AHD void pg_tri(long long k, int* i, int* j) {
  int r = (int)((sqrt(8.0 * (double)k + 1.0) - 1.0) * 0.5);
  while ((long long)r * (r + 1) / 2 > k) r--;
  while ((long long)(r + 1) * (r + 2) / 2 <= k) r++;
  *i = r;
  *j = (int)(k - (long long)r * (r + 1) / 2);
}

GB_AHD int pg_padded(int n) { return (n + PG_TILE - 1) / PG_TILE * PG_TILE; }

// The between term of m at poses T_i, T_j: its error 2 rho(|r|_L) and, when rec is given, its record in the layout of the
// sweep's (gb_linearized6: H_ii | H_jj | H_ij column-major, b_i, b_j, error, 0 inliers) with t = i, s = j.
GB_AHD double pg_between_term(const double* Ti, const double* Tj, const gb_between_term& m, double* rec) {
  double Tinv[16], D[16], Zi[16], E[16], r[6];
  ct_inverse(Ti, Tinv);
  align_compose(Tinv, Tj, D);
  ct_inverse(m.Z, Zi);
  align_compose(Zi, D, E);
  ct_log(E, r);
  double Lr[6], m2 = 0.0;
  for (int a = 0; a < 6; a++) {
    double s = 0.0;
    for (int c = 0; c < 6; c++) s += m.information[c * 6 + a] * r[c];
    Lr[a] = s;
    m2 += r[a] * s;
  }
  const double mah = sqrt(m2 > 0.0 ? m2 : 0.0), k = m.huber_width;
  const bool robust = k > 0.0 && mah > k;
  const double w = robust ? k / mah : 1.0;
  const double err = robust ? 2.0 * k * mah - k * k : m2;
  if (!rec) return err;
  double Jj[36], Di[16], Ad[36], Ji[36];
  ct_se3_jr(r, true, Jj);
  ct_inverse(D, Di);
  ct_adjoint(Di, Ad);
  ct_mul6(Jj, Ad, Ji);
  for (int e = 0; e < 36; e++) Ji[e] = -Ji[e];
  double LJi[36], LJj[36];  // L J (row-major)
  PG_ROLLED
  for (int a = 0; a < 6; a++)
    for (int c = 0; c < 6; c++) {
      double si = 0.0, sj = 0.0;
      for (int q = 0; q < 6; q++) {
        si += m.information[q * 6 + a] * Ji[q * 6 + c];
        sj += m.information[q * 6 + a] * Jj[q * 6 + c];
      }
      LJi[a * 6 + c] = si;
      LJj[a * 6 + c] = sj;
    }
  PG_ROLLED
  for (int a = 0; a < 6; a++) {
    for (int c = 0; c < 6; c++) {
      double hii = 0.0, hjj = 0.0, hij = 0.0;
      for (int q = 0; q < 6; q++) {
        hii += Ji[q * 6 + a] * LJi[q * 6 + c];
        hjj += Jj[q * 6 + a] * LJj[q * 6 + c];
        hij += Ji[q * 6 + a] * LJj[q * 6 + c];
      }
      rec[c * 6 + a] = w * hii;
      rec[36 + c * 6 + a] = w * hjj;
      rec[72 + c * 6 + a] = w * hij;
    }
    double bi = 0.0, bj = 0.0;
    for (int q = 0; q < 6; q++) {
      bi += Ji[q * 6 + a] * Lr[q];
      bj += Jj[q * 6 + a] * Lr[q];
    }
    rec[108 + a] = w * bi;
    rec[114 + a] = w * bj;
  }
  rec[120] = err;
  rec[121] = 0.0;
  return err;
}

// A prior's record at pose T: its block and vector as se3_prior_term adds them to zeros, and its error
GB_AHD void pg_prior_record(const double* T, const double* Z, double w, double* rec) {
  for (int e = 0; e < 42; e++) rec[e] = 0.0;
  rec[42] = se3_prior_term(T, Z, w, rec, 6, rec + 36);
}

// The priors grouped by key, in prior order within a key: key k's are qidx[qptr[k] .. qptr[k + 1]).  qptr holds K + 1.
GB_AHD void pg_prior_index(int K, int Q, const int* qkeys, int* qptr, int* qidx) {
  for (int k = 0; k <= K; k++) qptr[k] = 0;
  for (int q = 0; q < Q; q++) qptr[qkeys[q] + 1]++;
  for (int k = 0; k < K; k++) qptr[k + 1] += qptr[k];
  for (int q = 0; q < Q; q++) qidx[qptr[qkeys[q]]++] = q;
  for (int k = K; k > 0; k--) qptr[k] = qptr[k - 1];
  qptr[0] = 0;
}

// Device pointers (or host arrays) of one call.  The block CSR (cptr, contrib) is graph_contributions' over the F factors'
// keys followed by the B between terms' (key_i as target, key_j as source), then the NI IMU terms' and NV vector terms' slots:
// a contribution's record index f < F reads the sweep's records, f < F + B the between records, the rest the nav records.
// The K slots hold the poses, then KV velocities, then KB biases (each slot 16 doubles of T / Tn: a pose's 4x4, a velocity's 3
// or a bias's 6 leading entries); KV = KB = NI = NV = 0 is gb_pose_graph_optimize's graph.
struct PoseGraphCall {
  int K, n, N;  // keys, 6K, n padded to PG_TILE
  int F, B, Q;
  const int* cptr;
  const GraphContrib* contrib;
  const int* qptr;
  const int* qidx;
  const int* fkeys;               // F x 2 (target, source)
  const gb_between_term* bt;      // B
  const int* pkeys;               // Q
  const double* pposes;           // Q x 16
  const double* pw;               // Q
  double* brec;                   // B x 122: the between terms at T
  double* prec;                   // Q x PG_PRIOR_DOUBLES: the priors at T
  double* bterm;                  // B: the between errors at T'
  double* pterm;                  // Q: the prior errors at T'
  double* T;                      // K x 16: the current poses
  double* Tn;                     // K x 16: the trial poses
  double* H;                      // n x n: the last linearization's system
  double* b;                      // n
  double* A;                      // N x N: the damped factor
  double* x;                      // N: -b, then the step
  double* steps;                  // 2 K: each key's translation and rotation step
  int* ok;                        // the factorization's verdict, shared by the grid
  AlignState* st;
  double* poses;                  // F x 16: the sweep's linearization rows
  double* poses_eval;             // F x 16: the sweep's evaluation rows
  const double* out;              // F x 122: the sweep's records
  int KV, KB;                     // velocity and bias slots
  int NI, NV;                     // IMU terms, vector terms
  const gb_imu_term* it;          // NI
  const gb_vector_term* vt;       // NV
  const int* nslots;              // (NI + NV) x 5: each term's slots, -1 past its last
  double* nrec;                   // (NI + NV) x PG_NAV_DOUBLES: the terms at T
  double* nterm;                  // NI + NV: the terms' errors at T'
  const double* nchol;            // NI x 81: the lower Cholesky factor of each IMU record's covariance, factored by the host
};

GB_AHD int pg_num_poses(const PoseGraphCall& c) { return c.K - c.KV - c.KB; }

// A dead dof: the last three of a velocity slot
GB_AHD bool pg_pinned(const PoseGraphCall& c, int i) {
  const int v0 = 6 * pg_num_poses(c), v1 = 6 * (c.K - c.KB);
  return i >= v0 && i < v1 && i % 6 >= 3;
}

// IMU or vector term m (IMU terms first) at the slot states X: its error and, when rec is given, its record.  An IMU term is
// whitened by the Cholesky factor L of its covariance (r^T S^-1 r = |L^-1 r|^2), the one the host factored when it validated
// the record; a vector term weighs w.
PG_OUT_OF_LINE double pg_nav_term(const PoseGraphCall& c, int m, const double* X, double* rec) {
  const int* sl = c.nslots + 5 * (size_t)m;
  double J[9 * IMU_TERM_COLS], r[9], w = 1.0;
  int d, ld, cols;
  if (m < c.NI) {
    const gb_imu_preintegrated& p = c.it[m].pim;
    imu_residual(X + 16 * sl[0], X + 16 * sl[1], X + 16 * sl[2], X + 16 * sl[3], X + 16 * sl[4], p, r, rec ? J : nullptr);
    const double* L = c.nchol + 81 * (size_t)m;
    d = 9;
    ld = cols = IMU_TERM_COLS;
    for (int i = 0; i < 9; i++) {  // L y = r and L Y = J
      for (int k = 0; k < i; k++) r[i] -= L[i * 9 + k] * r[k];
      r[i] /= L[i * 9 + i];
      if (rec)
        for (int a = 0; a < cols; a++) {
          double s = J[i * ld + a];
          for (int k = 0; k < i; k++) s -= L[i * 9 + k] * J[k * ld + a];
          J[i * ld + a] = s / L[i * 9 + i];
        }
    }
  } else {
    const gb_vector_term& v = c.vt[m - c.NI];
    d = vector_residual(v, X + 16 * sl[0], sl[1] >= 0 ? X + 16 * sl[1] : nullptr, r, rec ? J : nullptr);
    w = v.precision;
    ld = 12;
    cols = sl[1] >= 0 ? 12 : 6;
  }
  double e = 0.0;
  for (int k = 0; k < d; k++) e += r[k] * r[k];
  e *= w;
  if (!rec) return e;
  PG_ROLLED
  for (int a = 0; a < cols; a++) {
    for (int b = 0; b <= a; b++) {
      double s = 0.0;
      for (int k = 0; k < d; k++) s += J[k * ld + a] * J[k * ld + b];
      rec[a * 30 + b] = rec[b * 30 + a] = w * s;
    }
    double s = 0.0;
    for (int k = 0; k < d; k++) s += J[k * ld + a] * r[k];
    rec[900 + a] = w * s;
  }
  rec[930] = e;
  return e;
}

GB_AHD double pg_entry(const PoseGraphCall& c, GraphContrib x, int r, int col) {
  if (x.factor < c.F) return graph_entry(c.out, x, r, col);
  if (x.factor < c.F + c.B) {
    GraphContrib y{x.factor - c.F, x.role};
    return graph_entry(c.brec, y, r, col);
  }
  const double* rec = c.nrec + (size_t)(x.factor - c.F - c.B) * PG_NAV_DOUBLES;
  if (x.role >= GB_GRAPH_NAV_B) return rec[900 + 6 * (x.role - GB_GRAPH_NAV_B) + r];
  const int a = (x.role - GB_GRAPH_NAV_H) / 5, b = (x.role - GB_GRAPH_NAV_H) % 5;
  return rec[(6 * a + r) * 30 + 6 * b + col];
}

// Rule step 1 before the sums: every between, prior, IMU and vector record at T, one term per thread.
GB_AHD void pg_terms_at(const PoseGraphCall& c, int tid, int nt) {
  for (int m = tid; m < c.B + c.Q + c.NI + c.NV; m += nt) {
    if (m < c.B) pg_between_term(c.T + 16 * c.bt[m].key_i, c.T + 16 * c.bt[m].key_j, c.bt[m], c.brec + 122 * (size_t)m);
    else if (m >= c.B + c.Q) {
      const int t = m - c.B - c.Q;
      pg_nav_term(c, t, c.T, c.nrec + PG_NAV_DOUBLES * (size_t)t);
    } else {
      const int q = m - c.B;
      pg_prior_record(c.T + 16 * c.pkeys[q], c.pposes + 16 * q, c.pw[q], c.prec + PG_PRIOR_DOUBLES * (size_t)q);
    }
  }
}

// The lower 6x6 blocks of H and b: every entry the sum of the factor records in record order, then the between terms, the IMU
// terms and the vector terms in term order (one CSR), then the priors of its key in prior order, from 0.0.  One entry per thread; a block's row and column come
// from its packed index, not from a search.
GB_AHD void pg_assemble(const PoseGraphCall& c, int tid, int nt) {
  const int K = c.K, n = c.n, tri = K * (K + 1) / 2;
  const long long total = (long long)graph_num_blocks(K) * 36;
  for (long long x = tid; x < total; x += nt) {
    const int k = (int)(x / 36), r = (int)(x % 36) / 6, col = (int)(x % 6);
    if (k >= tri && col != 0) continue;
    double s = 0.0;
    for (int m = c.cptr[k]; m < c.cptr[k + 1]; m++) s += pg_entry(c, c.contrib[m], r, col);
    if (k >= tri) {
      const int key = k - tri;
      for (int q = c.qptr[key]; q < c.qptr[key + 1]; q++) s += c.prec[PG_PRIOR_DOUBLES * (size_t)c.qidx[q] + 36 + r];
      c.b[6 * key + r] = s;
    } else {
      int i, j;
      pg_tri(k, &i, &j);
      if (i == j)
        for (int q = c.qptr[i]; q < c.qptr[i + 1]; q++) s += c.prec[PG_PRIOR_DOUBLES * (size_t)c.qidx[q] + r * 6 + col];
      c.H[(size_t)(6 * i + r) * n + 6 * j + col] = s;
    }
  }
}

// Rule step 1 after the sums (one thread): e and n in the stated order; DEGENERATE only for a graph with factors.
GB_AHD void pg_linearized(const PoseGraphCall& c) {
  AlignState& s = *c.st;
  double e = 0.0, m = 0.0;
  for (int f = 0; f < c.F; f++) {
    e += c.out[(size_t)f * 122 + 120];
    m += c.out[(size_t)f * 122 + 121];
  }
  for (int t = 0; t < c.B; t++) e += c.brec[(size_t)t * 122 + 120];
  for (int t = 0; t < c.NI + c.NV; t++) e += c.nrec[PG_NAV_DOUBLES * (size_t)t + 930];
  for (int q = 0; q < c.Q; q++) e += c.prec[PG_PRIOR_DOUBLES * (size_t)q + 42];
  s.e = e;
  s.n = m;
  s.iterations += 1;
  s.need_lin = 0;
  if (c.F > 0 && m == 0.0 && s.iterations == 1) s.status = GB_ALIGN_DEGENERATE;
}

// A = H + lambda I on the lower tiles (0 above the diagonal of a diagonal tile), a unit diagonal on the padded rows and the
// pinned velocity dofs (whose rows and columns of H are zero); x = -b, 0 on the padded rows and the pinned dofs.
GB_AHD void pg_damped_copy(const PoseGraphCall& c, double lambda, int tid, int nt) {
  const int n = c.n, N = c.N;
  for (long long e = tid; e < (long long)N * N; e += nt) {
    const int i = (int)(e / N), j = (int)(e % N);
    if (j / PG_TILE > i / PG_TILE) continue;
    double v = 0.0;
    if (j <= i) v = i < n && !pg_pinned(c, i) ? c.H[(size_t)i * n + j] + (i == j ? lambda : 0.0) : (i == j ? 1.0 : 0.0);
    c.A[e] = v;
  }
  for (int i = tid; i < N; i += nt) c.x[i] = i < n && !pg_pinned(c, i) ? -c.b[i] : 0.0;
}

// ---- the tile steps of the factorization and the substitution ----

// In place: the lower triangle of the PG_TILE x PG_TILE tile D (leading dimension ld) into its Cholesky factor, right-looking
// column by column.  Every thread returns the same value: false when a pivot is not positive (or not finite).  *flag is shared
// by the threads.
template <class Sync>
GB_AHD bool pg_potrf_tile(double* D, int ld, int tid, int nt, Sync sync, int* flag) {
  for (int j = 0; j < PG_TILE; j++) {
    if (tid == 0) {
      const double p = D[j * ld + j];
      *flag = (p > 0.0) && (p < INFINITY);
      D[j * ld + j] = *flag ? sqrt(p) : 0.0;
    }
    sync();
    if (!*flag) return false;
    const double d = D[j * ld + j];
    for (int i = j + 1 + tid; i < PG_TILE; i += nt) D[i * ld + j] /= d;
    sync();
    const int m = PG_TILE - 1 - j;
    for (int e = tid; e < m * m; e += nt) {
      const int i = j + 1 + e / m, k = j + 1 + e % m;
      if (k <= i) D[i * ld + k] -= D[i * ld + j] * D[k * ld + j];
    }
    sync();
  }
  return true;
}

// One row x (PG_TILE entries) of a panel tile: x := x L^-T with L the factored diagonal tile (leading dimension ld)
GB_AHD void pg_trsm_row(double* x, const double* L, int ld) {
  for (int c = 0; c < PG_TILE; c++) {
    double s = x[c];
    for (int m = 0; m < c; m++) s -= x[m] * L[c * ld + m];
    x[c] = s / L[c * ld + c];
  }
}

// The trailing update of tile (it, jt) by tile column kt with scalar products: A_it,jt -= L_it,kt L_jt,kt^T, each entry's
// products subtracted in ascending k (the device takes these products on the fp64 tensor cores)
GB_AHD void pg_tile_update(double* A, int N, int it, int jt, int kt) {
  for (int r = 0; r < PG_TILE; r++)
    for (int col = 0; col < PG_TILE; col++) {
      const double* a = A + (size_t)(it * PG_TILE + r) * N + kt * PG_TILE;
      const double* bb = A + (size_t)(jt * PG_TILE + col) * N + kt * PG_TILE;
      double* cc = A + (size_t)(it * PG_TILE + r) * N + jt * PG_TILE + col;
      double s = *cc;
      for (int k = 0; k < PG_TILE; k++) s -= a[k] * bb[k];
      *cc = s;
    }
}

// The diagonal tile's triangular solve in place on x (PG_TILE entries): L y = x (forward) or L^T y = x (backward), column by
// column, by nt threads
template <class Sync>
GB_AHD void pg_trsv_tile(const double* L, int ld, double* x, bool backward, int tid, int nt, Sync sync) {
  for (int s = 0; s < PG_TILE; s++) {
    const int c = backward ? PG_TILE - 1 - s : s;
    if (tid == 0) x[c] /= L[c * ld + c];
    sync();
    if (backward)
      for (int r = tid; r < c; r += nt) x[r] -= L[c * ld + r] * x[c];
    else
      for (int r = c + 1 + tid; r < PG_TILE; r += nt) x[r] -= L[r * ld + c] * x[c];
    sync();
  }
}

// Row R's update by the solved block kt: forward x_R -= L_R,kt x_kt; backward x_R -= L_kt,R^T x_kt
GB_AHD void pg_substitute_row(const double* A, int N, int kt, double* x, int R, bool backward) {
  double s = x[R];
  for (int c = 0; c < PG_TILE; c++) {
    const int C = kt * PG_TILE + c;
    s -= (backward ? A[(size_t)C * N + R] : A[(size_t)R * N + C]) * x[C];
  }
  x[R] = s;
}

// The tile schedule of the factorization A = L L^T and of L L^T d = x.  G supplies the steps: potrf(kt) factors the diagonal
// tile and returns its verdict to every thread; panel(kt) the triangular solves of the tiles below it; trailing(kt) the update
// of every tile (it, jt), kt < jt <= it; trsv(kt, backward) the diagonal tile's solve of x; rows(kt, backward) every row
// update by that block; sync() a barrier of everything that shares the work.  Returns false on a failed pivot (x untouched
// then).
template <class G>
GB_AHD bool pg_cholesky_solve(G& g, int N) {
  const int T = N / PG_TILE;
  for (int kt = 0; kt < T; kt++) {
    if (!g.potrf(kt)) return false;
    g.panel(kt);
    g.sync();
    g.trailing(kt);
    g.sync();
  }
  for (int kt = 0; kt < T; kt++) {
    g.trsv(kt, false);
    g.sync();
    g.rows(kt, false);
    g.sync();
  }
  for (int kt = T - 1; kt >= 0; kt--) {
    g.trsv(kt, true);
    g.sync();
    g.rows(kt, true);
    g.sync();
  }
  return true;
}

// The rows a grid-strided row step updates: forward, the rows below block kt; backward, the rows above it
GB_AHD int pg_rows_begin(int kt, bool backward) { return backward ? 0 : (kt + 1) * PG_TILE; }
GB_AHD int pg_rows_end(int kt, int N, bool backward) { return backward ? kt * PG_TILE : N; }

// Rule step 2 after the solve, by a grid of nt threads (two phases around sync): T'_k = T_k Exp(delta_k) with each pose's
// step, v' = v + delta, b' = b + delta (X' = X when the factorization failed); then the largest pose steps, the trial count
// and, for every thread, the between, prior, IMU and vector errors at T' and each factor's evaluation row.
template <class Sync>
GB_AHD void pg_retract(const PoseGraphCall& c, bool solved, int tid, int nt, Sync sync) {
  const int KX = pg_num_poses(c);
  for (int k = tid; k < c.K; k += nt) {
    if (solved && k >= KX) {
      const int dof = k < KX + c.KV ? 3 : 6;
      for (int e = 0; e < 16; e++) c.Tn[16 * k + e] = e < dof ? c.T[16 * k + e] + c.x[6 * k + e] : c.T[16 * k + e];
    } else if (solved) {
      double E[16];
      align_exp(c.x + 6 * k, E);
      align_compose(c.T + 16 * k, E, c.Tn + 16 * k);
      align_step_norms(E, c.x + 6 * k, c.steps + 2 * k, c.steps + 2 * k + 1);
    } else {
      for (int e = 0; e < 16; e++) c.Tn[16 * k + e] = c.T[16 * k + e];
    }
  }
  sync();
  if (tid == 0) {
    AlignState& s = *c.st;
    s.trials += 1;
    s.solved = solved ? 1 : 0;
    s.dt = 0.0;
    s.dr = 0.0;
    if (solved)
      for (int k = 0; k < KX; k++) {
        s.dt = c.steps[2 * k] > s.dt ? c.steps[2 * k] : s.dt;
        s.dr = c.steps[2 * k + 1] > s.dr ? c.steps[2 * k + 1] : s.dr;
      }
  }
  for (int m = tid; m < c.B + c.Q + c.NI + c.NV; m += nt) {
    if (m < c.B) c.bterm[m] = pg_between_term(c.Tn + 16 * c.bt[m].key_i, c.Tn + 16 * c.bt[m].key_j, c.bt[m], nullptr);
    else if (m >= c.B + c.Q) c.nterm[m - c.B - c.Q] = pg_nav_term(c, m - c.B - c.Q, c.Tn, nullptr);
    else {
      const int q = m - c.B;
      c.pterm[q] = se3_prior_term(c.Tn + 16 * c.pkeys[q], c.pposes + 16 * q, c.pw[q], nullptr, 0, nullptr);
    }
  }
  for (int f = tid; f < c.F; f += nt) graph_row(c.Tn, c.fkeys[2 * f], c.fkeys[2 * f + 1], c.poses_eval + 16 * (size_t)f);
}

// Rule steps 3-5 (one thread): e' = the factors' errors at T' in record order, then the between terms', the IMU and vector
// terms', then the priors'; align_conclude.  Returns whether the trial was accepted (pg_accept_rows follows).
GB_AHD bool pg_conclude(const PoseGraphCall& c, const gb_align_params& prm) {
  double e = 0.0;
  for (int f = 0; f < c.F; f++) e += c.out[(size_t)f * 122 + 120];
  for (int m = 0; m < c.B; m++) e += c.bterm[m];
  for (int m = 0; m < c.NI + c.NV; m++) e += c.nterm[m];
  for (int q = 0; q < c.Q; q++) e += c.pterm[q];
  align_conclude(*c.st, prm, e);
  return c.st->need_lin != 0;
}

// An accepted trial: T = T' and every factor's linearization row at the new poses, by nt threads.  Ends with a barrier.
template <class Sync>
GB_AHD void pg_accept_rows(const PoseGraphCall& c, int tid, int nt, Sync sync) {
  for (int k = tid; k < 16 * c.K; k += nt) c.T[k] = c.Tn[k];
  sync();
  for (int f = tid; f < c.F; f += nt) graph_row(c.T, c.fkeys[2 * f], c.fkeys[2 * f + 1], c.poses + 16 * (size_t)f);
  sync();
}

}  // namespace

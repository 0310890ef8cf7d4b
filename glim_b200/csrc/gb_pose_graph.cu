// gb_pose_graph.cu -- gb_pose_graph_optimize: Levenberg-Marquardt over one graph of up to 1024 poses, and gb_nav_graph_optimize:
// the same solver over up to 2048 slots of poses, velocities and IMU biases with IMU and vector terms (sm_90a).
//
// Solves GLIM's global map on the device: the X(0) anchor, the matching-cost factors between overlapping submaps and the between
// factors of global mapping (global_mapping.cpp:360-377, :285-351, :546), or the odometry and Huber loop factors of the
// pose-graph back-end (global_mapping_pose_graph.cpp).  The rule is stated once, in include/glim_b200.h (gb_graph_optimize's
// rule for one problem, plus between terms); its arithmetic lives in gb_pose_graph_math.cuh (also compiled for the host by the
// CPU test) and its round loop is gb_align_rounds (gb_internal.cuh).
//
// One private gb_sweep covers every factor; its pose rows are T_t^-1 T_s.  A round is at most four launches whatever K, F or
// the number of between terms:
//   linearize sweep (when a linearization is needed and F > 0) -> k_pose_graph_step -> error sweep (F > 0) -> k_pose_graph_accept,
// then one 8-byte device-to-host copy of the status word and a stream sync.  k_pose_graph_step is one cooperative grid with
// grid.sync() between its phases: on a fresh linearization the between and prior terms, then the assembly of H and b into
// scratch; the damped padded copy; the right-looking tiled Cholesky (64 x 64 fp64 tiles: the diagonal tile by CTA 0 in shared
// memory, the panel's rows over the grid, the trailing tiles one per CTA on the fp64 tensor cores); the blocked forward and
// backward substitution; the retraction and the terms at the trial poses.  No sum uses an atomic, so two identical calls give
// bit-identical results.  gb_pose_graph_optimize is the call of gb_nav_graph_optimize without velocities, biases, IMU terms and
// vector terms (GLIM's enable_imu: false); both run optimize() below.
#include "gb_internal.cuh"
#include "gb_pose_graph_math.cuh"

#include <cooperative_groups.h>

#include <algorithm>
#include <vector>

namespace {

namespace cg = cooperative_groups;

constexpr int kStepThreads = 256;
constexpr int kAcceptThreads = 256;
constexpr int kLd = PG_TILE + 4;  // leading dimension of a tile in shared memory: a warp's fragment loads hit distinct banks
constexpr size_t kStepSmem = sizeof(double) * 2 * PG_TILE * kLd;  // two tiles: 68 KB

struct CtaSync {
  __device__ void operator()() const { __syncthreads(); }
};
struct WarpSync {
  __device__ void operator()() const { __syncwarp(); }
};
struct GridSync {
  cg::grid_group* g;
  __device__ void operator()() const { g->sync(); }
};

__device__ __forceinline__ void tile_load(double* s, const double* A, int N, int it, int jt) {
  const double* g = A + (size_t)it * PG_TILE * N + jt * PG_TILE;
  for (int e = threadIdx.x; e < PG_TILE * PG_TILE / 2; e += blockDim.x) {
    const int r = e / (PG_TILE / 2), c = 2 * (e % (PG_TILE / 2));
    const double2 v = *(const double2*)(g + (size_t)r * N + c);
    s[r * kLd + c] = v.x;
    s[r * kLd + c + 1] = v.y;
  }
}

// A_it,jt -= L_it,kt L_jt,kt^T by one CTA of 8 warps: warp w owns rows 8w .. 8w + 7 of the tile, eight 8 x 8 accumulators
// of mma.m8n8k4 f64 (A fragment: row lane / 4, column lane % 4; B: row lane % 4, column lane / 4; C: row lane / 4, columns
// 2 (lane % 4) + 0, 1), started from the tile and fed -L_it,kt.
__device__ void tile_update_dmma(double* A, int N, int it, int jt, int kt, double* sa, double* sb) {
  tile_load(sa, A, N, it, kt);
  tile_load(sb, A, N, jt, kt);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  double* C = A + (size_t)(it * PG_TILE + 8 * warp + g) * N + jt * PG_TILE + 2 * q;
  double acc[8][2];
#pragma unroll
  for (int nb = 0; nb < 8; nb++) {
    const double2 v = *(const double2*)(C + 8 * nb);
    acc[nb][0] = v.x;
    acc[nb][1] = v.y;
  }
#pragma unroll 4
  for (int k0 = 0; k0 < PG_TILE; k0 += 4) {
    const double a = -sa[(8 * warp + g) * kLd + k0 + q];
#pragma unroll
    for (int nb = 0; nb < 8; nb++) {
      const double b = sb[(8 * nb + g) * kLd + k0 + q];
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
                   : "+d"(acc[nb][0]), "+d"(acc[nb][1])
                   : "d"(a), "d"(b));
    }
  }
#pragma unroll
  for (int nb = 0; nb < 8; nb++) *(double2*)(C + 8 * nb) = make_double2(acc[nb][0], acc[nb][1]);
  __syncthreads();  // the next tile's loads overwrite sa, sb
}

__device__ __forceinline__ int volatile_load(const int* p) { return *(const volatile int*)p; }

// The tile steps of pg_cholesky_solve on the cooperative grid
struct DeviceTiles {
  const PoseGraphCall& c;
  cg::grid_group& grid;
  double* smem;
  int* flag;  // __shared__
  __device__ bool potrf(int kt) {
    if (blockIdx.x == 0) {
      double* D = c.A + (size_t)kt * PG_TILE * (c.N + 1);
      for (int e = threadIdx.x; e < PG_TILE * PG_TILE; e += blockDim.x) smem[(e / PG_TILE) * kLd + e % PG_TILE] = D[(size_t)(e / PG_TILE) * c.N + e % PG_TILE];
      __syncthreads();
      const bool ok = pg_potrf_tile(smem, kLd, (int)threadIdx.x, (int)blockDim.x, CtaSync{}, flag);
      for (int e = threadIdx.x; e < PG_TILE * PG_TILE; e += blockDim.x) D[(size_t)(e / PG_TILE) * c.N + e % PG_TILE] = smem[(e / PG_TILE) * kLd + e % PG_TILE];
      if (threadIdx.x == 0) *c.ok = ok ? 1 : 0;
    }
    grid.sync();
    return volatile_load(c.ok) != 0;
  }
  __device__ void panel(int kt) {
    const int first = (kt + 1) * PG_TILE + (int)blockIdx.x * (int)blockDim.x;
    if (first >= c.N) return;
    const double* D = c.A + (size_t)kt * PG_TILE * (c.N + 1);
    for (int e = threadIdx.x; e < PG_TILE * PG_TILE; e += blockDim.x) smem[(e / PG_TILE) * kLd + e % PG_TILE] = D[(size_t)(e / PG_TILE) * c.N + e % PG_TILE];
    __syncthreads();
    for (int R = first + (int)threadIdx.x; R < c.N; R += (int)(gridDim.x * blockDim.x)) pg_trsm_row(c.A + (size_t)R * c.N + kt * PG_TILE, smem, kLd);
    __syncthreads();
  }
  __device__ void trailing(int kt) {
    const int m = c.N / PG_TILE - 1 - kt;
    for (long long t = blockIdx.x; t < (long long)m * (m + 1) / 2; t += gridDim.x) {
      int i, j;
      pg_tri(t, &i, &j);
      tile_update_dmma(c.A, c.N, kt + 1 + i, kt + 1 + j, kt, smem, smem + PG_TILE * kLd);
    }
  }
  __device__ void trsv(int kt, bool backward) {
    if (blockIdx.x == 0 && threadIdx.x < 32)
      pg_trsv_tile(c.A + (size_t)kt * PG_TILE * (c.N + 1), c.N, c.x + kt * PG_TILE, backward, (int)threadIdx.x, 32, WarpSync{});
  }
  __device__ void rows(int kt, bool backward) {
    const int stride = (int)(gridDim.x * blockDim.x);
    for (int R = pg_rows_begin(kt, backward) + (int)(blockIdx.x * blockDim.x + threadIdx.x); R < pg_rows_end(kt, c.N, backward); R += stride)
      pg_substitute_row(c.A, c.N, kt, c.x, R, backward);
  }
  __device__ void sync() { grid.sync(); }
};

// The between and prior records, out of line: their 6x6 arithmetic gets registers of its own instead of crowding the tile loops'
__device__ __noinline__ void terms_at(const PoseGraphCall& c, int tid, int nt) { pg_terms_at(c, tid, nt); }

// Rule steps 1-2 on the whole grid.  Block 0 clears the status word.
__global__ void __launch_bounds__(kStepThreads, 1) k_pose_graph_step(PoseGraphCall c, unsigned* __restrict__ counters) {
  extern __shared__ double smem[];
  __shared__ int flag;
  cg::grid_group grid = cg::this_grid();
  align_status_clear(counters);
  const int tid = (int)(blockIdx.x * blockDim.x + threadIdx.x), nt = (int)(gridDim.x * blockDim.x);
  AlignState* s = c.st;
  if (volatile_load(&s->status) != GB_ALIGN_ACTIVE) return;  // the whole grid alike
  if (volatile_load(&s->need_lin)) {
    terms_at(c, tid, nt);
    grid.sync();
    pg_assemble(c, tid, nt);
    if (tid == 0) pg_linearized(c);
    grid.sync();
    if (volatile_load(&s->status) != GB_ALIGN_ACTIVE) return;
  }
  pg_damped_copy(c, *(const volatile double*)&s->lambda, tid, nt);
  grid.sync();
  DeviceTiles g{c, grid, smem, &flag};
  const bool solved = pg_cholesky_solve(g, c.N);
  pg_retract(c, solved, tid, nt, GridSync{&grid});
}

// One CTA: rule steps 3-5 (pg_conclude) and, for an accepted trial, the new poses and linearization rows; then the status word.
__global__ void __launch_bounds__(kAcceptThreads) k_pose_graph_accept(PoseGraphCall c, gb_align_params prm, unsigned* __restrict__ counters) {
  __shared__ int accepted;
  if (c.st->status != GB_ALIGN_ACTIVE) return;
  if (threadIdx.x == 0) {
    pg_conclude(c, prm);
    accepted = align_status_tally(*c.st, counters) & 1;
  }
  __syncthreads();
  if (accepted) pg_accept_rows(c, (int)threadIdx.x, (int)blockDim.x, CtaSync{});
}

struct Inputs {
  size_t K, F, Q, B;  // K: pose keys
  const double* T_init;
  gb_factor* const* factors;
  const int32_t* fkeys;
  const int32_t* qkeys;
  const double* qposes;
  const double* qw;
  const gb_between_term* bt;
  // the navigation part (gb_nav_graph_optimize)
  size_t KV, KB, NI, NV;
  const double* v_init;
  const double* b_init;
  const gb_imu_term* it;
  const gb_vector_term* vt;
};

// the pose graph's size
gb_status validate_size(const Inputs& in, const gb_align_params* prm) {
  GB_REQUIRE(in.T_init && prm, "null argument");
  GB_REQUIRE(in.K >= 2 && in.K <= GB_POSE_GRAPH_MAX_KEYS, "a pose graph needs 2 to GB_POSE_GRAPH_MAX_KEYS keys");
  GB_REQUIRE(in.F + in.B >= 1, "a pose graph needs a factor or a between term");
  return GB_OK;
}

// the pose graph's checks that do not concern its size
gb_status validate_terms(gb_ctx* ctx, const Inputs& in, const gb_align_params* prm) {
  GB_REQUIRE(in.F < ((size_t)1 << 28) && in.B < ((size_t)1 << 24) && in.Q < ((size_t)1 << 20), "too many factors, between terms or priors");
  GB_REQUIRE(in.F == 0 || (in.factors && in.fkeys), "null factor arrays");
  GB_REQUIRE(in.Q == 0 || (in.qkeys && in.qposes && in.qw), "null prior arrays");
  GB_REQUIRE(in.B == 0 || in.bt, "null between terms");
  const int64_t K = (int64_t)in.K;
  for (size_t f = 0; f < in.F; f++) {
    const int32_t t = in.fkeys[2 * f], s = in.fkeys[2 * f + 1];
    GB_REQUIRE(t >= 0 && s >= 0 && t < K && s < K && t != s, "factor keys must be in range and differ");
  }
  for (size_t q = 0; q < in.Q; q++) GB_REQUIRE(in.qkeys[q] >= 0 && in.qkeys[q] < K, "prior keys must be in range");
  for (size_t m = 0; m < in.B; m++) {
    const gb_between_term& b = in.bt[m];
    GB_REQUIRE(b.key_i >= 0 && b.key_j >= 0 && b.key_i < K && b.key_j < K && b.key_i != b.key_j, "between keys must be in range and differ");
    GB_REQUIRE(gb_all_finite(b.Z, 16), "between measurements must be finite");
    GB_REQUIRE(gb_all_finite(b.information, 36), "between information must be finite");
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < i; j++) GB_REQUIRE(b.information[i * 6 + j] == b.information[j * 6 + i], "between information must be exactly symmetric");
    GB_REQUIRE(isfinite(b.huber_width) && b.huber_width >= 0.0, "huber_width must be finite and >= 0");
  }
  for (size_t f = 0; f < in.F; f++) {
    const gb_factor* fa = in.factors[f];
    GB_REQUIRE(fa, "null factor");
    GB_REQUIRE(fa->kind == GB_FACTOR_POSE, "not a pose factor: CT and plane factors have no place in a graph");
    GB_REQUIRE(fa->source->device == ctx->device && fa->target->device == ctx->device, "factor lives on another device");
    GB_REQUIRE(gb_factor_class(fa) == gb_factor_class(in.factors[0]),
               "the factors of one call must all be VGICP factors, all GICP factors on iVoxes, all GICP factors on point grids or all ICP factors");
  }
  GB_REQUIRE(gb_all_finite(in.T_init, 16 * in.K), "T_init must be finite");
  GB_REQUIRE(in.Q == 0 || gb_all_finite(in.qposes, 16 * in.Q), "prior poses must be finite");
  for (size_t q = 0; q < in.Q; q++) GB_REQUIRE(isfinite(in.qw[q]) && in.qw[q] >= 0.0, "prior precisions must be finite and >= 0");
  return gb_align_params_check(prm);
}

// the navigation graph's own checks (its size, its velocities, biases, IMU and vector terms)
gb_status validate_nav(const Inputs& in, const gb_align_params* prm) {
  GB_REQUIRE(in.T_init && prm, "null argument");
  GB_REQUIRE(in.K >= 1 && in.K <= GB_NAV_GRAPH_MAX_SLOTS && in.KV <= GB_NAV_GRAPH_MAX_SLOTS && in.KB <= GB_NAV_GRAPH_MAX_SLOTS && in.K + in.KV + in.KB >= 2 &&
                 in.K + in.KV + in.KB <= GB_NAV_GRAPH_MAX_SLOTS,
             "a navigation graph needs a pose and 2 to GB_NAV_GRAPH_MAX_SLOTS variables");
  GB_REQUIRE(in.NI < ((size_t)1 << 24) && in.NV < ((size_t)1 << 24), "too many IMU or vector terms");
  GB_REQUIRE(in.F + in.B + in.NI + in.NV >= 1, "a navigation graph needs a factor, a between, an IMU or a vector term");
  GB_REQUIRE(in.KV == 0 || in.v_init, "null velocities");
  GB_REQUIRE(in.KB == 0 || in.b_init, "null biases");
  GB_REQUIRE(in.NI == 0 || in.it, "null IMU terms");
  GB_REQUIRE(in.NV == 0 || in.vt, "null vector terms");
  GB_REQUIRE(in.KV == 0 || gb_all_finite(in.v_init, 3 * in.KV), "v_init must be finite");
  GB_REQUIRE(in.KB == 0 || gb_all_finite(in.b_init, 6 * in.KB), "b_init must be finite");
  const int64_t KX = (int64_t)in.K, KV = (int64_t)in.KV, KB = (int64_t)in.KB;
  for (size_t m = 0; m < in.NI; m++) {
    const gb_imu_term& t = in.it[m];
    GB_REQUIRE(t.pose_i >= 0 && t.pose_j >= 0 && t.pose_i < KX && t.pose_j < KX && t.pose_i != t.pose_j, "IMU term poses must be in range and differ");
    GB_REQUIRE(t.vel_i >= 0 && t.vel_j >= 0 && t.vel_i < KV && t.vel_j < KV && t.vel_i != t.vel_j, "IMU term velocities must be in range and differ");
    GB_REQUIRE(t.bias_i >= 0 && t.bias_i < KB, "IMU term bias must be in range");
    const gb_imu_preintegrated& p = t.pim;
    GB_REQUIRE(isfinite(p.delta_t) && p.delta_t > 0.0, "IMU record delta_t must be finite and > 0");
    GB_REQUIRE(gb_all_finite(p.preintegrated, 9) && gb_all_finite(p.H_bias_acc, 27) && gb_all_finite(p.H_bias_omega, 27) &&
                   gb_all_finite(p.covariance, 81) && gb_all_finite(p.bias_hat, 6) && gb_all_finite(p.gravity, 3),
               "IMU records must be finite");
    for (int i = 0; i < 9; i++)
      for (int j = 0; j < i; j++) GB_REQUIRE(p.covariance[i * 9 + j] == p.covariance[j * 9 + i], "IMU covariance must be exactly symmetric");
    // positive definiteness: optimize() factors each covariance once, before any launch, and refuses a failed pivot
  }
  for (size_t m = 0; m < in.NV; m++) {
    const gb_vector_term& v = in.vt[m];
    const int64_t a = v.key_a, b = v.key_b;
    switch (v.kind) {
      case GB_VECTOR_VELOCITY_PRIOR: GB_REQUIRE(a >= 0 && a < KV, "vector term keys must be in range"); break;
      case GB_VECTOR_BIAS_PRIOR: GB_REQUIRE(a >= 0 && a < KB, "vector term keys must be in range"); break;
      case GB_VECTOR_VELOCITY_BETWEEN: GB_REQUIRE(a >= 0 && b >= 0 && a < KV && b < KV && a != b, "vector between keys must be in range and differ"); break;
      case GB_VECTOR_BIAS_BETWEEN: GB_REQUIRE(a >= 0 && b >= 0 && a < KB && b < KB && a != b, "vector between keys must be in range and differ"); break;
      case GB_VECTOR_ROTATE_VELOCITY: GB_REQUIRE(a >= 0 && b >= 0 && a < KX && b < KV, "vector term keys must be in range"); break;
      default: GB_REQUIRE(false, "unknown vector term kind");
    }
    GB_REQUIRE(gb_all_finite(v.z, 6), "vector measurements must be finite");
    GB_REQUIRE(isfinite(v.precision) && v.precision >= 0.0, "vector precisions must be finite and >= 0");
  }
  return GB_OK;
}

// The slots of nav term m (IMU terms first): poses at their keys, velocities from K_X, biases from K_X + K_V
void nav_slots(const Inputs& in, std::vector<int>& slots) {
  const int v0 = (int)in.K, b0 = (int)(in.K + in.KV);
  slots.assign(5 * (in.NI + in.NV), -1);
  for (size_t m = 0; m < in.NI; m++) {
    const gb_imu_term& t = in.it[m];
    const int s[5] = {t.pose_i, v0 + t.vel_i, t.pose_j, v0 + t.vel_j, b0 + t.bias_i};
    for (int a = 0; a < 5; a++) slots[5 * m + a] = s[a];
  }
  for (size_t m = 0; m < in.NV; m++) {
    const gb_vector_term& v = in.vt[m];
    int* s = slots.data() + 5 * (in.NI + m);
    switch (v.kind) {
      case GB_VECTOR_VELOCITY_PRIOR: s[0] = v0 + v.key_a; break;
      case GB_VECTOR_BIAS_PRIOR: s[0] = b0 + v.key_a; break;
      case GB_VECTOR_VELOCITY_BETWEEN: s[0] = v0 + v.key_a; s[1] = v0 + v.key_b; break;
      case GB_VECTOR_BIAS_BETWEEN: s[0] = b0 + v.key_a; s[1] = b0 + v.key_b; break;
      default: s[0] = v.key_a; s[1] = v0 + v.key_b; break;
    }
  }
}

// The solve of a validated graph, entered in ctx.  v_out / b_out receive the velocities and biases (none for a pose graph).
gb_status optimize(gb_ctx* ctx, const Inputs& in, const gb_align_params* prm, double* T_out, double* v_out, double* b_out, gb_graph_result* result) {
  const int KX = (int)in.K, KV = (int)in.KV, KB = (int)in.KB, F = (int)in.F, Q = (int)in.Q, B = (int)in.B, NI = (int)in.NI, NV = (int)in.NV;
  const int K = KX + KV + KB, n = 6 * K, N = pg_padded(n);

  // everything derived on the host once per call: the slot states, the block CSR of the factors, between, IMU and vector terms,
  // the priors by key, the rows
  std::vector<double> X(16 * (size_t)K, 0.0);
  std::copy(in.T_init, in.T_init + 16 * (size_t)KX, X.begin());
  for (int k = 0; k < KV; k++) std::copy(in.v_init + 3 * k, in.v_init + 3 * k + 3, X.begin() + 16 * (size_t)(KX + k));
  for (int k = 0; k < KB; k++) std::copy(in.b_init + 6 * k, in.b_init + 6 * k + 6, X.begin() + 16 * (size_t)(KX + KV + k));
  std::vector<int> keys(2 * (size_t)(F + B));
  for (int f = 0; f < F; f++) {
    keys[2 * f] = in.fkeys[2 * f];
    keys[2 * f + 1] = in.fkeys[2 * f + 1];
  }
  for (int m = 0; m < B; m++) {
    keys[2 * (F + m)] = in.bt[m].key_i;
    keys[2 * (F + m) + 1] = in.bt[m].key_j;
  }
  std::vector<int> nslots;
  nav_slots(in, nslots);
  std::vector<double> nchol(81 * (size_t)NI);  // each IMU covariance factored once, here; the device whitens with these factors
  for (int m = 0; m < NI; m++) {
    std::copy(in.it[m].pim.covariance, in.it[m].pim.covariance + 81, nchol.begin() + 81 * (size_t)m);
    GB_REQUIRE(imu_cholesky(nchol.data() + 81 * (size_t)m, 9), "IMU covariance must be positive definite");
  }
  std::vector<int> cptr(graph_num_blocks(K) + 1), qptr(K + 1), qidx(Q), qkeys(in.qkeys, in.qkeys + Q);
  std::vector<GraphContrib> contrib(5 * (size_t)(F + B) + 20 * (size_t)(NI + NV));
  graph_contributions(K, F + B, keys.data(), 0, cptr.data(), contrib.data(), NI + NV, nslots.data());
  pg_prior_index(K, Q, qkeys.data(), qptr.data(), qidx.data());
  AlignState st;
  align_init(st, in.T_init, prm->lambda_initial);
  std::vector<double> rows(16 * (size_t)F);
  for (int f = 0; f < F; f++) graph_row(in.T_init, keys[2 * f], keys[2 * f + 1], rows.data() + 16 * f);

  gb_sweep* sweep = nullptr;
  if (F > 0) GB_CHECK(gb_sweep_create(ctx, in.F, in.factors, nullptr, &sweep));
  const gb_owned<gb_sweep> s(sweep, sweep_free);  // its blocks go back to the context's pool on every exit
  PoseGraphCall c{};
  c.K = K; c.n = n; c.N = N; c.F = F; c.B = B; c.Q = Q;
  c.KV = KV; c.KB = KB; c.NI = NI; c.NV = NV;
  unsigned* d_ctr = nullptr;
  unsigned* h_ctr = nullptr;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    c.cptr = cv.take<int>(cptr.size());
    c.contrib = cv.take<GraphContrib>(contrib.size());
    c.qptr = cv.take<int>(qptr.size());
    c.qidx = cv.take<int>(Q);
    c.fkeys = cv.take<int>(2 * (size_t)F);
    c.bt = cv.take<gb_between_term>(B);
    c.pkeys = cv.take<int>(Q);
    c.pposes = cv.take<double>(16 * (size_t)Q);
    c.pw = cv.take<double>(Q);
    c.brec = cv.take<double>(122 * (size_t)B);
    c.prec = cv.take<double>(PG_PRIOR_DOUBLES * (size_t)Q);
    c.bterm = cv.take<double>(B);
    c.pterm = cv.take<double>(Q);
    c.T = cv.take<double>(16 * (size_t)K);
    c.Tn = cv.take<double>(16 * (size_t)K);
    c.H = cv.take<double>((size_t)n * n);
    c.b = cv.take<double>(n);
    c.A = cv.take<double>((size_t)N * N);
    c.x = cv.take<double>(N);
    c.steps = cv.take<double>(2 * (size_t)K);
    c.ok = cv.take<int>(1);
    c.st = cv.take<AlignState>(1);
    c.it = cv.take<gb_imu_term>(NI);
    c.vt = cv.take<gb_vector_term>(NV);
    c.nslots = cv.take<int>(nslots.size());
    c.nrec = cv.take<double>(PG_NAV_DOUBLES * (size_t)(NI + NV));
    c.nterm = cv.take<double>(NI + NV);
    c.nchol = cv.take<double>(nchol.size());
    d_ctr = cv.take<unsigned>(2);
  }));
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) { h_ctr = cv.take<unsigned>(2); }));
  if (F > 0) {
    c.poses = s->d_poses;
    c.poses_eval = s->d_poses_eval;
    c.out = s->d_out;
  }
  GB_CHECK(gb_upload(ctx, {{(void*)c.cptr, cptr.data(), sizeof(int) * cptr.size()},
                           {(void*)c.contrib, contrib.data(), sizeof(GraphContrib) * contrib.size()},
                           {(void*)c.qptr, qptr.data(), sizeof(int) * qptr.size()},
                           {(void*)c.qidx, qidx.data(), sizeof(int) * Q},
                           {(void*)c.fkeys, keys.data(), sizeof(int) * 2 * (size_t)F},
                           {(void*)c.bt, in.bt, sizeof(gb_between_term) * B},
                           {(void*)c.pkeys, qkeys.data(), sizeof(int) * Q},
                           {(void*)c.pposes, in.qposes, sizeof(double) * 16 * Q},
                           {(void*)c.pw, in.qw, sizeof(double) * Q},
                           {c.T, X.data(), sizeof(double) * X.size()},
                           {c.Tn, X.data(), sizeof(double) * X.size()},
                           {c.st, &st, sizeof(AlignState)},
                           {c.poses, rows.data(), sizeof(double) * 16 * F},
                           {c.poses_eval, rows.data(), sizeof(double) * 16 * F},
                           {(void*)c.it, in.it, sizeof(gb_imu_term) * NI},
                           {(void*)c.vt, in.vt, sizeof(gb_vector_term) * NV},
                           {(void*)c.nslots, nslots.data(), sizeof(int) * nslots.size()},
                           {(void*)c.nchol, nchol.data(), sizeof(double) * nchol.size()}}));
  // a persistent grid: as many CTAs as can be resident at once (the cooperative launch refuses more)
  GB_CUDA(cudaFuncSetAttribute(k_pose_graph_step, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStepSmem));
  int per_sm = 0;
  GB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pose_graph_step, kStepThreads, kStepSmem));
  GB_REQUIRE(per_sm > 0, "k_pose_graph_step cannot be resident");
  const int grid = per_sm * ctx->num_sms;
  GB_CHECK(gb_align_rounds(ctx, d_ctr, h_ctr, [&](bool need_lin) -> gb_status {
    if (need_lin && F > 0) GB_CHECK(gb_launch_sweep(s.get(), GB_MODE_LINEARIZE));
    GB_CHECK(gb_launch(ctx, "k_pose_graph_step", gb_cooperative, k_pose_graph_step, grid, kStepThreads, kStepSmem, c, d_ctr));
    if (F > 0) GB_CHECK(gb_launch_sweep(s.get(), GB_MODE_ERROR));
    return gb_launch(ctx, "k_pose_graph_accept", k_pose_graph_accept, 1, kAcceptThreads, 0, c, *prm, d_ctr);
  }));
  GB_CHECK(gb_download(ctx, {{&st, c.st, sizeof(AlignState)}, {X.data(), c.T, sizeof(double) * X.size()}}));
  std::copy(X.begin(), X.begin() + 16 * (size_t)KX, T_out);
  for (int k = 0; k < KV; k++) std::copy(X.begin() + 16 * (size_t)(KX + k), X.begin() + 16 * (size_t)(KX + k) + 3, v_out + 3 * k);
  for (int k = 0; k < KB; k++) std::copy(X.begin() + 16 * (size_t)(KX + KV + k), X.begin() + 16 * (size_t)(KX + KV + k) + 6, b_out + 6 * k);
  align_result(st, *result);
  return GB_OK;
}

}  // namespace

extern "C" gb_status gb_pose_graph_optimize(gb_ctx* ctx, size_t num_keys, const double* T_init, size_t num_factors, gb_factor* const* factors,
                                            const int32_t* factor_keys, size_t num_priors, const int32_t* prior_keys, const double* prior_poses,
                                            const double* prior_precisions, size_t num_betweens, const gb_between_term* betweens, const gb_align_params* prm,
                                            double* T_out, gb_graph_result* result) {
  GB_REQUIRE(ctx, "null ctx");
  GB_REQUIRE(T_out && result, "null output");
  Inputs in{};
  in.K = num_keys; in.F = num_factors; in.Q = num_priors; in.B = num_betweens;
  in.T_init = T_init; in.factors = factors; in.fkeys = factor_keys; in.qkeys = prior_keys; in.qposes = prior_poses; in.qw = prior_precisions; in.bt = betweens;
  GB_CHECK(validate_size(in, prm));
  GB_CHECK(validate_terms(ctx, in, prm));
  GB_ENTER(ctx);
  return optimize(ctx, in, prm, T_out, nullptr, nullptr, result);
}

extern "C" gb_status gb_nav_graph_optimize(gb_ctx* ctx, size_t num_poses, const double* T_init, size_t num_velocities, const double* v_init, size_t num_biases,
                                           const double* b_init, size_t num_factors, gb_factor* const* factors, const int32_t* factor_keys, size_t num_priors,
                                           const int32_t* prior_keys, const double* prior_poses, const double* prior_precisions, size_t num_betweens,
                                           const gb_between_term* betweens, size_t num_imu_terms, const gb_imu_term* imu_terms, size_t num_vector_terms,
                                           const gb_vector_term* vector_terms, const gb_align_params* prm, double* T_out, double* v_out, double* b_out,
                                           gb_graph_result* result) {
  GB_REQUIRE(ctx, "null ctx");
  GB_REQUIRE(T_out && result && (num_velocities == 0 || v_out) && (num_biases == 0 || b_out), "null output");
  Inputs in{};
  in.K = num_poses; in.F = num_factors; in.Q = num_priors; in.B = num_betweens;
  in.T_init = T_init; in.factors = factors; in.fkeys = factor_keys; in.qkeys = prior_keys; in.qposes = prior_poses; in.qw = prior_precisions; in.bt = betweens;
  in.KV = num_velocities; in.KB = num_biases; in.NI = num_imu_terms; in.NV = num_vector_terms;
  in.v_init = v_init; in.b_init = b_init; in.it = imu_terms; in.vt = vector_terms;
  GB_CHECK(validate_nav(in, prm));
  GB_CHECK(validate_terms(ctx, in, prm));
  GB_ENTER(ctx);
  return optimize(ctx, in, prm, T_out, v_out, b_out, result);
}

// gb_pose_graph.cu -- gb_pose_graph_optimize: Levenberg-Marquardt over one graph of up to 1024 poses (sm_90a).
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
// bit-identical results.
#include "gb_internal.cuh"
#include "gb_pose_graph_math.cuh"

#include <cooperative_groups.h>

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
  size_t K, F, Q, B;
  const double* T_init;
  gb_factor* const* factors;
  const int32_t* fkeys;
  const int32_t* qkeys;
  const double* qposes;
  const double* qw;
  const gb_between_term* bt;
};

gb_status validate(gb_ctx* ctx, const Inputs& in, const gb_align_params* prm) {
  GB_REQUIRE(in.T_init && prm, "null argument");
  GB_REQUIRE(in.K >= 2 && in.K <= GB_POSE_GRAPH_MAX_KEYS, "a pose graph needs 2 to GB_POSE_GRAPH_MAX_KEYS keys");
  GB_REQUIRE(in.F + in.B >= 1, "a pose graph needs a factor or a between term");
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

}  // namespace

extern "C" gb_status gb_pose_graph_optimize(gb_ctx* ctx, size_t num_keys, const double* T_init, size_t num_factors, gb_factor* const* factors,
                                            const int32_t* factor_keys, size_t num_priors, const int32_t* prior_keys, const double* prior_poses,
                                            const double* prior_precisions, size_t num_betweens, const gb_between_term* betweens, const gb_align_params* prm,
                                            double* T_out, gb_graph_result* result) {
  GB_REQUIRE(ctx, "null ctx");
  GB_REQUIRE(T_out && result, "null output");
  const Inputs in{num_keys, num_factors, num_priors, num_betweens, T_init, factors, factor_keys, prior_keys, prior_poses, prior_precisions, betweens};
  GB_CHECK(validate(ctx, in, prm));
  const int K = (int)num_keys, F = (int)num_factors, Q = (int)num_priors, B = (int)num_betweens;
  const int n = 6 * K, N = pg_padded(n);

  // everything derived on the host once per call: the block CSR of the factors and between terms, the priors by key, the rows
  std::vector<int> keys(2 * (size_t)(F + B));
  for (int f = 0; f < F; f++) {
    keys[2 * f] = factor_keys[2 * f];
    keys[2 * f + 1] = factor_keys[2 * f + 1];
  }
  for (int m = 0; m < B; m++) {
    keys[2 * (F + m)] = betweens[m].key_i;
    keys[2 * (F + m) + 1] = betweens[m].key_j;
  }
  std::vector<int> cptr(graph_num_blocks(K) + 1), qptr(K + 1), qidx(Q), qkeys(prior_keys, prior_keys + Q);
  std::vector<GraphContrib> contrib(5 * (size_t)(F + B));
  graph_contributions(K, F + B, keys.data(), 0, cptr.data(), contrib.data());
  pg_prior_index(K, Q, qkeys.data(), qptr.data(), qidx.data());
  AlignState st;
  align_init(st, T_init, prm->lambda_initial);
  std::vector<double> rows(16 * (size_t)F);
  for (int f = 0; f < F; f++) graph_row(T_init, keys[2 * f], keys[2 * f + 1], rows.data() + 16 * f);

  GB_ENTER(ctx);
  gb_sweep* sweep = nullptr;
  if (F > 0) GB_CHECK(gb_sweep_create(ctx, num_factors, factors, nullptr, &sweep));
  const gb_owned<gb_sweep> s(sweep, sweep_free);  // its blocks go back to the context's pool on every exit
  PoseGraphCall c{};
  c.K = K; c.n = n; c.N = N; c.F = F; c.B = B; c.Q = Q;
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
                           {(void*)c.bt, betweens, sizeof(gb_between_term) * B},
                           {(void*)c.pkeys, qkeys.data(), sizeof(int) * Q},
                           {(void*)c.pposes, prior_poses, sizeof(double) * 16 * Q},
                           {(void*)c.pw, prior_precisions, sizeof(double) * Q},
                           {c.T, T_init, sizeof(double) * 16 * K},
                           {c.Tn, T_init, sizeof(double) * 16 * K},
                           {c.st, &st, sizeof(AlignState)},
                           {c.poses, rows.data(), sizeof(double) * 16 * F},
                           {c.poses_eval, rows.data(), sizeof(double) * 16 * F}}));
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
  GB_CHECK(gb_download(ctx, {{&st, c.st, sizeof(AlignState)}, {T_out, c.T, sizeof(double) * 16 * K}}));
  align_result(st, *result);
  return GB_OK;
}

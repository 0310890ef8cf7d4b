// gb_graph.cu -- gb_graph_optimize: Levenberg-Marquardt over several poses per problem, many problems in one call (sm_90a).
//
// Replaces the LevenbergMarquardtOptimizer GLIM runs over matching-cost factors and pose priors: sub-mapping's submap
// optimization (sub_mapping.cpp:428-452), global mapping's between factor (global_mapping.cpp:393-426) and the manual loop
// closure's align (manual_loop_close_modal.cpp:476-517).  The rule is stated once, in include/glim_b200.h (gb_vgicp_align's
// rule at 6K dof); its per-problem arithmetic lives in gb_graph_math.cuh (also compiled for the host by the CPU test) and its
// round loop is gb_align_rounds (gb_internal.cuh), shared with the other aligners.
//
// One private gb_sweep covers every factor of every problem, in CSR order; its pose rows are T_t^-1 T_s.  A round is at most
// four launches:
//   linearize sweep (if any problem needs a linearization) -> k_graph_step -> error sweep -> k_graph_accept,
// then one 8-byte device-to-host copy of the status word and a stream sync.  k_graph_step runs one CTA per problem and factors
// the damped system as a packed lower triangle in dynamic shared memory: (6K)(6K + 1) / 2 + 6K + 64 doubles, 149.8 KB at
// K = 32, within the 227 KB a CTA can opt into.
#include "gb_internal.cuh"
#include "gb_graph_math.cuh"

#include <string.h>

#include <vector>

namespace {

constexpr int kGraphThreads = 256;
constexpr int kAcceptThreads = 256;  // 8 problems (one warp each) per CTA

struct CtaSync {
  __device__ void operator()() const { __syncthreads(); }
};
struct WarpSync {
  __device__ void operator()() const { __syncwarp(); }
};

// One CTA per problem: graph_step.  Block 0 clears the status word.
__global__ void __launch_bounds__(kGraphThreads) k_graph_step(GraphCall c, unsigned* __restrict__ counters) {
  extern __shared__ double smem[];
  __shared__ int flag;
  align_status_clear(counters);
  graph_step(c, (int)blockIdx.x, smem, (int)threadIdx.x, (int)blockDim.x, CtaSync{}, &flag);
}

// One warp per problem: rule steps 3-5 (graph_conclude) and, for an accepted trial, the new poses into the linearization rows;
// then count active problems and those that need a linearization.
__global__ void __launch_bounds__(kAcceptThreads) k_graph_accept(GraphCall c, int P, gb_align_params prm, unsigned* __restrict__ counters) {
  const int p = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= P || c.st[p].a.status != GB_ALIGN_ACTIVE) return;
  int flags = 0;
  if (lane == 0) {
    graph_conclude(c, p, prm);
    flags = align_status_tally(c.st[p].a, counters);
  }
  flags = __shfl_sync(0xffffffffu, flags, 0);
  if (flags & 1) graph_accept_rows(c, p, lane, 32, WarpSync{});
}

struct Inputs {
  size_t P;
  const size_t* koff;
  const double* T_init;
  const size_t* foff;
  gb_factor* const* factors;
  const int32_t* fkeys;
  const size_t* qoff;
  const int32_t* qkeys;
  const double* qposes;
  const double* qw;
};

gb_status validate(gb_ctx* ctx, const Inputs& in, const gb_align_params* prm) {
  GB_REQUIRE(in.koff && in.T_init && in.foff && in.factors && in.fkeys && in.qoff && prm, "null argument");
  GB_REQUIRE(in.koff[0] == 0 && in.foff[0] == 0 && in.qoff[0] == 0, "key_offsets, factor_offsets and prior_offsets must start at 0");
  for (size_t p = 0; p < in.P; p++) {
    const size_t K = in.koff[p + 1] - in.koff[p];
    GB_REQUIRE(in.koff[p + 1] >= in.koff[p] && K >= 2 && K <= GB_GRAPH_MAX_KEYS, "every problem needs 2 to GB_GRAPH_MAX_KEYS keys");
    GB_REQUIRE(in.foff[p + 1] > in.foff[p], "factor_offsets must increase strictly (every problem needs a factor)");
    GB_REQUIRE(in.qoff[p + 1] >= in.qoff[p], "prior_offsets must not decrease");
    GB_REQUIRE(in.qoff[p + 1] - in.qoff[p] < ((size_t)1 << 20), "too many priors");
    for (size_t f = in.foff[p]; f < in.foff[p + 1] && f < ((size_t)1 << 30); f++) {
      const int32_t t = in.fkeys[2 * f], s = in.fkeys[2 * f + 1];
      GB_REQUIRE(t >= 0 && s >= 0 && (size_t)t < K && (size_t)s < K && t != s, "factor keys must be in range and differ");
    }
    for (size_t q = in.qoff[p]; q < in.qoff[p + 1]; q++) GB_REQUIRE(in.qkeys[q] >= 0 && (size_t)in.qkeys[q] < K, "prior keys must be in range");
  }
  const size_t F = in.foff[in.P], Q = in.qoff[in.P], NK = in.koff[in.P];
  GB_REQUIRE(F < ((size_t)1 << 30) && NK < ((size_t)1 << 24), "too many factors or keys");
  GB_REQUIRE(Q == 0 || (in.qkeys && in.qposes && in.qw), "null prior arrays");
  for (size_t f = 0; f < F; f++) {
    const gb_factor* fa = in.factors[f];
    GB_REQUIRE(fa, "null factor");
    GB_REQUIRE(fa->kind == GB_FACTOR_POSE, "not a pose factor: CT and plane factors have no place in a graph");
    GB_REQUIRE(fa->source->device == ctx->device && fa->target->device == ctx->device, "factor lives on another device");
    GB_REQUIRE(gb_factor_class(fa) == gb_factor_class(in.factors[0]),
               "the factors of one call must all be VGICP factors, all GICP factors on iVoxes, all GICP factors on point grids or all ICP factors");
  }
  GB_REQUIRE(gb_all_finite(in.T_init, 16 * NK), "T_init must be finite");
  GB_REQUIRE(Q == 0 || gb_all_finite(in.qposes, 16 * Q), "prior poses must be finite");
  for (size_t q = 0; q < Q; q++) GB_REQUIRE(isfinite(in.qw[q]) && in.qw[q] >= 0.0, "prior precisions must be finite and >= 0");
  return gb_align_params_check(prm);
}

}  // namespace

extern "C" gb_status gb_graph_optimize(gb_ctx* ctx, size_t P, const size_t* key_offsets, const double* T_init, const size_t* factor_offsets,
                                       gb_factor* const* factors, const int32_t* factor_keys, const size_t* prior_offsets, const int32_t* prior_keys,
                                       const double* prior_poses, const double* prior_precisions, const gb_align_params* prm, double* T_out,
                                       gb_graph_result* results) {
  GB_REQUIRE(ctx, "null ctx");
  if (P == 0) return GB_OK;
  GB_REQUIRE(T_out && results, "null output");
  const Inputs in{P, key_offsets, T_init, factor_offsets, factors, factor_keys, prior_offsets, prior_keys, prior_poses, prior_precisions};
  GB_CHECK(validate(ctx, in, prm));
  const size_t F = factor_offsets[P], Q = prior_offsets[P], NK = key_offsets[P];

  // everything derived on the host once per call: the problems, their block CSRs and contributions, the first rows
  std::vector<GraphProblem> prob(P);
  std::vector<int> cptr;
  std::vector<GraphContrib> contrib(5 * F);
  std::vector<int> fkeys(factor_keys, factor_keys + 2 * F);
  std::vector<int> qkeys(prior_keys, prior_keys + Q);
  std::vector<GraphState> st(P);
  std::vector<double> rows(16 * F);
  size_t sys = 0;
  int n_max = 0;
  for (size_t p = 0; p < P; p++) {
    GraphProblem& g = prob[p];
    g.K = (int)(key_offsets[p + 1] - key_offsets[p]);
    g.n = 6 * g.K;
    g.key0 = (int)key_offsets[p];
    g.f0 = (int)factor_offsets[p];
    g.f1 = (int)factor_offsets[p + 1];
    g.q0 = (int)prior_offsets[p];
    g.q1 = (int)prior_offsets[p + 1];
    g.cp0 = (int)cptr.size();
    g.pad = 0;
    g.sys = (long long)sys;
    sys += (size_t)g.n * g.n + g.n;
    n_max = std::max(n_max, g.n);
    cptr.resize(cptr.size() + graph_num_blocks(g.K) + 1);
    graph_contributions(g.K, g.f1 - g.f0, fkeys.data() + 2 * g.f0, g.f0, cptr.data() + g.cp0, contrib.data() + 5 * g.f0);
    align_init(st[p].a, T_init + 16 * g.key0, prm->lambda_initial);
    for (int f = g.f0; f < g.f1; f++) graph_row(T_init + 16 * g.key0, fkeys[2 * f], fkeys[2 * f + 1], rows.data() + 16 * f);
  }

  GB_ENTER(ctx);
  gb_sweep* sweep = nullptr;
  GB_CHECK(gb_sweep_create(ctx, F, factors, nullptr, &sweep));
  const gb_owned<gb_sweep> s(sweep, sweep_free);  // its blocks go back to the context's pool on every exit
  GraphCall c{};
  unsigned* d_ctr = nullptr;
  unsigned* h_ctr = nullptr;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    c.prob = cv.take<GraphProblem>(P);
    c.st = cv.take<GraphState>(P);
    c.cptr = cv.take<int>(cptr.size());
    c.contrib = cv.take<GraphContrib>(contrib.size());
    c.fkeys = cv.take<int>(2 * F);
    c.pkeys = cv.take<int>(Q);
    c.pposes = cv.take<double>(16 * Q);
    c.pw = cv.take<double>(Q);
    c.pterm = cv.take<double>(Q);
    c.T = cv.take<double>(16 * NK);
    c.Tn = cv.take<double>(16 * NK);
    c.sys = cv.take<double>(sys);
    d_ctr = cv.take<unsigned>(2);
  }));
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) { h_ctr = cv.take<unsigned>(2); }));
  c.poses = s->d_poses;
  c.poses_eval = s->d_poses_eval;
  c.out = s->d_out;
  GB_CHECK(gb_upload(ctx, {{(void*)c.prob, prob.data(), sizeof(GraphProblem) * P},
                           {c.st, st.data(), sizeof(GraphState) * P},
                           {(void*)c.cptr, cptr.data(), sizeof(int) * cptr.size()},
                           {(void*)c.contrib, contrib.data(), sizeof(GraphContrib) * contrib.size()},
                           {(void*)c.fkeys, fkeys.data(), sizeof(int) * 2 * F},
                           {(void*)c.pkeys, qkeys.data(), sizeof(int) * Q},
                           {(void*)c.pposes, prior_poses, sizeof(double) * 16 * Q},
                           {(void*)c.pw, prior_precisions, sizeof(double) * Q},
                           {c.T, T_init, sizeof(double) * 16 * NK},
                           {c.Tn, T_init, sizeof(double) * 16 * NK},
                           {c.poses, rows.data(), sizeof(double) * 16 * F},
                           {c.poses_eval, rows.data(), sizeof(double) * 16 * F}}));
  const size_t smem = sizeof(double) * graph_smem_doubles(n_max);
  GB_CUDA(cudaFuncSetAttribute(k_graph_step, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int accept_grid = (int)((P * 32 + kAcceptThreads - 1) / kAcceptThreads);
  GB_CHECK(gb_align_rounds(ctx, d_ctr, h_ctr, [&](bool need_lin) -> gb_status {
    if (need_lin) GB_CHECK(gb_launch_sweep(s.get(), GB_MODE_LINEARIZE));
    GB_CHECK(gb_launch(ctx, "k_graph_step", k_graph_step, (int)P, kGraphThreads, smem, c, d_ctr));
    GB_CHECK(gb_launch_sweep(s.get(), GB_MODE_ERROR));
    return gb_launch(ctx, "k_graph_accept", k_graph_accept, accept_grid, kAcceptThreads, 0, c, (int)P, *prm, d_ctr);
  }));
  GB_CHECK(gb_download(ctx, {{st.data(), c.st, sizeof(GraphState) * P}, {T_out, c.T, sizeof(double) * 16 * NK}}));
  for (size_t p = 0; p < P; p++) align_result(st[p].a, results[p]);
  return GB_OK;
}

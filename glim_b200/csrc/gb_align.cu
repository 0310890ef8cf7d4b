// gb_align.cu -- gb_vgicp_align: Levenberg-Marquardt registration of many VGICP problems in one call (sm_90a).
//
// Replaces the loop LevenbergMarquardtOptimizerExt runs around IntegratedVGICPFactor(Pose3(), X(current), voxelmap, frame)
// (odometry_estimation_cpu.cpp:105-150; global_mapping_pose_graph.cpp:405-417).  The rule is stated once, in
// include/glim_b200.h; its per-problem arithmetic lives in gb_align_math.cuh (also compiled for the host by the CPU test).
//
// One private gb_sweep covers every factor of every problem, in CSR order.  A round is at most four launches:
//   linearize sweep (if any problem needs a linearization) -> k_align_step -> error sweep -> k_align_accept,
// then one 8-byte device-to-host copy of the status word and a stream sync.  The host loop stops when no problem is active.
// The rounds are plain launches, not a captured graph: k_vgicp_sweep3 takes its queue head as a kernel argument that
// advances with every launch, so a captured round would replay a stale head.
#include "gb_internal.cuh"
#include "gb_align_math.cuh"

#include <math.h>
#include <float.h>
#include <string.h>

#include <algorithm>

namespace {

constexpr int kAlignThreads = 256;  // 8 problems (one warp each) per CTA

// Per problem (one warp): gather the records of a fresh linearization into the state (the error sweep that follows overwrites
// them), solve, form T' and write it into the eval-pose rows of the problem's factors.  Block 0 clears the status word.
__global__ void __launch_bounds__(kAlignThreads) k_align_step(AlignState* __restrict__ st, const int* __restrict__ off, int P, const double* __restrict__ out,
                                                               double* __restrict__ poses_eval, unsigned* __restrict__ counters) {
  if (blockIdx.x == 0 && threadIdx.x < 2) counters[threadIdx.x] = 0u;
  const int p = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= P) return;
  AlignState& s = st[p];
  if (s.status != GB_ALIGN_ACTIVE) return;
  const int f0 = off[p], f1 = off[p + 1];
  if (s.need_lin) {
    for (int k = lane; k < GB_ALIGN_STATE_ENTRIES; k += 32) {
      const double v = align_record_entry(out, f0, f1, k);
      if (k < 36) s.H[k] = v;
      else if (k < 42) s.b[k - 36] = v;
      else if (k == 42) s.e = v;
      else s.n = v;
    }
    __syncwarp();
    int active = 0;
    if (lane == 0) {
      align_linearized(s);
      active = s.status == GB_ALIGN_ACTIVE;
    }
    if (!__shfl_sync(0xffffffffu, active, 0)) return;
  }
  if (lane == 0) align_trial(s);
  __syncwarp();
  for (int k = lane; k < (f1 - f0) * 16; k += 32) poses_eval[(size_t)f0 * 16 + k] = s.Tn[k & 15];
}

// Per problem (one warp): the trial's error (sum over the problem's factors in record order), rule steps 4-5, the accepted
// pose into the linearization-pose rows; then count active problems and those that need a linearization.
__global__ void __launch_bounds__(kAlignThreads) k_align_accept(AlignState* __restrict__ st, const int* __restrict__ off, int P, const double* __restrict__ out,
                                                                 double* __restrict__ poses, gb_align_params prm, unsigned* __restrict__ counters) {
  const int p = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= P) return;
  AlignState& s = st[p];
  if (s.status != GB_ALIGN_ACTIVE) return;
  const int f0 = off[p], f1 = off[p + 1];
  int flags = 0;
  if (lane == 0) {
    align_conclude(s, prm, align_record_entry(out, f0, f1, 42));
    flags = (s.need_lin ? 1 : 0) | (s.status == GB_ALIGN_ACTIVE ? 2 : 0);
    if (flags & 2) atomicAdd(&counters[0], 1u);
    if (flags == 3) atomicAdd(&counters[1], 1u);
  }
  flags = __shfl_sync(0xffffffffu, flags, 0);
  if (flags & 1)
    for (int k = lane; k < (f1 - f0) * 16; k += 32) poses[(size_t)f0 * 16 + k] = s.T[k & 15];
}

gb_status validate(size_t P, const size_t* off, gb_factor* const* factors, const double* T_init, const gb_align_params* prm) {
  GB_REQUIRE(off && T_init && prm, "null argument");
  GB_REQUIRE(off[0] == 0, "factor_offsets[0] must be 0");
  for (size_t p = 0; p < P; p++) GB_REQUIRE(off[p + 1] > off[p], "factor_offsets must increase strictly (no empty problem)");
  GB_REQUIRE(off[P] < ((size_t)1 << 30), "too many factors");
  GB_REQUIRE(factors, "null factor list");
  for (size_t f = 0; f < off[P]; f++) GB_REQUIRE(factors[f], "null factor");
  for (size_t k = 0; k < 16 * P; k++) GB_REQUIRE(isfinite(T_init[k]), "T_init must be finite");
  return gb_align_params_check(prm);
}

}  // namespace

gb_status gb_align_params_check(const gb_align_params* prm) {
  GB_REQUIRE(prm, "null params");
  GB_REQUIRE(prm->max_iterations >= 1, "max_iterations must be >= 1");
  GB_REQUIRE(prm->lambda_factor > 1.0 && isfinite(prm->lambda_factor), "lambda_factor must be a finite number > 1");
  GB_REQUIRE(prm->lambda_initial > 0.0 && isfinite(prm->lambda_initial), "lambda_initial must be a finite number > 0");
  GB_REQUIRE(isfinite(prm->lambda_upper_bound), "lambda_upper_bound must be finite");
  // lambda shrinks by lambda_factor at most max_iterations times: it must stay a normal number (lambda == 0 would never
  // exceed the upper bound, and the rejections would not end)
  GB_REQUIRE(log(prm->lambda_initial) - prm->max_iterations * log(prm->lambda_factor) > log(DBL_MIN), "lambda_initial / lambda_factor^max_iterations underflows");
  GB_REQUIRE(!isnan(prm->relative_error_tol) && !isnan(prm->absolute_error_tol) && !isnan(prm->step_translation_tol) && !isnan(prm->step_rotation_tol), "NaN tolerance");
  return GB_OK;
}

extern "C" gb_status gb_align_default_params(gb_align_params* p) {
  GB_REQUIRE(p, "null params");
  p->max_iterations = 8;  // config_odometry_cpu.json:23
  p->lambda_initial = 1e-5;
  p->lambda_factor = 10.0;
  p->lambda_upper_bound = 1e5;
  p->relative_error_tol = 1e-5;
  p->absolute_error_tol = 0.1;              // odometry_estimation_cpu.cpp:118
  p->step_translation_tol = 1e-3;           // odometry_estimation_cpu.cpp:135
  p->step_rotation_tol = 1e-3 * M_PI / 180.0;
  return GB_OK;
}

extern "C" gb_status gb_vgicp_align(gb_ctx* ctx, size_t P, const size_t* off, gb_factor* const* factors, const double* T_init, const gb_align_params* prm, gb_align_result* results) {
  GB_REQUIRE(ctx, "null ctx");
  if (P == 0) return GB_OK;
  GB_REQUIRE(results, "null results");
  GB_CHECK(validate(P, off, factors, T_init, prm));
  const size_t F = off[P];
  GB_ENTER(ctx);
  gb_sweep* sweep = nullptr;
  GB_CHECK(gb_sweep_create(ctx, F, factors, nullptr, &sweep));
  const gb_owned<gb_sweep> s(sweep, sweep_free);  // its blocks go back to the context's pool on every exit
  // the same layout in scratch and in pinned staging: states | offsets | status word; the pinned side also stages the poses
  struct Block { AlignState* st; int* off; unsigned* ctr; } d, h;
  auto layout = [&](Carver& cv, Block& b) {
    b.st = cv.take<AlignState>(P);
    b.off = cv.take<int>(P + 1);
    b.ctr = cv.take<unsigned>(2);
  };
  double* h_poses = nullptr;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) { layout(cv, d); }));
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) {
    layout(cv, h);
    h_poses = cv.take<double>(16 * F);
  }));
  for (size_t p = 0; p < P; p++) align_init(h.st[p], T_init + 16 * p, prm->lambda_initial);
  for (size_t p = 0; p <= P; p++) h.off[p] = (int)off[p];
  for (size_t p = 0; p < P; p++)
    for (size_t f = off[p]; f < off[p + 1]; f++) memcpy(h_poses + 16 * f, T_init + 16 * p, sizeof(double) * 16);
  cudaStream_t stream = ctx->stream;
  GB_CUDA(cudaMemcpyAsync(d.st, h.st, (char*)h.ctr - (char*)h.st, cudaMemcpyHostToDevice, stream));  // states and offsets
  GB_CUDA(cudaMemcpyAsync(s->d_poses, h_poses, sizeof(double) * 16 * F, cudaMemcpyHostToDevice, stream));
  GB_CUDA(cudaMemcpyAsync(s->d_poses_eval, h_poses, sizeof(double) * 16 * F, cudaMemcpyHostToDevice, stream));
  GB_CUDA(cudaStreamSynchronize(stream));
  const int grid = (int)((P * 32 + kAlignThreads - 1) / kAlignThreads);
  bool need_lin = true;
  for (;;) {
    if (need_lin) GB_CHECK(gb_launch_sweep(s.get(), GB_MODE_LINEARIZE));
    GB_CHECK(gb_launch(ctx, "k_align_step", k_align_step, grid, kAlignThreads, 0, d.st, d.off, (int)P, s->d_out, s->d_poses_eval, d.ctr));
    GB_CHECK(gb_launch_sweep(s.get(), GB_MODE_ERROR));
    GB_CHECK(gb_launch(ctx, "k_align_accept", k_align_accept, grid, kAlignThreads, 0, d.st, d.off, (int)P, s->d_out, s->d_poses, *prm, d.ctr));
    GB_CUDA(cudaMemcpyAsync(h.ctr, d.ctr, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, stream));
    GB_CUDA(cudaStreamSynchronize(stream));
    if (h.ctr[0] == 0) break;
    need_lin = h.ctr[1] > 0;
  }
  GB_CUDA(cudaMemcpyAsync(h.st, d.st, sizeof(AlignState) * P, cudaMemcpyDeviceToHost, stream));
  GB_CUDA(cudaStreamSynchronize(stream));
  for (size_t p = 0; p < P; p++) {
    const AlignState& a = h.st[p];
    gb_align_result& r = results[p];
    memcpy(r.T_target_source, a.T, sizeof(double) * 16);
    r.error = a.e;
    r.num_inliers = a.n;
    r.lambda = a.lambda;
    r.iterations = a.iterations;
    r.trials = a.trials;
    r.status = a.status;
  }
  return GB_OK;
}

// gb_kernels_plane.cu -- the interactive viewer's plane bundle adjustment on the device (sm_90a): the patch of submap points
// around a picked point (gb_plane_patch), its auto radius (gb_plane_auto_radius), and the PlaneEVMFactor made of it
// (gb_plane_evm_factor_create, gb_plane_evm_linearize, gb_plane_evm_error).  The rules are written once in
// include/glim_b200.h; the per-factor arithmetic is gb_plane_math.cuh, which the host test build compiles as well.
//
//   selection            the participating frames (host), k_merge_transform over them at the shifted poses [R | t - c]
//                        (gb_transform_frames, without covariances), k_plane_flags (inside the sphere), a cub inclusive
//                        scan, k_plane_emit (the candidates' fp64 q, ids and, for a factor, stored local points, frame-major)
//   statistics           k_plane_reduce: one fixed-grid fp64 reduction of {n, sum q, sum q q^T} over the candidates inside a
//                        radius, whose last block turns it into the eigenvalues; one 32-byte copy back
//   factor               k_plane_moments: one CTA per participating frame, two passes over its selected points; one copy back
//   linearize / error    k_plane_evm: one CTA per factor builds C from the moments and decomposes it; its threads then fill
//                        b and the (6K)^2 Hessian
#include "gb_internal.cuh"
#include "gb_plane_math.cuh"

#include <cub/cub.cuh>
#include <cmath>
#include <new>

namespace {

constexpr int kPlaneThreads = 256;
constexpr int kReduceBlocks = 128;  // fixed: the reduction's order depends on the candidate count only

struct PlaneStatsOut {
  double n, ev[3];
};

__device__ __forceinline__ double plane_d2(double4 q) { return __dadd_rn(__dadd_rn(__dmul_rn(q.x, q.x), __dmul_rn(q.y, q.y)), __dmul_rn(q.z, q.z)); }

// v[0 .. W) summed over the block in a fixed tree order; the block's sums in v of thread 0.  sh: W x blockDim doubles.
template <int W>
__device__ void block_sum(double (&v)[W], double* sh) {
  const int t = threadIdx.x;
  for (int w = 0; w < W; w++) sh[w * blockDim.x + t] = v[w];
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (t < s)
      for (int w = 0; w < W; w++) sh[w * blockDim.x + t] += sh[w * blockDim.x + t + s];
    __syncthreads();
  }
  for (int w = 0; w < W; w++) v[w] = sh[w * blockDim.x];
  __syncthreads();
}

// flags[g] = point g (fp64 q about the centre) lies inside the sphere; NaN never does
__global__ void __launch_bounds__(kPlaneThreads) k_plane_flags(int n, const double4* __restrict__ pts, double r2, int* __restrict__ flags) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) flags[g] = plane_d2(pts[g]) < r2 ? 1 : 0;
}

// one thread per point g: a flagged point goes to slot pos[g] - 1 with its q, its id and (loc given) its stored local point
__global__ void __launch_bounds__(kPlaneThreads) k_plane_emit(int n, int K, const gb_frame* __restrict__ frames, const int* __restrict__ flags,
                                                              const int* __restrict__ pos, const double4* __restrict__ pts, double4* __restrict__ cand,
                                                              unsigned long long* __restrict__ ids, float4* __restrict__ loc) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n || !flags[g]) return;
  const gb_frame& F = frames[gb_frame_of(frames, K, g)];
  const int i = g - F.offset, o = pos[g] - 1;
  cand[o] = pts[g];
  ids[o] = ((unsigned long long)F.index << 32) | (unsigned)i;
  if (loc) loc[o] = F.p0[F.inv_perm ? F.inv_perm[i] : i];
}

// {n, sum q, sum q q^T} over the first *count candidates inside r2: block b takes the b-th contiguous share, each thread
// every blockDim-th candidate of it, in a fixed tree; the last block to finish sums the blocks' partials in block order
// and writes n and the eigenvalues (plane_stats).  *ticket is zero on entry.
__global__ void __launch_bounds__(kPlaneThreads) k_plane_reduce(const double4* __restrict__ cand, const int* __restrict__ count, double r2, double* __restrict__ partials,
                                                                unsigned* __restrict__ ticket, PlaneStatsOut* __restrict__ out) {
  __shared__ double sh[10 * kPlaneThreads];
  __shared__ bool last;
  const int n = *count;
  const int share = (n + gridDim.x - 1) / gridDim.x;
  const int begin = blockIdx.x * share, end = min(n, begin + share);
  double v[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = begin + threadIdx.x; i < end; i += blockDim.x) {
    const double4 q = cand[i];
    if (!(plane_d2(q) < r2)) continue;
    const double p[3] = {q.x, q.y, q.z};
    v[0] += 1.0;
    for (int r = 0; r < 3; r++) v[1 + r] = __dadd_rn(v[1 + r], p[r]);
    for (int r = 0; r < 3; r++)
      for (int c = r; c < 3; c++) v[4 + sym6(r, c)] = __dadd_rn(v[4 + sym6(r, c)], __dmul_rn(p[r], p[c]));
  }
  block_sum(v, sh);
  if (threadIdx.x == 0) {
    for (int w = 0; w < 10; w++) partials[10 * blockIdx.x + w] = v[w];
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int w = 0; w < 10; w++) v[w] = 0.0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x)
    for (int w = 0; w < 10; w++) v[w] = __dadd_rn(v[w], ((volatile double*)partials)[10 * b + w]);
  block_sum(v, sh);
  if (threadIdx.x == 0) {
    out->n = v[0];
    plane_stats(v[0], v + 1, v + 4, out->ev);
  }
}

// one CTA per participating frame f: the moments {N, mean, scatter} (GB_PLANE_MOMENTS) of its selected stored points, widened
// to fp64, in two passes over its share of the compacted candidates [pos[o0 - 1], pos[o1 - 1]), [o0, o1) its points
__global__ void __launch_bounds__(kPlaneThreads) k_plane_moments(const gb_frame* __restrict__ frames, const int* __restrict__ pos, const float4* __restrict__ loc,
                                                                 double* __restrict__ moments) {
  __shared__ double sh[6 * kPlaneThreads];
  const int f = blockIdx.x;
  const int o0 = frames[f].offset, o1 = o0 + frames[f].n;
  const int begin = o0 > 0 ? pos[o0 - 1] : 0, end = o1 > 0 ? pos[o1 - 1] : 0;
  double s[3] = {0, 0, 0};
  for (int i = begin + threadIdx.x; i < end; i += blockDim.x) {
    const float4 a = loc[i];
    s[0] = __dadd_rn(s[0], (double)a.x);
    s[1] = __dadd_rn(s[1], (double)a.y);
    s[2] = __dadd_rn(s[2], (double)a.z);
  }
  block_sum(s, sh);
  const double N = (double)(end - begin);
  const double m[3] = {s[0] / N, s[1] / N, s[2] / N};
  double S[6] = {0, 0, 0, 0, 0, 0};
  for (int i = begin + threadIdx.x; i < end; i += blockDim.x) {
    const float4 a = loc[i];
    const double d[3] = {__dsub_rn((double)a.x, m[0]), __dsub_rn((double)a.y, m[1]), __dsub_rn((double)a.z, m[2])};
    for (int r = 0; r < 3; r++)
      for (int c = r; c < 3; c++) S[sym6(r, c)] = __dadd_rn(S[sym6(r, c)], __dmul_rn(d[r], d[c]));
  }
  block_sum(S, sh);
  if (threadIdx.x == 0) {
    double* M = moments + GB_PLANE_MOMENTS * f;
    M[0] = N;
    for (int r = 0; r < 3; r++) M[1 + r] = end > begin ? m[r] : 0.0;
    for (int w = 0; w < 6; w++) M[4 + w] = S[w];
  }
}

// a factor of a linearization batch: its keys [key0, key0 + K) of the moments, poses and terms, and its output offsets
struct PlaneEvmDesc {
  int K, key0;
  long long h0;  // first entry of its (6K)^2 Hessian
  int b0;        // first entry of its 6K gradient
  int pad;
};

// one CTA per factor: C, pbar and N from the moments at the poses, their eigen decomposition, then (H given) the keys' terms
// and b, then every entry of H.  A degenerate factor gets H = 0, b = 0 and its error.
__global__ void __launch_bounds__(kPlaneThreads) k_plane_evm(const PlaneEvmDesc* __restrict__ descs, const double* __restrict__ moments, const double* __restrict__ poses,
                                                             const double* __restrict__ offsets, double* __restrict__ terms, double* __restrict__ H, double* __restrict__ b,
                                                             double* __restrict__ errors, int* __restrict__ status) {
  __shared__ double ev[3], U[9], pbar[3], N;
  __shared__ bool degenerate;
  const PlaneEvmDesc D = descs[blockIdx.x];
  const double* mom = moments + (size_t)GB_PLANE_MOMENTS * D.key0;
  const double* X = poses + (size_t)16 * D.key0;
  const double* o = offsets + 3 * (size_t)blockIdx.x;
  if (threadIdx.x == 0) {
    double C[9];
    plane_evm_cov(D.K, mom, X, o, C, pbar, &N);
    eigen_sym3_direct(C, ev, U);
    degenerate = plane_evm_degenerate(ev);
    errors[blockIdx.x] = ev[0];
    if (status) status[blockIdx.x] = degenerate ? GB_PLANE_EVM_DEGENERATE : GB_PLANE_EVM_OK;
  }
  __syncthreads();
  if (!H) return;
  const int n6 = 6 * D.K;
  double* Hf = H + D.h0;
  double* bf = b + D.b0;
  double* T = terms + (size_t)GB_PLANE_KEY_TERMS * D.key0;
  if (degenerate) {
    for (long long e = threadIdx.x; e < (long long)n6 * n6; e += blockDim.x) Hf[e] = 0.0;
    for (int e = threadIdx.x; e < n6; e += blockDim.x) bf[e] = 0.0;
    return;
  }
  for (int k = threadIdx.x; k < D.K; k += blockDim.x) {
    double g[6];
    plane_evm_key(mom + GB_PLANE_MOMENTS * k, X + 16 * k, o, pbar, N, U, T + GB_PLANE_KEY_TERMS * k, g);
    for (int r = 0; r < 6; r++) bf[6 * k + r] = 0.5 * g[r];
  }
  __syncthreads();
  for (long long e = threadIdx.x; e < (long long)n6 * n6; e += blockDim.x) {
    const int c = (int)(e / n6), r = (int)(e % n6);  // column-major
    Hf[e] = plane_evm_entry(r, c, T, N, ev);
  }
}

// The selection shared by the three patch calls: the candidates inside the sphere of radius r about the centre, from the
// frames within max_frame_distance of it.  Host side: the participating frames and their shifted poses; on the device, their one
// descriptor table.
struct PlaneSelection {
  std::vector<int> part;          // caller's indices of the participating frames
  size_t total = 0;               // their points
  gb_frame* d_frames = nullptr;   // their descriptors (gb_frame_table)
  int* d_pos = nullptr;           // inclusive scan of the flags; d_pos[total - 1] = the candidates
  double4* d_cand = nullptr;      // candidates' fp64 q, frame-major
  unsigned long long* d_ids = nullptr;
  float4* d_loc = nullptr;        // candidates' stored local points (factor only)
  double* d_partials = nullptr;
  unsigned* d_ticket = nullptr;
  PlaneStatsOut* d_stats = nullptr;
  double* d_moments = nullptr;    // factor only: one record per participating frame
};

// validation shared by the three patch calls: every input before any launch
gb_status plane_args(const gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* p) {
  GB_REQUIRE(ctx && p, "null argument");
  size_t total = 0;
  GB_CHECK(gb_frame_list_check(ctx, K, frames, poses, &total));
  GB_REQUIRE(gb_all_finite(poses, 16 * K), "a non-finite pose");
  GB_REQUIRE(K < ((size_t)1 << 31), "too many frames");
  for (int a = 0; a < 3; a++) GB_REQUIRE(std::isfinite(p->center[a]), "a non-finite center");
  GB_REQUIRE(std::isfinite(p->radius) && p->radius > 0.0, "radius must be positive and finite");
  GB_REQUIRE(std::isfinite(p->min_radius) && std::isfinite(p->max_radius) && p->min_radius > 0.0 && p->min_radius <= p->max_radius,
             "min_radius and max_radius must be finite with 0 < min_radius <= max_radius");
  GB_REQUIRE(std::isfinite(p->plane_eps) && p->plane_eps >= 0.0, "plane_eps must be finite and >= 0");
  GB_REQUIRE(p->max_frame_distance >= 0.0, "max_frame_distance must be >= 0 (+inf allowed)");
  return GB_OK;
}

// The candidates at radius r (selection rules 1-4): nothing launched when the participating frames hold no point.  Four
// launches otherwise (the frame transform, the flags, their scan, the emit).  Everything the calls need later is carved here.
gb_status plane_select(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* p, double r, bool local,
                       PlaneSelection& s) {
  std::vector<const gb_cloud*> pf;
  std::vector<double> shifted;
  for (size_t k = 0; k < K; k++) {
    const double* T = poses + 16 * k;
    const double u[3] = {T[12] - p->center[0], T[13] - p->center[1], T[14] - p->center[2]};
    if (!(std::sqrt((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]) <= p->max_frame_distance)) continue;
    s.part.push_back((int)k);
    s.total += frames[k]->n;
    pf.push_back(frames[k]);
    shifted.insert(shifted.end(), T, T + 16);
    for (int a = 0; a < 3; a++) shifted[shifted.size() - 4 + a] = u[a];
  }
  if (s.total == 0) return GB_OK;
  const size_t N = s.total, P = s.part.size(), cub_b = gb_cub_temp_bytes(N);
  const int n = (int)N;
  const std::vector<gb_frame> table = gb_frame_table(P, pf.data(), shifted.data(), s.part.data());
  char* d_cub;
  int* d_flags;
  double4* d_pts;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_cub = cv.take<char>(cub_b);
    s.d_frames = cv.take<gb_frame>(P);
    d_flags = cv.take<int>(N);
    s.d_pos = cv.take<int>(N);
    d_pts = cv.take<double4>(N);
    s.d_cand = cv.take<double4>(N);
    s.d_ids = cv.take<unsigned long long>(N);
    s.d_loc = local ? cv.take<float4>(N) : nullptr;
    s.d_partials = cv.take<double>(10 * kReduceBlocks);
    s.d_ticket = cv.take<unsigned>(1);
    s.d_stats = cv.take<PlaneStatsOut>(1);
    s.d_moments = cv.take<double>(GB_PLANE_MOMENTS * P);
  }));
  GB_CHECK(gb_upload(ctx, {{s.d_frames, table.data(), sizeof(gb_frame) * P}}));
  GB_CHECK(gb_transform_frames(ctx, P, s.d_frames, n, d_pts, nullptr));
  const int gb = (n + kPlaneThreads - 1) / kPlaneThreads;
  GB_CHECK(gb_launch(ctx, "k_plane_flags", k_plane_flags, gb, kPlaneThreads, 0, n, d_pts, r * r, d_flags));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, d_cub, cub_b, d_flags, s.d_pos, n);
  return gb_launch(ctx, "k_plane_emit", k_plane_emit, gb, kPlaneThreads, 0, n, (int)P, s.d_frames, d_flags, s.d_pos, d_pts, s.d_cand, s.d_ids, s.d_loc);
}

// n and the eigenvalues of the candidates inside radius r: one launch and one 32-byte copy with its synchronisation (none
// without candidates: n = 0 and NaN eigenvalues)
gb_status plane_stats_at(gb_ctx* ctx, const PlaneSelection& s, double r, size_t* n, double* ev) {
  PlaneStatsOut h{0.0, {NAN, NAN, NAN}};
  if (s.total > 0) {
    GB_CUDA(cudaMemsetAsync(s.d_ticket, 0, sizeof(unsigned), ctx->stream));
    GB_CHECK(gb_launch(ctx, "k_plane_reduce", k_plane_reduce, kReduceBlocks, kPlaneThreads, 0, s.d_cand, s.d_pos + (s.total - 1), r * r, s.d_partials, s.d_ticket,
                       s.d_stats));
    GB_CHECK(gb_download(ctx, {{&h, s.d_stats, sizeof(h)}}));
  }
  *n = (size_t)h.n;
  for (int a = 0; a < 3; a++) ev[a] = h.ev[a];
  return GB_OK;
}

void result_stats(gb_plane_patch_result* res, double r, size_t n, const double* ev) {
  res->radius = r;
  res->num_points = n;
  for (int a = 0; a < 3; a++) res->eigenvalues[a] = ev[a];
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// entry points
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_plane_patch_default_params(gb_plane_patch_params* p) {
  GB_REQUIRE(p, "null argument");
  for (int a = 0; a < 3; a++) p->center[a] = 0.0;
  p->radius = 1.0;
  p->max_frame_distance = 25.0;
  p->min_radius = 0.1;
  p->max_radius = 5.0;
  p->plane_eps = 0.01;
  return GB_OK;
}

extern "C" gb_status gb_plane_patch(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* params,
                                    gb_plane_patch_result* result, uint64_t* ids) {
  GB_REQUIRE(result, "null argument");
  GB_CHECK(plane_args(ctx, K, frames, poses, params));
  GB_ENTER(ctx);
  *result = gb_plane_patch_result{};
  PlaneSelection s;
  GB_CHECK(plane_select(ctx, K, frames, poses, params, params->radius, false, s));
  size_t n = 0;
  double ev[3];
  GB_CHECK(plane_stats_at(ctx, s, params->radius, &n, ev));
  if (ids && n > 0) GB_CHECK(gb_download(ctx, {{ids, s.d_ids, sizeof(uint64_t) * n}}));
  result_stats(result, params->radius, n, ev);
  return GB_OK;
}

extern "C" gb_status gb_plane_auto_radius(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* params,
                                          gb_plane_patch_result* result) {
  GB_REQUIRE(result, "null argument");
  GB_CHECK(plane_args(ctx, K, frames, poses, params));
  GB_ENTER(ctx);
  *result = gb_plane_patch_result{};
  const gb_plane_patch_params& p = *params;
  PlaneSelection s;
  GB_CHECK(plane_select(ctx, K, frames, poses, params, std::max(p.radius, p.max_radius), false, s));
  double r = p.radius, ev[3];
  size_t n = 0;
  GB_CHECK(plane_stats_at(ctx, s, r, &n, ev));
  for (int i = 0; i < GB_PLANE_MAX_TRIALS; i++) {
    const double trial = ev[0] / ev[2] > p.plane_eps ? r * 0.8 : r * 1.1;
    if (trial < p.min_radius || trial > p.max_radius) break;
    size_t n2 = 0;
    double ev2[3];
    GB_CHECK(plane_stats_at(ctx, s, trial, &n2, ev2));
    result->trial_radius[result->num_trials] = trial;
    result->trial_points[result->num_trials] = n2;
    result->num_trials++;
    if (n2 < 10) break;
    if (trial > p.radius && ev2[0] / ev2[2] > p.plane_eps) break;
    r = trial;
    n = n2;
    for (int a = 0; a < 3; a++) ev[a] = ev2[a];
  }
  result_stats(result, r, n, ev);
  return GB_OK;
}

extern "C" gb_status gb_plane_evm_factor_create(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, const gb_plane_patch_params* params,
                                                gb_factor** out) {
  GB_REQUIRE(out, "null argument");
  *out = nullptr;
  GB_CHECK(plane_args(ctx, K, frames, poses, params));
  GB_ENTER(ctx);
  PlaneSelection s;
  GB_CHECK(plane_select(ctx, K, frames, poses, params, params->radius, true, s));
  const size_t P = s.part.size();
  std::vector<double> mom(GB_PLANE_MOMENTS * P);
  if (s.total > 0) {
    GB_CHECK(gb_launch(ctx, "k_plane_moments", k_plane_moments, (unsigned)P, kPlaneThreads, 0, s.d_frames, s.d_pos, s.d_loc, s.d_moments));
    GB_CHECK(gb_download(ctx, {{mom.data(), s.d_moments, sizeof(double) * mom.size()}}));
  }
  size_t num_points = 0;
  for (size_t f = 0; f < P; f++) num_points += (size_t)mom[GB_PLANE_MOMENTS * f];
  GB_REQUIRE(num_points >= 3, "fewer than 3 points within the radius: PlaneEVMFactor needs at least 3");
  gb_factor* f = factor_new(ctx, GB_FACTOR_PLANE_EVM, nullptr, nullptr);
  if (!f) return GB_ERR_INTERNAL;
  for (size_t i = 0; i < P; i++) {
    if (mom[GB_PLANE_MOMENTS * i] == 0.0) continue;
    f->plane_frames.push_back(s.part[i]);
    f->plane_moments.insert(f->plane_moments.end(), mom.begin() + GB_PLANE_MOMENTS * i, mom.begin() + GB_PLANE_MOMENTS * (i + 1));
  }
  for (int a = 0; a < 3; a++) f->plane_offset[a] = params->center[a];
  f->plane_points = num_points;
  *out = f;
  return GB_OK;
}

extern "C" gb_status gb_plane_evm_factor_info(const gb_factor* f, size_t* num_keys, size_t* num_points, int32_t* frame_indices, uint64_t* key_points) {
  GB_REQUIRE(f, "null argument");
  GB_REQUIRE(f->kind == GB_FACTOR_PLANE_EVM, "not a plane factor (gb_plane_evm_factor_create)");
  GB_ENTER(f->ctx);
  const size_t K = f->plane_frames.size();
  if (num_keys) *num_keys = K;
  if (num_points) *num_points = f->plane_points;
  for (size_t k = 0; k < K; k++) {
    if (frame_indices) frame_indices[k] = f->plane_frames[k];
    if (key_points) key_points[k] = (uint64_t)f->plane_moments[GB_PLANE_MOMENTS * k];
  }
  return GB_OK;
}

// the arguments of gb_plane_evm_linearize / gb_plane_evm_error, checked before any launch, and the batch's layout
static gb_status plane_evm_args(const gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* poses, const double* errors, std::vector<PlaneEvmDesc>& descs,
                                size_t& keys, size_t& h_total) {
  GB_REQUIRE(ctx && errors, "null argument");
  GB_REQUIRE(F == 0 || (factors && poses), "null factors / poses");
  GB_REQUIRE(F < ((size_t)1 << 24), "too many factors");
  keys = h_total = 0;
  descs.resize(F);
  for (size_t f = 0; f < F; f++) {
    GB_REQUIRE(factors[f], "null factor");
    GB_REQUIRE(factors[f]->kind == GB_FACTOR_PLANE_EVM, "not a plane factor (gb_plane_evm_factor_create)");
    const size_t K = factors[f]->plane_frames.size();
    GB_REQUIRE(keys + K < ((size_t)1 << 24), "too many keys");
    descs[f] = {(int)K, (int)keys, (long long)h_total, (int)(6 * keys), 0};
    keys += K;
    h_total += 36 * K * K;
  }
  GB_REQUIRE(gb_all_finite(poses, 16 * keys), "a non-finite pose");
  return GB_OK;
}

// linearize (H and b given) or only evaluate F plane factors: one upload, one launch, one download
static gb_status plane_evm_run(gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* poses, const std::vector<PlaneEvmDesc>& descs, size_t keys, size_t h_total,
                               double* H, double* b, double* errors, int32_t* status) {
  if (F == 0) return GB_OK;
  std::vector<double> mom, off(3 * F);
  mom.reserve(GB_PLANE_MOMENTS * keys);
  for (size_t f = 0; f < F; f++) {
    mom.insert(mom.end(), factors[f]->plane_moments.begin(), factors[f]->plane_moments.end());
    for (int a = 0; a < 3; a++) off[3 * f + a] = factors[f]->plane_offset[a];
  }
  const bool lin = H != nullptr;
  PlaneEvmDesc* d_descs;
  double *d_mom, *d_poses, *d_off, *d_terms, *d_H, *d_b, *d_err;
  int* d_status;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_descs = cv.take<PlaneEvmDesc>(F);
    d_mom = cv.take<double>(mom.size());
    d_poses = cv.take<double>(16 * keys);
    d_off = cv.take<double>(3 * F);
    d_terms = lin ? cv.take<double>(GB_PLANE_KEY_TERMS * keys) : nullptr;
    d_H = lin ? cv.take<double>(h_total) : nullptr;
    d_b = lin ? cv.take<double>(6 * keys) : nullptr;
    d_err = cv.take<double>(F);
    d_status = status ? cv.take<int>(F) : nullptr;
  }));
  GB_CHECK(gb_upload(ctx, {{d_descs, descs.data(), sizeof(PlaneEvmDesc) * F}, {d_mom, mom.data(), sizeof(double) * mom.size()},
                           {d_poses, poses, sizeof(double) * 16 * keys}, {d_off, off.data(), sizeof(double) * 3 * F}}));
  GB_CHECK(gb_launch(ctx, "k_plane_evm", k_plane_evm, (unsigned)F, kPlaneThreads, 0, d_descs, d_mom, d_poses, d_off, d_terms, d_H, d_b, d_err, d_status));
  return gb_download(ctx, {{H, d_H, lin ? sizeof(double) * h_total : 0}, {b, d_b, lin ? sizeof(double) * 6 * keys : 0}, {errors, d_err, sizeof(double) * F},
                           {status, d_status, sizeof(int32_t) * F}});
}

extern "C" gb_status gb_plane_evm_linearize(gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* poses, double* H, double* b, double* errors, int32_t* status) {
  GB_REQUIRE(H && b, "null argument");
  std::vector<PlaneEvmDesc> descs;
  size_t keys = 0, h_total = 0;
  GB_CHECK(plane_evm_args(ctx, F, factors, poses, errors, descs, keys, h_total));
  GB_ENTER(ctx);
  return plane_evm_run(ctx, F, factors, poses, descs, keys, h_total, H, b, errors, status);
}

extern "C" gb_status gb_plane_evm_error(gb_ctx* ctx, size_t F, gb_factor* const* factors, const double* poses, double* errors) {
  std::vector<PlaneEvmDesc> descs;
  size_t keys = 0, h_total = 0;
  GB_CHECK(plane_evm_args(ctx, F, factors, poses, errors, descs, keys, h_total));
  GB_ENTER(ctx);
  return plane_evm_run(ctx, F, factors, poses, descs, keys, h_total, nullptr, nullptr, errors, nullptr);
}

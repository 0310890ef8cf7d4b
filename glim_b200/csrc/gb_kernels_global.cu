// gb_kernels_global.cu -- global registration on the device (sm_90a): FPFH features of a cloud (gb_cloud_estimate_fpfh), exact
// feature matching (gb_fpfh_match), RANSAC pose hypotheses (gb_ransac_align) and GNC over reciprocal matches (gb_gnc_align), the
// pieces of GLIM's manual loop closure (ManualLoopCloseModal::align_global, manual_loop_close_modal.cpp:370-468) that run
// without an initial guess.  The rules are written once in include/glim_b200.h; the per-pair and per-hypothesis arithmetic is
// gb_global_math.cuh, which the host test build compiles as well.
//
//   gb_cloud_estimate_normals  k_cloud_normals: one launch, each point's normal from its own covariance (covariance_normal,
//                           gb_cov_math.cuh, which the host test build compiles as well), into the normals plane.
//   gb_cloud_estimate_fpfh  a point grid of the cloud (gb_point_grid_build, cell 1.05 r), then k_fpfh_spfh (every point's SPFH,
//                           fp64, in scratch) and k_fpfh_final (the weighted sum of the neighbours' SPFH plus the own, stored
//                           fp32): the grid build's launches + 2.  Neighbour lists are never stored.
//   gb_fpfh_match           k_fpfh_match: one launch.
//   gb_ransac_align         a point grid of the target at the inlier resolution, the match, then per wave of kRansacWave
//                           hypotheses k_ransac_pose and k_ransac_score and one copy of the wave's counts; the host applies the
//                           selection rule and stops after the wave that holds the first hypothesis to reach the early-stop rate.
//   gb_gnc_align            a point grid of the target at kGncInlierVoxel; with more source points than samples, gb_thin, one cub
//                           compaction of the kept indices and k_gnc_gather of their features; the forward match (k_fpfh_match of
//                           the samples against the target), k_gnc_gather of the matched target rows, the backward match (those
//                           rows against every source feature), k_gnc_pairs and one cub compaction of the pairs (K stays on the
//                           device), k_gnc_solve (one CTA: the whole schedule), k_ransac_score of the one pose; one copy back and
//                           one stream synchronisation.
#include "gb_internal.cuh"
#include "gb_global_math.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <new>
#include <vector>

namespace {

constexpr int kNormalThreads = 256;
constexpr int kFpfhThreads = 128;
constexpr int kMatchThreads = 128;
constexpr int kMatchTile = 128;     // target features per shared-memory tile
constexpr int kMatchStride = 36;    // floats per staged feature: 33 padded to whole float4s
constexpr int kRansacWave = 512;    // hypotheses per wave (include/glim_b200.h states it: `evaluated` depends on it)
constexpr int kScoreThreads = 256;
constexpr int kScorePerThread = 4;
// k_gnc_solve's one CTA.  Not 1024: __launch_bounds__(1024) caps a thread at 64 registers, and thread 0's Horn solve (N and V,
// 32 doubles) then spills about 1 KB; at 512 nothing spills, and each thread takes twice the pairs, small next to the matches.
constexpr int kGncThreads = 512;

// the point grid of a cloud and the radius search over it
struct FpfhGrid {
  const int4* buckets;
  const int2* cells;
  const float4* points;
  uint32_t mask;
  int max_scan, m;
  float inv, max_d2;
};

__device__ __forceinline__ void load3(const float4 p, double* x) { x[0] = p.x; x[1] = p.y; x[2] = p.z; }

// one thread per stored point: its normal from its own covariance (covariance_normal), into the normals plane in stored order
__global__ void __launch_bounds__(kNormalThreads) k_cloud_normals(int n, const float4* __restrict__ p0, const float4* __restrict__ p1, const float* __restrict__ p2,
                                                                  float4* __restrict__ normals) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const float4 a = p0[j], b = p1[j];
  float v[3];
  covariance_normal(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, p2[j], v);
  normals[j] = make_float4(v[0], v[1], v[2], 0.f);
}

// one thread per grid record: the SPFH of the record's point, cnt_b * (100 / K) for the K neighbours, into spfh (caller order)
__global__ void __launch_bounds__(kFpfhThreads) k_fpfh_spfh(int n, FpfhGrid G, const float4* __restrict__ normals, const int* __restrict__ inv_perm,
                                                            double* __restrict__ spfh) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float4 a = G.points[3 * (size_t)r];
  const int i = grid_record_index(G.points, r);
  double ps[3], ns[3];
  load3(a, ps);
  load3(normals[inv_perm ? inv_perm[i] : i], ns);
  int cnt[kFpfhDim];
#pragma unroll
  for (int b = 0; b < kFpfhDim; b++) cnt[b] = 0;
  int K = 0;
  grid_within(G.buckets, G.mask, G.max_scan, G.cells, G.points, G.m, G.inv, G.max_d2, a.x, a.y, a.z, [&](int q) {
    const int j = grid_record_index(G.points, q);
    if (j == i) return;
    double pt[3], nt[3], f[3];
    load3(G.points[3 * (size_t)q], pt);
    load3(normals[inv_perm ? inv_perm[j] : j], nt);
    fpfh_pair(ps, ns, pt, nt, f);
    int bins[3];
    fpfh_bins(f, bins);
    cnt[bins[0]]++;
    cnt[bins[1]]++;
    cnt[bins[2]]++;
    K++;
  });
  const double inc = K > 0 ? 100.0 / (double)K : 0.0;
  double* out = spfh + (size_t)i * kFpfhDim;
#pragma unroll
  for (int b = 0; b < kFpfhDim; b++) out[b] = __dmul_rn((double)cnt[b], inc);
}

// one thread per grid record: FPFH_b = (sum_j SPFH_j,b / d2_ij) * 100 / (its block's sum) + SPFH_i,b, fp64, stored fp32
__global__ void __launch_bounds__(kFpfhThreads) k_fpfh_final(int n, FpfhGrid G, const double* __restrict__ spfh, float* __restrict__ fpfh) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float4 a = G.points[3 * (size_t)r];
  const int i = grid_record_index(G.points, r);
  double ps[3];
  load3(a, ps);
  double acc[kFpfhDim], sum[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int b = 0; b < kFpfhDim; b++) acc[b] = 0.0;
  grid_within(G.buckets, G.mask, G.max_scan, G.cells, G.points, G.m, G.inv, G.max_d2, a.x, a.y, a.z, [&](int q) {
    const int j = grid_record_index(G.points, q);
    if (j == i) return;
    double pt[3];
    load3(G.points[3 * (size_t)q], pt);
    const double d[3] = {__dsub_rn(pt[0], ps[0]), __dsub_rn(pt[1], ps[1]), __dsub_rn(pt[2], ps[2])};
    const double dd = dot3(d, d);
    if (dd == 0.0) return;
    const double* sj = spfh + (size_t)j * kFpfhDim;
#pragma unroll
    for (int b = 0; b < kFpfhDim; b++) {
      const double v = sj[b] / dd;
      acc[b] = __dadd_rn(acc[b], v);
      sum[b / kFpfhBins] = __dadd_rn(sum[b / kFpfhBins], v);
    }
  });
  double scale[3];
#pragma unroll
  for (int k = 0; k < 3; k++) scale[k] = sum[k] != 0.0 ? 100.0 / sum[k] : 0.0;
  const double* si = spfh + (size_t)i * kFpfhDim;
  float* out = fpfh + (size_t)i * kFpfhDim;
#pragma unroll
  for (int b = 0; b < kFpfhDim; b++) out[b] = (float)__dadd_rn(__dmul_rn(acc[b], scale[b / kFpfhBins]), si[b]);
}

// One thread per source feature, its 33 values in registers; target features staged through shared memory a tile at a time and
// visited in ascending index: the running argmin of d2 = sum_k (a_k - b_k)^2, summed sequentially in fp32 without contraction,
// keeps the first (smallest) index among equal distances.  NaN distances never win; -1 when nothing does.
__global__ void __launch_bounds__(kMatchThreads) k_fpfh_match(int ns, const float* __restrict__ src, int nt, const float* __restrict__ tgt, int* __restrict__ nearest) {
  __shared__ __align__(16) float tile[kMatchTile * kMatchStride];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float a[kFpfhDim];
#pragma unroll
  for (int k = 0; k < kFpfhDim; k++) a[k] = i < ns ? src[(size_t)i * kFpfhDim + k] : 0.f;
  float best = INFINITY;
  int best_j = -1;
  for (int t0 = 0; t0 < nt; t0 += kMatchTile) {
    const int cnt = min(kMatchTile, nt - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < cnt * kFpfhDim; e += blockDim.x) {
      const int t = e / kFpfhDim, k = e - t * kFpfhDim;
      tile[t * kMatchStride + k] = tgt[(size_t)t0 * kFpfhDim + e];
    }
    __syncthreads();
    for (int t = 0; t < cnt; t++) {
      const float4* b4 = reinterpret_cast<const float4*>(tile + t * kMatchStride);
      float b[kMatchStride];
#pragma unroll
      for (int k = 0; k < kMatchStride / 4; k++) {
        const float4 v = b4[k];
        b[4 * k] = v.x; b[4 * k + 1] = v.y; b[4 * k + 2] = v.z; b[4 * k + 3] = v.w;
      }
      float e0 = __fsub_rn(a[0], b[0]);
      float d2 = __fmul_rn(e0, e0);
#pragma unroll
      for (int k = 1; k < kFpfhDim; k++) {
        const float e = __fsub_rn(a[k], b[k]);
        d2 = __fadd_rn(d2, __fmul_rn(e, e));
      }
      if (d2 < best) {
        best = d2;
        best_j = t0 + t;
      }
    }
  }
  if (i < ns) nearest[i] = best_j;
}

// one thread per hypothesis h0 + k of the wave: the sample, its matches and the pose (T: 16 doubles per hypothesis, column-major);
// counts[h] = 0 for a valid sample, -1 for an invalid one
__global__ void k_ransac_pose(int h0, int w, unsigned long long seed, int ns, int dof, const int* __restrict__ nearest, const float4* __restrict__ sp0,
                              const int* __restrict__ sinv, const float4* __restrict__ tp0, const int* __restrict__ tinv, double* __restrict__ T, int* __restrict__ counts) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= w) return;
  const int h = h0 + k;
  int s[3];
  ransac_sample(seed, h, ns, s);
  bool ok = s[0] != s[1] && s[0] != s[2] && s[1] != s[2];
  double a[9], b[9];
  for (int j = 0; j < 3 && ok; j++) {
    const int t = nearest[s[j]];
    if (t < 0) { ok = false; break; }
    load3(sp0[sinv ? sinv[s[j]] : s[j]], a + 3 * j);
    load3(tp0[tinv ? tinv[t] : t], b + 3 * j);
  }
  ok = ok && ransac_pose(a, b, dof, T + 16 * (size_t)h);
  counts[h] = ok ? 0 : -1;
}

// blockIdx.y = hypothesis of the wave, x = a chunk of source points: the inliers of the chunk, one integer atomic per warp
__global__ void __launch_bounds__(kScoreThreads) k_ransac_score(int h0, int ns, const float4* __restrict__ sp0, const double* __restrict__ T, const int4* __restrict__ buckets,
                                                                uint32_t mask, int max_scan, float inv, int* __restrict__ counts) {
  const int h = h0 + (int)blockIdx.y;
  if (counts[h] < 0) return;
  const PoseF P = pose_from_colmajor(T + 16 * (size_t)h);
  int c = 0;
  const int base = blockIdx.x * kScoreThreads * kScorePerThread + threadIdx.x;
#pragma unroll
  for (int u = 0; u < kScorePerThread; u++) {
    const int j = base + u * kScoreThreads;
    if (j < ns) {
      const float4 a = sp0[j];
      c += ransac_inlier(P, a.x, a.y, a.z, buckets, mask, max_scan, inv) ? 1 : 0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c > 0) atomicAdd(&counts[h], c);
}

// rows[r] = the 33 features of row idx[r] of feat, or a NaN row (which matches nothing) for idx[r] < 0; one thread per value
__global__ void k_gnc_gather(int m, const int* __restrict__ idx, const float* __restrict__ feat, float* __restrict__ rows) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)m * kFpfhDim) return;
  const int r = (int)(e / kFpfhDim), k = (int)(e - (size_t)r * kFpfhDim);
  const int i = idx[r];
  rows[e] = i >= 0 ? feat[(size_t)i * kFpfhDim + k] : __int_as_float(0x7fffffff);
}

// one thread per sample r (source index i = samples[r], or r without sampling): pair (i, fwd[r]), kept iff the match exists, the
// source feature nearest to it is i (back[r]) and both fp32 positions are finite
__global__ void k_gnc_pairs(int m, const int* __restrict__ samples, const int* __restrict__ fwd, const int* __restrict__ back, const float4* __restrict__ sp0,
                            const int* __restrict__ sinv, const float4* __restrict__ tp0, const int* __restrict__ tinv, int2* __restrict__ all, int* __restrict__ flags) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const int i = samples ? samples[r] : r, j = fwd[r];
  bool ok = j >= 0 && back[r] == i;
  if (ok) {
    const float4 a = sp0[sinv ? sinv[i] : i], b = tp0[tinv ? tinv[j] : j];
    ok = isfinite(a.x) && isfinite(a.y) && isfinite(a.z) && isfinite(b.x) && isfinite(b.y) && isfinite(b.z);
  }
  all[r] = make_int2(i, j);
  flags[r] = ok ? 1 : 0;
}

// What k_gnc_solve leaves for the host (one copy): the pose, then inliers (k_ransac_score's count, reset here), iterations,
// status and K (written by the pair compaction).
struct GncOut {
  double T[16];
  int inliers, iterations, status, K;
};

// The sum of every thread's v over the block, the same on every run: a shuffle tree in each warp, then threads 0 .. N-1 fold
// the warp partials in warp order into out (shared).  Ends with the block synchronised.
template <int N, typename Op>
__device__ __forceinline__ void gnc_block_reduce(double (&v)[N], double* part, double* out, Op op) {
#pragma unroll
  for (int k = 0; k < N; k++)
    for (int o = 16; o > 0; o >>= 1) v[k] = op(v[k], __shfl_down_sync(0xffffffffu, v[k], o));
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < N; k++) part[(threadIdx.x >> 5) * N + k] = v[k];
  __syncthreads();
  if (threadIdx.x < N) {
    double s = part[threadIdx.x];
    for (int w = 1; w < kGncThreads / 32; w++) s = op(s, part[w * N + threadIdx.x]);
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// The whole Geman-McClure schedule of include/glim_b200.h in one CTA, over the K pairs of out->K (thread t owns k = t mod
// kGncThreads).  Passes: the shifts (the means of a and b), the unit-weight pose, the largest r^2 at it, then one pass per
// iteration (r^2 at the previous T, the weight, the 16 sums) after which thread 0 solves the pose and steps mu.  The weights of
// the last iteration go to weights[k].  K < 3: DEGENERATE, T = I, 0 iterations, weights 0.
__global__ void __launch_bounds__(kGncThreads) k_gnc_solve(const int2* __restrict__ pairs, const float4* __restrict__ sp0, const int* __restrict__ sinv,
                                                           const float4* __restrict__ tp0, const int* __restrict__ tinv, int dof, double* __restrict__ weights,
                                                           GncOut* __restrict__ out) {
  __shared__ double part[(kGncThreads / 32) * kGncSums];
  __shared__ double red[kGncSums];
  __shared__ double T[16], shift[6], mu;
  const int K = out->K, tid = threadIdx.x;
  const auto add = [](double x, double y) { return __dadd_rn(x, y); };
  const auto load = [&](int k, double* a, double* b) {
    const int2 p = pairs[k];
    load3(sp0[sinv ? sinv[p.x] : p.x], a);
    load3(tp0[tinv ? tinv[p.y] : p.y], b);
  };
  if (K < 3) {
    if (tid < 16) out->T[tid] = tid % 5 == 0 ? 1.0 : 0.0;
    if (tid == 0) { out->inliers = 0; out->iterations = 0; out->status = GB_GNC_DEGENERATE; }
    if (weights && tid < K) weights[tid] = 0.0;
    return;
  }
  {
    double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = tid; k < K; k += kGncThreads) {
      double a[3], b[3];
      load(k, a, b);
      for (int r = 0; r < 3; r++) { v[r] = __dadd_rn(v[r], a[r]); v[3 + r] = __dadd_rn(v[3 + r], b[r]); }
    }
    gnc_block_reduce(v, part, red, add);
    if (tid < 6) shift[tid] = red[tid] / (double)K;
    __syncthreads();
  }
  int iterations = 0;
  for (int it = -1;; it++) {  // it = -1: the unit-weight pose
    const bool last = it >= 0 && mu == kGncMinScale;
    double v[kGncSums];
#pragma unroll
    for (int s = 0; s < kGncSums; s++) v[s] = 0.0;
    for (int k = tid; k < K; k += kGncThreads) {
      double a[3], b[3];
      load(k, a, b);
      double w = 1.0;
      if (it >= 0) {
        w = gnc_weight(mu, gnc_residual2(T, a, b));
        if (last && weights) weights[k] = w;
      }
      for (int r = 0; r < 3; r++) { a[r] = __dsub_rn(a[r], shift[r]); b[r] = __dsub_rn(b[r], shift[3 + r]); }
      gnc_accumulate(v, w, a, b);
    }
    gnc_block_reduce(v, part, red, add);
    if (tid == 0) gnc_pose(red, shift, shift + 3, dof, T);
    __syncthreads();
    if (it < 0) {
      double m[1] = {0.0};
      for (int k = tid; k < K; k += kGncThreads) {
        double a[3], b[3];
        load(k, a, b);
        m[0] = fmax(m[0], gnc_residual2(T, a, b));
      }
      gnc_block_reduce(m, part, red, [](double x, double y) { return fmax(x, y); });
      if (tid == 0) mu = gnc_initial_scale(red[0]);
      __syncthreads();
      continue;
    }
    iterations++;
    if (last) break;
    if (tid == 0) mu = gnc_next_scale(mu);
    __syncthreads();
  }
  if (tid < 16) out->T[tid] = T[tid];
  if (tid == 0) { out->inliers = 0; out->iterations = iterations; out->status = GB_GNC_FOUND; }
}

FpfhGrid fpfh_grid(const gb_voxelmap* g, int m, float max_d2) {
  return FpfhGrid{g->buckets, g->cells, g->voxels, (uint32_t)(g->num_buckets - 1), g->max_scan, m, g->inv_res, max_d2};
}

gb_status match_launch(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source, int* d_nearest) {
  if (source->n == 0) return GB_OK;
  return gb_launch(ctx, "k_fpfh_match", k_fpfh_match, (int)((source->n + kMatchThreads - 1) / kMatchThreads), kMatchThreads, 0, (int)source->n, source->fpfh,
                   (int)target->n, target->fpfh, d_nearest);
}

gb_status match_args(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source) {
  GB_REQUIRE(ctx && target && source, "null argument");
  GB_REQUIRE(target->fpfh && source->fpfh, "a cloud without FPFH features (gb_cloud_estimate_fpfh)");
  GB_REQUIRE(target->device == ctx->device && source->device == ctx->device, "a cloud lives on another device");
  return GB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// entry points
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_cloud_estimate_normals(gb_ctx* ctx, gb_cloud* cloud) {
  GB_REQUIRE(ctx && cloud, "null argument");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(cloud->covs, "normals are estimated from covariances: the cloud carries none");
  GB_ENTER(ctx);
  {  // the features were computed from the old normals: their block goes back to the pool here
    gb_dev_block old(ctx->device);
    old.hand_over(cloud->f_base);
    cloud->fpfh = nullptr;
  }
  const size_t n = cloud->n;
  if (n == 0) return GB_OK;
  gb_dev_block block(ctx->device);  // a cloud built without normals: a block of their own, handed over on success
  float4* normals = cloud->normals;
  if (!normals) GB_CHECK(gb_dev_carve(ctx, block, [&](Carver& cv) { normals = cv.take<float4>(n); }));
  GB_CHECK(gb_launch(ctx, "k_cloud_normals", k_cloud_normals, (int)((n + kNormalThreads - 1) / kNormalThreads), kNormalThreads, 0, (int)n, cloud->p0, cloud->p1,
                     cloud->p2, normals));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (!cloud->normals) {
    block.hand_over(cloud->n_base);
    cloud->normals = normals;
  }
  return GB_OK;
}

extern "C" gb_status gb_cloud_normals(const gb_cloud* cloud, float* out) {
  GB_REQUIRE(cloud && out, "null argument");
  if (cloud->n == 0) return GB_OK;
  GB_REQUIRE(cloud->normals, "the cloud has no normals (gb_cloud_estimate_normals)");
  std::vector<float4> h(cloud->n);
  std::vector<int> perm;
  // every producer returned after its stream had drained: plain synchronous copies are safe
  GB_CUDA(cudaMemcpy(h.data(), cloud->normals, sizeof(float4) * cloud->n, cudaMemcpyDefault));
  if (cloud->perm) { perm.resize(cloud->n); GB_CUDA(cudaMemcpy(perm.data(), cloud->perm, sizeof(int) * cloud->n, cudaMemcpyDefault)); }
  for (size_t j = 0; j < cloud->n; j++) {
    float* o = out + 3 * (cloud->perm ? (size_t)perm[j] : j);  // stored slot j holds the caller's point perm[j]
    o[0] = h[j].x; o[1] = h[j].y; o[2] = h[j].z;
  }
  return GB_OK;
}

extern "C" gb_status gb_cloud_estimate_fpfh(gb_ctx* ctx, gb_cloud* cloud, double search_radius) {
  GB_REQUIRE(ctx && cloud, "null argument");
  GB_REQUIRE(std::isfinite(search_radius) && search_radius > 0.0, "search_radius must be positive and finite");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(cloud->n == 0 || cloud->normals, "FPFH needs the cloud's normals");
  GB_ENTER(ctx);
  const size_t n = cloud->n;
  gb_dev_block block(ctx->device);  // replaces the old features only on success
  float* fpfh = nullptr;
  GB_CHECK(gb_dev_carve(ctx, block, [&](Carver& cv) { fpfh = cv.take<float>(kFpfhDim * n); }));
  if (n > 0) {
    gb_point_grid* gh = nullptr;
    const gb_status st = gb_point_grid_build(ctx, cloud, 1.05 * search_radius, &gh);
    gb_owned<gb_point_grid> grid(gh, grid_release);
    GB_CHECK(st);
    const gb_voxelmap* g = grid_map(gh);
    const float max_d2 = (float)(search_radius * search_radius);
    const int m = grid_half_width(g->inv_res, max_d2, g->key_extent);
    if (m > kGridMaxHalfWidth) {
      gb_set_error("FPFH search half-width %d exceeds %d", m, kGridMaxHalfWidth);
      return GB_ERR_INTERNAL;
    }
    double* spfh = nullptr;
    GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) { spfh = cv.take<double>(kFpfhDim * n); }));
    const FpfhGrid G = fpfh_grid(g, m, max_d2);
    const int blocks = (int)((n + kFpfhThreads - 1) / kFpfhThreads);
    GB_CHECK(gb_launch(ctx, "k_fpfh_spfh", k_fpfh_spfh, blocks, kFpfhThreads, 0, (int)n, G, cloud->normals, cloud->inv_perm, spfh));
    GB_CHECK(gb_launch(ctx, "k_fpfh_final", k_fpfh_final, blocks, kFpfhThreads, 0, (int)n, G, spfh, fpfh));
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
      gb_set_error("FPFH estimation failed: %s", cudaGetErrorString(cudaGetLastError()));
      return GB_ERR_CUDA;
    }
  }
  block.hand_over(cloud->f_base);
  cloud->fpfh = fpfh;
  return GB_OK;
}

extern "C" gb_status gb_cloud_fpfh(const gb_cloud* cloud, float* out) {
  GB_REQUIRE(cloud && out, "null argument");
  GB_REQUIRE(cloud->fpfh, "the cloud has no FPFH features (gb_cloud_estimate_fpfh)");
  if (cloud->n) GB_CUDA(cudaMemcpy(out, cloud->fpfh, sizeof(float) * kFpfhDim * cloud->n, cudaMemcpyDefault));
  return GB_OK;
}

extern "C" gb_status gb_fpfh_match(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source, int32_t* nearest) {
  GB_CHECK(match_args(ctx, target, source));
  GB_REQUIRE(nearest || source->n == 0, "null output");
  GB_ENTER(ctx);
  const size_t ns = source->n;
  if (ns == 0) return GB_OK;
  int* d_nearest = nullptr;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) { d_nearest = cv.take<int>(ns); }));
  GB_CHECK(match_launch(ctx, target, source, d_nearest));
  return gb_download(ctx, {{nearest, d_nearest, sizeof(int) * ns}});
}

extern "C" gb_status gb_ransac_default_params(gb_ransac_params* p) {
  GB_REQUIRE(p, "null argument");
  p->max_iterations = 5000;
  p->early_stop_inlier_rate = 0.9;
  p->inlier_voxel_resolution = 1.0;
  p->dof = 4;
  p->seed = 53123;
  return GB_OK;
}

extern "C" gb_status gb_ransac_align(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source, const gb_ransac_params* prm, gb_ransac_result* result,
                                     int32_t* hypothesis_inliers) {
  GB_REQUIRE(prm && result, "null argument");
  GB_REQUIRE(prm->max_iterations >= 1 && prm->max_iterations <= (1 << 28), "max_iterations must be in [1, 2^28]");
  GB_REQUIRE(std::isfinite(prm->early_stop_inlier_rate) && prm->early_stop_inlier_rate > 0.0, "early_stop_inlier_rate must be positive and finite");
  GB_REQUIRE(std::isfinite(prm->inlier_voxel_resolution) && prm->inlier_voxel_resolution > 0.0, "inlier_voxel_resolution must be positive and finite");
  GB_REQUIRE(prm->dof == 4 || prm->dof == 6, "dof must be 4 or 6");
  GB_CHECK(match_args(ctx, target, source));
  GB_REQUIRE(source->n >= 1 && target->n >= 1, "empty cloud");
  GB_ENTER(ctx);
  // the grid first: its build carves the context's scratch, which then holds this call's arrays
  gb_point_grid* gh = nullptr;
  GB_CHECK(gb_point_grid_build(ctx, target, prm->inlier_voxel_resolution, &gh));
  gb_owned<gb_point_grid> grid(gh, grid_release);
  const gb_voxelmap* g = grid_map(gh);
  const int ns = (int)source->n, H = prm->max_iterations;
  int *d_nearest, *d_counts, *h_counts;
  double *d_T, *h_T;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_nearest = cv.take<int>((size_t)ns);
    d_counts = cv.take<int>((size_t)H);
    d_T = cv.take<double>(16 * (size_t)H);
  }));
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) {
    h_counts = cv.take<int>((size_t)H);
    h_T = cv.take<double>(16);
  }));
  GB_CHECK(match_launch(ctx, target, source, d_nearest));
  // the rule of include/glim_b200.h: the lowest h whose rate reaches the early-stop rate, else the most inliers (ties: lowest h)
  int best = -1, best_count = 0, stop = -1, evaluated = 0;
  for (int h0 = 0; h0 < H && stop < 0; h0 += kRansacWave) {
    const int w = std::min(kRansacWave, H - h0);
    GB_CHECK(gb_launch(ctx, "k_ransac_pose", k_ransac_pose, (w + 127) / 128, 128, 0, h0, w, (unsigned long long)prm->seed, ns, prm->dof, d_nearest, source->p0,
                       source->inv_perm, target->p0, target->inv_perm, d_T, d_counts));
    const dim3 sgrid((unsigned)((ns + kScoreThreads * kScorePerThread - 1) / (kScoreThreads * kScorePerThread)), (unsigned)w);
    GB_CHECK(gb_launch(ctx, "k_ransac_score", k_ransac_score, sgrid, kScoreThreads, 0, h0, ns, source->p0, d_T, g->buckets, (uint32_t)(g->num_buckets - 1),
                       g->max_scan, g->inv_res, d_counts));
    GB_CUDA(cudaMemcpyAsync(h_counts + h0, d_counts + h0, sizeof(int) * w, cudaMemcpyDeviceToHost, ctx->stream));
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    evaluated = h0 + w;
    for (int h = h0; h < h0 + w; h++) {
      const int c = h_counts[h];
      if (c > best_count) { best_count = c; best = h; }
      if (stop < 0 && c >= 0 && (double)c / (double)ns >= prm->early_stop_inlier_rate) stop = h;
    }
  }
  memset(result, 0, sizeof(*result));
  for (int k = 0; k < 16; k++) result->T_target_source[k] = (k % 5 == 0) ? 1.0 : 0.0;
  const int chosen = stop >= 0 ? stop : best;
  result->evaluated = evaluated;
  result->best_hypothesis = -1;
  result->status = GB_RANSAC_DEGENERATE;
  if (chosen >= 0) {
    GB_CUDA(cudaMemcpyAsync(h_T, d_T + 16 * (size_t)chosen, sizeof(double) * 16, cudaMemcpyDeviceToHost, ctx->stream));
    GB_CUDA(cudaStreamSynchronize(ctx->stream));
    memcpy(result->T_target_source, h_T, sizeof(double) * 16);
    result->best_hypothesis = chosen;
    result->inliers = h_counts[chosen];
    result->inlier_rate = (double)h_counts[chosen] / (double)ns;
    result->status = stop >= 0 ? GB_RANSAC_EARLY_STOP : GB_RANSAC_FOUND;
  }
  if (hypothesis_inliers) {
    for (int h = 0; h < H; h++) hypothesis_inliers[h] = h < evaluated ? h_counts[h] : -2;
  }
  return GB_OK;
}

extern "C" gb_status gb_gnc_default_params(gb_gnc_params* p) {
  GB_REQUIRE(p, "null argument");
  p->max_init_samples = 10000;
  p->dof = 4;
  p->seed = 53123;
  return GB_OK;
}

extern "C" gb_status gb_gnc_align(gb_ctx* ctx, const gb_cloud* target, const gb_cloud* source, const gb_gnc_params* prm, gb_gnc_result* result, int32_t* pairs,
                                  double* weights) {
  GB_REQUIRE(prm && result, "null argument");
  GB_REQUIRE(prm->max_init_samples >= 1 && prm->max_init_samples <= (1 << 28), "max_init_samples must be in [1, 2^28]");
  GB_REQUIRE(prm->dof == 4 || prm->dof == 6, "dof must be 4 or 6");
  GB_CHECK(match_args(ctx, target, source));
  GB_REQUIRE(source->n >= 1 && target->n >= 1, "empty cloud");
  GB_ENTER(ctx);
  // the grid first: its build carves the context's scratch, which then holds this call's arrays
  gb_point_grid* gh = nullptr;
  GB_CHECK(gb_point_grid_build(ctx, target, kGncInlierVoxel, &gh));
  gb_owned<gb_point_grid> grid(gh, grid_release);
  const gb_voxelmap* g = grid_map(gh);
  const int ns = (int)source->n, nt = (int)target->n;
  const bool sampled = ns > prm->max_init_samples;
  const int m = sampled ? prm->max_init_samples : ns;
  size_t cub_b = 0, select_b = 0;
  cub::DeviceSelect::Flagged(nullptr, select_b, (const int2*)nullptr, (const int*)nullptr, (int2*)nullptr, (int*)nullptr, m);
  cub_b = select_b;
  if (sampled) {
    cub::DeviceSelect::Flagged(nullptr, select_b, thrust::counting_iterator<int>(0), (const int*)nullptr, (int*)nullptr, (int*)nullptr, ns);
    cub_b = std::max({cub_b, select_b, gb_cub_temp_bytes((size_t)ns)});
  }
  gb_sort_tmp t{};
  void* d_cub;
  int *d_keep = nullptr, *d_samples = nullptr, *d_fwd, *d_back, *d_flags;
  float* d_rows;
  int2 *d_all, *d_pairs;
  double* d_w;
  GncOut* d_out;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_cub = cv.take<char>(cub_b);
    if (sampled) {
      t = gb_take_sort_tmp(cv, (size_t)ns, d_cub, cub_b);
      d_keep = cv.take<int>((size_t)ns);
      d_samples = cv.take<int>((size_t)m);
    }
    d_rows = cv.take<float>((size_t)m * kFpfhDim);
    d_fwd = cv.take<int>((size_t)m);
    d_back = cv.take<int>((size_t)m);
    d_flags = cv.take<int>((size_t)m);
    d_all = cv.take<int2>((size_t)m);
    d_pairs = cv.take<int2>((size_t)m);
    d_w = cv.take<double>((size_t)m);
    d_out = cv.take<GncOut>(1);
  }));
  GncOut* h_out;
  int2* h_pairs = nullptr;
  double* h_w = nullptr;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) {
    h_out = cv.take<GncOut>(1);
    if (pairs) h_pairs = cv.take<int2>((size_t)m);
    if (weights) h_w = cv.take<double>((size_t)m);
  }));
  const int mb = (m + kMatchThreads - 1) / kMatchThreads;
  const int gather_blocks = (int)(((size_t)m * kFpfhDim + 255) / 256);
  const float* src_rows = source->fpfh;
  if (sampled) {  // the m smallest rg_hash(seed, i), in ascending i
    GB_CHECK(gb_thin(ctx, ns, nullptr, nullptr, m, (unsigned long long)prm->seed, t, d_keep));
    GB_CUB(ctx, cub::DeviceSelect::Flagged, d_cub, cub_b, thrust::counting_iterator<int>(0), d_keep, d_samples, &d_out->K, ns);
    GB_CHECK(gb_launch(ctx, "k_gnc_gather", k_gnc_gather, gather_blocks, 256, 0, m, d_samples, source->fpfh, d_rows));
    src_rows = d_rows;
  }
  GB_CHECK(gb_launch(ctx, "k_fpfh_match", k_fpfh_match, mb, kMatchThreads, 0, m, src_rows, nt, target->fpfh, d_fwd));
  GB_CHECK(gb_launch(ctx, "k_gnc_gather", k_gnc_gather, gather_blocks, 256, 0, m, d_fwd, target->fpfh, d_rows));
  GB_CHECK(gb_launch(ctx, "k_fpfh_match", k_fpfh_match, mb, kMatchThreads, 0, m, d_rows, ns, source->fpfh, d_back));
  GB_CHECK(gb_launch(ctx, "k_gnc_pairs", k_gnc_pairs, (m + 255) / 256, 256, 0, m, d_samples, d_fwd, d_back, source->p0, source->inv_perm, target->p0, target->inv_perm,
                     d_all, d_flags));
  GB_CUB(ctx, cub::DeviceSelect::Flagged, d_cub, cub_b, d_all, d_flags, d_pairs, &d_out->K, m);
  GB_CHECK(gb_launch(ctx, "k_gnc_solve", k_gnc_solve, 1, kGncThreads, 0, d_pairs, source->p0, source->inv_perm, target->p0, target->inv_perm, prm->dof,
                     weights ? d_w : nullptr, d_out));
  const int sblocks = (ns + kScoreThreads * kScorePerThread - 1) / (kScoreThreads * kScorePerThread);
  GB_CHECK(gb_launch(ctx, "k_ransac_score", k_ransac_score, dim3((unsigned)sblocks, 1u), kScoreThreads, 0, 0, ns, source->p0, d_out->T, g->buckets,
                     (uint32_t)(g->num_buckets - 1), g->max_scan, g->inv_res, &d_out->inliers));
  GB_CUDA(cudaMemcpyAsync(h_out, d_out, sizeof(GncOut), cudaMemcpyDeviceToHost, ctx->stream));
  if (pairs) GB_CUDA(cudaMemcpyAsync(h_pairs, d_pairs, sizeof(int2) * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
  if (weights) GB_CUDA(cudaMemcpyAsync(h_w, d_w, sizeof(double) * (size_t)m, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(cudaStreamSynchronize(ctx->stream));
  memset(result, 0, sizeof(*result));
  memcpy(result->T_target_source, h_out->T, sizeof(double) * 16);
  result->inliers = h_out->inliers;
  result->inlier_rate = (double)h_out->inliers / (double)ns;
  result->samples = m;
  result->correspondences = h_out->K;
  result->iterations = h_out->iterations;
  result->status = h_out->status;
  const size_t K = (size_t)h_out->K;
  if (pairs) memcpy(pairs, h_pairs, sizeof(int2) * K);
  if (weights) memcpy(weights, h_w, sizeof(double) * K);
  return GB_OK;
}

// gb_kernels_segment.cu -- the map editor's segmentation on the device (sm_90a): submaps concatenated into one world-frame
// cloud (gb_concat_frames) and region growing from a picked point (gb_region_growing).  The rules are written once in
// include/glim_b200.h; the per-point and per-pair arithmetic is gb_segment_math.cuh, which the host test build compiles as well.
//
//   gb_concat_frames    k_merge_transform over every frame through one descriptor table (gb_transform_frames, shared with
//                       gb_merge_frames), k_concat_flags (the window), a cub inclusive scan of the flags, k_concat_emit (the
//                       kept points' fp32 planes, rotated normals and ids in output order), one copy of the kept count and a
//                       stream synchronisation, then gb_cloud_build and the copy of the ids.
//   gb_region_growing   the point grids of the cloud (gb_point_grid_build at 1.05 distance_threshold, and at 1.05
//                       dilation_radius), then k_rg_init (every parent its own index; the seed by a 64-bit atomicMin of
//                       seg_seed_key), k_rg_hook (one thread per grid record: each join (i, j > i) hooked once, ECL-CC),
//                       k_rg_label (the labels, which also compress the parents, the region and the counts), k_rg_dilate,
//                       and one cub compaction of the selection; one copy back and one stream synchronisation.
#include "gb_internal.cuh"
#include "gb_segment_math.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <cmath>
#include <cstring>
#include <new>

namespace {

constexpr int kSegThreads = 256;
constexpr int kHookThreads = 128;

// what gb_concat_frames' emit needs of frame k beyond the shared transform: its normals, its storage order, R row-major
struct ConcatFrame {
  const float4* normals;
  const int* inv_perm;
  double R[9];
};

// flags[g] = 1 iff point g of the concatenation (fp64 q) is kept: always without a window
__global__ void k_concat_flags(int n, const double4* __restrict__ pts, int windowed, double inv, int3 lo, int3 hi, int* __restrict__ flags) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const double4 p = pts[g];
  const double q[3] = {p.x, p.y, p.z};
  const int l[3] = {lo.x, lo.y, lo.z}, h[3] = {hi.x, hi.y, hi.z};
  flags[g] = !windowed || seg_in_window(q, inv, l, h) ? 1 : 0;
}

// one thread per point g of the concatenation: a kept point goes to slot pos[g] - 1 as fp32 planes (zero covariances unless
// every frame has them), its rotated normal and its id
__global__ void k_concat_emit(int n, int K, const int* __restrict__ offsets, const ConcatFrame* __restrict__ frames, const int* __restrict__ flags,
                              const int* __restrict__ pos, const double4* __restrict__ pts, const double* __restrict__ cov6, int covs, float4* __restrict__ s0,
                              float4* __restrict__ s1, float* __restrict__ s2, float4* __restrict__ sn, unsigned long long* __restrict__ ids) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n || !flags[g]) return;
  int a = 0, b = K - 1;  // the last frame whose first point is at or before g
  while (a < b) {
    const int mid = (a + b + 1) / 2;
    if (offsets[mid] <= g) a = mid; else b = mid - 1;
  }
  const int i = g - offsets[a], o = pos[g] - 1;
  const double4 p = pts[g];
  const double* c = cov6 + 6 * (size_t)g;
  s0[o] = make_float4((float)p.x, (float)p.y, (float)p.z, covs ? (float)c[0] : 0.f);
  s1[o] = covs ? make_float4((float)c[1], (float)c[2], (float)c[3], (float)c[4]) : make_float4(0.f, 0.f, 0.f, 0.f);
  s2[o] = covs ? (float)c[5] : 0.f;
  if (sn) {
    const ConcatFrame& F = frames[a];
    const float4 nr = F.normals[F.inv_perm ? F.inv_perm[i] : i];
    float v[3];
    seg_rotate_normal(F.R, nr.x, nr.y, nr.z, v);
    sn[o] = make_float4(v[0], v[1], v[2], 0.f);
  }
  ids[o] = ((unsigned long long)a << 32) | (unsigned)i;
}

// What gb_region_growing leaves for the host, ahead of the selection and the labels in one copy.
struct RgOut {
  unsigned long long seed_key;  // seg_seed_key of the seed, ~0 for none
  int num_region, num_components, num_selected, pad;
};

__device__ __forceinline__ void warp_count(bool c, int* counter) {
  const unsigned b = __ballot_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(counter, __popc(b));
}

// one thread per stored slot: parent[i] = i for its original index i, and the seed's key (the warp's minimum, then one atomic)
__global__ void __launch_bounds__(kSegThreads) k_rg_init(int n, const float4* __restrict__ p0, const int* __restrict__ perm, float qx, float qy, float qz,
                                                         int* __restrict__ parent, RgOut* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long key = ~0ull;
  if (j < n) {
    const int i = perm ? perm[j] : j;
    parent[i] = i;
    key = seg_seed_key(p0[j], qx, qy, qz, i);
  }
  for (int o = 16; o > 0; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
  if ((threadIdx.x & 31) == 0 && key != ~0ull) atomicMin(&out->seed_key, key);
}

// one thread per record of the connectivity grid (point i): every join (i, j) with j > i, hooked
__global__ void __launch_bounds__(kHookThreads) k_rg_hook(int n, const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells,
                                                          const float4* __restrict__ points, int m, float inv, float max_d2, const float4* __restrict__ normals,
                                                          const int* __restrict__ inv_perm, double cos_t, int* __restrict__ parent) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float4 a = points[3 * (size_t)r];
  if (!seg_keyed(a.x, a.y, a.z, inv)) return;
  const int i = grid_record_index(points, r);
  const float4 ni = normals[inv_perm ? inv_perm[i] : i];
  grid_within(buckets, mask, max_scan, cells, points, m, inv, max_d2, a.x, a.y, a.z, [&](int q) {
    const int j = grid_record_index(points, q);
    if (j <= i) return;
    const float4 nj = normals[inv_perm ? inv_perm[j] : j];
    if (seg_normals_join(ni.x, ni.y, ni.z, nj.x, nj.y, nj.z, cos_t)) seg_hook(parent, i, j);
  });
}

// one thread per stored slot (original index i): labels[i] = its root (the component's minimum index, also written back as
// its parent) or -1, region[i] = label == the seed's label, and the component and region counts
__global__ void __launch_bounds__(kSegThreads) k_rg_label(int n, const float4* __restrict__ p0, const int* __restrict__ perm, int* __restrict__ parent,
                                                          int* __restrict__ labels, int* __restrict__ region, RgOut* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  bool root = false, in = false;
  if (j < n) {
    const int i = perm ? perm[j] : j;
    const float4 a = p0[j];
    int label = -1;
    if (isfinite(a.x) && isfinite(a.y) && isfinite(a.z)) {
      label = seg_find(parent, i);
      parent[i] = label;
    }
    const unsigned long long key = out->seed_key;
    in = label >= 0 && key != ~0ull && label == seg_find(parent, (int)(uint32_t)key);
    root = label == i;
    labels[i] = label;
    region[i] = in ? 1 : 0;
  }
  warp_count(root, &out->num_components);
  warp_count(in, &out->num_region);
}

// one thread per record of the dilation grid (point j): sel[j] = j in R, or j finite and keyed with a point of R within the
// dilation radius
__global__ void __launch_bounds__(kHookThreads) k_rg_dilate(int n, const int4* __restrict__ buckets, uint32_t mask, int max_scan, const int2* __restrict__ cells,
                                                            const float4* __restrict__ points, int m, float inv, float max_d2, const int* __restrict__ region,
                                                            int* __restrict__ sel) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const int j = grid_record_index(points, r);
  int s = region[j];
  if (!s) {
    const float4 a = points[3 * (size_t)r];
    s = seg_keyed(a.x, a.y, a.z, inv) && seg_grid_any(buckets, mask, max_scan, cells, points, m, inv, max_d2, a.x, a.y, a.z, region) ? 1 : 0;
  }
  sel[j] = s;
}

void grid_release(gb_point_grid* g) { gb_point_grid_destroy(g); }

// a point grid of the cloud at 1.05 r and its search half-width for (float)(r^2)
gb_status rg_grid(gb_ctx* ctx, const gb_cloud* cloud, double r, gb_owned<gb_point_grid>& grid, int& m, float& max_d2) {
  gb_point_grid* gh = nullptr;
  const gb_status st = gb_point_grid_build(ctx, cloud, 1.05 * r, &gh);
  grid.reset(gh);
  GB_CHECK(st);
  const gb_voxelmap* g = grid_map(gh);
  max_d2 = (float)(r * r);
  m = grid_half_width(g->inv_res, max_d2, g->key_extent);
  if (m > kGridMaxHalfWidth) {
    gb_set_error("region growing search half-width %d exceeds %d", m, kGridMaxHalfWidth);
    return GB_ERR_INTERNAL;
  }
  return GB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// entry points
// ---------------------------------------------------------------------------------------------
extern "C" gb_status gb_concat_frames(gb_ctx* ctx, size_t K, const gb_cloud* const* frames, const double* poses, const gb_cell_window* window, gb_cloud** out_cloud,
                                      uint64_t* ids, size_t* num_out) {
  GB_REQUIRE(ctx && out_cloud && num_out, "null argument");
  *out_cloud = nullptr;
  *num_out = 0;
  GB_REQUIRE(K == 0 || (frames && poses), "null frames / poses");
  size_t total = 0;
  bool covs = K > 0, normals = K > 0;
  for (size_t k = 0; k < K; k++) {
    GB_REQUIRE(frames[k] && frames[k]->device == ctx->device, "null frame / frame on another device");
    GB_REQUIRE(frames[k]->n < ((size_t)1 << 32), "a frame of 2^32 points or more");
    for (int e = 0; e < 16; e++) GB_REQUIRE(std::isfinite(poses[16 * k + e]), "a non-finite pose");
    total += frames[k]->n;
    covs = covs && frames[k]->covs;
    normals = normals && (frames[k]->normals || frames[k]->n == 0);
  }
  GB_REQUIRE(total < ((size_t)1 << 30), "too many points");
  if (window) {
    GB_REQUIRE(std::isfinite(window->cell_size) && window->cell_size > 0.0, "cell_size must be positive and finite");
    for (int a = 0; a < 3; a++) GB_REQUIRE(window->lo[a] <= window->hi[a], "lo > hi");
  }
  GB_ENTER(ctx);
  gb_owned<gb_cloud> c(new (std::nothrow) gb_cloud(), cloud_free);
  if (!c) return GB_ERR_INTERNAL;
  c->device = ctx->device;
  c->covs = covs;
  if (total == 0) {
    *out_cloud = c.release();
    return GB_OK;
  }
  const int n = (int)total;
  const size_t N = total, cub_b = gb_cub_temp_bytes(N);
  gb_planes staged;
  gb_sort_tmp t;
  void* d_table;
  ConcatFrame* d_frames;
  int *d_offsets, *d_flags, *d_pos;
  double4* d_pts;
  double* d_cov;
  unsigned long long* d_ids;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    staged = gb_cloud_planes(cv, N, normals);
    t = gb_take_sort_tmp(cv, N, cv.take<char>(cub_b), cub_b);
    d_table = cv.take<char>(K * GB_FRAME_DESC_BYTES);
    d_frames = cv.take<ConcatFrame>(K);
    d_offsets = cv.take<int>(K);
    d_flags = cv.take<int>(N);
    d_pos = cv.take<int>(N);
    d_pts = cv.take<double4>(N);
    d_cov = cv.take<double>(6 * N);
    d_ids = cv.take<unsigned long long>(N);
  }));
  void* h_table;
  ConcatFrame* h_frames;
  int *h_offsets, *h_count;
  unsigned long long* h_ids = nullptr;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) {
    h_table = cv.take<char>(K * GB_FRAME_DESC_BYTES);
    h_frames = cv.take<ConcatFrame>(K);
    h_offsets = cv.take<int>(K);
    h_count = cv.take<int>(1);
    if (ids) h_ids = cv.take<unsigned long long>(N);
  }));
  size_t off = 0;
  for (size_t k = 0; k < K; k++) {
    const double* T = poses + 16 * k;
    h_frames[k].normals = frames[k]->normals;
    h_frames[k].inv_perm = frames[k]->inv_perm;
    for (int r = 0; r < 3; r++)
      for (int cc = 0; cc < 3; cc++) h_frames[k].R[3 * r + cc] = T[4 * cc + r];
    h_offsets[k] = (int)off;
    off += frames[k]->n;
  }
  cudaStream_t st = ctx->stream;
  GB_CUDA(cudaMemcpyAsync(d_frames, h_frames, sizeof(ConcatFrame) * K, cudaMemcpyHostToDevice, st));
  GB_CUDA(cudaMemcpyAsync(d_offsets, h_offsets, sizeof(int) * K, cudaMemcpyHostToDevice, st));
  GB_CHECK(gb_transform_frames(ctx, K, frames, poses, h_table, d_table, d_pts, d_cov));
  const int gb = (n + kSegThreads - 1) / kSegThreads;
  const double inv = window ? 1.0 / window->cell_size : 0.0;
  const int3 lo = window ? make_int3(window->lo[0], window->lo[1], window->lo[2]) : make_int3(0, 0, 0);
  const int3 hi = window ? make_int3(window->hi[0], window->hi[1], window->hi[2]) : make_int3(0, 0, 0);
  GB_CHECK(gb_launch(ctx, "k_concat_flags", k_concat_flags, gb, kSegThreads, 0, n, d_pts, window ? 1 : 0, inv, lo, hi, d_flags));
  GB_CUB(ctx, cub::DeviceScan::InclusiveSum, t.cub, cub_b, d_flags, d_pos, n);
  GB_CHECK(gb_launch(ctx, "k_concat_emit", k_concat_emit, gb, kSegThreads, 0, n, (int)K, d_offsets, d_frames, d_flags, d_pos, d_pts, d_cov, covs ? 1 : 0,
                     staged.p0, staged.p1, staged.p2, staged.normals, d_ids));
  GB_CUDA(cudaMemcpyAsync(h_count, d_pos + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  const size_t M = (size_t)*h_count;
  if (M > 0) {
    GB_CHECK(gb_cloud_build(ctx, c.get(), M, staged, t));
    if (ids) GB_CUDA(cudaMemcpyAsync(h_ids, d_ids, sizeof(unsigned long long) * M, cudaMemcpyDeviceToHost, st));
    GB_CUDA(cudaStreamSynchronize(st));
    if (ids) memcpy(ids, h_ids, sizeof(uint64_t) * M);
  }
  *num_out = M;
  *out_cloud = c.release();
  return GB_OK;
}

extern "C" gb_status gb_region_growing_default_params(gb_region_growing_params* p) {
  GB_REQUIRE(p, "null argument");
  p->distance_threshold = 0.5;
  p->angle_threshold = 10.0 * 3.141592653589793 / 180.0;
  p->dilation_radius = 0.0;
  return GB_OK;
}

extern "C" gb_status gb_region_growing(gb_ctx* ctx, const gb_cloud* cloud, const double seed_point[3], const gb_region_growing_params* prm,
                                       gb_region_growing_result* result, int32_t* selected, int32_t* labels) {
  GB_REQUIRE(ctx && cloud && seed_point && prm && result, "null argument");
  GB_REQUIRE(cloud->device == ctx->device, "the cloud lives on another device");
  GB_REQUIRE(cloud->n == 0 || cloud->normals, "region growing needs the cloud's normals");
  GB_REQUIRE(std::isfinite(seed_point[0]) && std::isfinite(seed_point[1]) && std::isfinite(seed_point[2]), "a non-finite seed point");
  GB_REQUIRE(std::isfinite(prm->distance_threshold) && prm->distance_threshold > 0.0, "distance_threshold must be positive and finite");
  GB_REQUIRE(prm->angle_threshold >= 0.0 && prm->angle_threshold <= 3.141592653589793, "angle_threshold must be in [0, pi]");
  GB_REQUIRE(std::isfinite(prm->dilation_radius) && prm->dilation_radius >= 0.0, "dilation_radius must be finite and non-negative");
  GB_ENTER(ctx);
  memset(result, 0, sizeof(*result));
  result->seed = -1;
  result->status = GB_REGION_NO_SEED;
  const size_t N = cloud->n;
  if (N == 0) return GB_OK;
  const int n = (int)N;
  const bool dilate = prm->dilation_radius > 0.0;
  // the grids first: their builds carve the context's scratch, which then holds this call's arrays
  gb_owned<gb_point_grid> conn(nullptr, grid_release), dil(nullptr, grid_release);
  int mc = 0, md = 0;
  float d2c = 0.f, d2d = 0.f;
  GB_CHECK(rg_grid(ctx, cloud, prm->distance_threshold, conn, mc, d2c));
  if (dilate) GB_CHECK(rg_grid(ctx, cloud, prm->dilation_radius, dil, md, d2d));
  size_t cub_b = 0;
  cub::DeviceSelect::Flagged(nullptr, cub_b, thrust::counting_iterator<int>(0), (const int*)nullptr, (int*)nullptr, (int*)nullptr, n);
  void* d_cub;
  int *d_parent, *d_region, *d_sel, *d_selected, *d_labels;
  RgOut* d_out;
  // out, selected and labels are adjacent: one copy brings them back, into the same layout of the pinned arena
  const auto tail = [&](Carver& cv, RgOut*& o, int*& s, int*& l) {
    o = cv.take<RgOut>(1);
    s = cv.take<int>(N);
    l = cv.take<int>(N);
  };
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_cub = cv.take<char>(cub_b);
    d_parent = cv.take<int>(N);
    d_region = cv.take<int>(N);
    d_sel = dilate ? cv.take<int>(N) : nullptr;
    tail(cv, d_out, d_selected, d_labels);
  }));
  RgOut* h_out;
  int *h_selected, *h_labels;
  GB_CHECK(gb_carve(ctx, ctx->pinned, [&](Carver& cv) { tail(cv, h_out, h_selected, h_labels); }));
  cudaStream_t st = ctx->stream;
  GB_CUDA(cudaMemsetAsync(d_out, 0, sizeof(RgOut), st));
  GB_CUDA(cudaMemsetAsync(&d_out->seed_key, 0xff, sizeof(unsigned long long), st));
  const int gb = (n + kSegThreads - 1) / kSegThreads, hb = (n + kHookThreads - 1) / kHookThreads;
  GB_CHECK(gb_launch(ctx, "k_rg_init", k_rg_init, gb, kSegThreads, 0, n, cloud->p0, cloud->perm, (float)seed_point[0], (float)seed_point[1], (float)seed_point[2],
                     d_parent, d_out));
  const gb_voxelmap* g = grid_map(conn.get());
  GB_CHECK(gb_launch(ctx, "k_rg_hook", k_rg_hook, hb, kHookThreads, 0, n, g->buckets, (uint32_t)(g->num_buckets - 1), g->max_scan, g->cells, g->voxels, mc,
                     g->inv_res, d2c, cloud->normals, cloud->inv_perm, cos(prm->angle_threshold), d_parent));
  GB_CHECK(gb_launch(ctx, "k_rg_label", k_rg_label, gb, kSegThreads, 0, n, cloud->p0, cloud->perm, d_parent, d_labels, d_region, d_out));
  if (dilate) {
    const gb_voxelmap* h = grid_map(dil.get());
    GB_CHECK(gb_launch(ctx, "k_rg_dilate", k_rg_dilate, hb, kHookThreads, 0, n, h->buckets, (uint32_t)(h->num_buckets - 1), h->max_scan, h->cells, h->voxels, md,
                       h->inv_res, d2d, d_region, d_sel));
  }
  GB_CUB(ctx, cub::DeviceSelect::Flagged, d_cub, cub_b, thrust::counting_iterator<int>(0), dilate ? d_sel : d_region, d_selected, &d_out->num_selected, n);
  const char* end = labels ? (const char*)(d_labels + N) : (const char*)(d_selected + N);
  GB_CUDA(cudaMemcpyAsync(h_out, d_out, (size_t)(end - (const char*)d_out), cudaMemcpyDeviceToHost, st));
  GB_CUDA(cudaStreamSynchronize(st));
  if (h_out->seed_key != ~0ull) {
    result->seed = (int32_t)(uint32_t)h_out->seed_key;
    result->status = GB_REGION_FOUND;
  }
  result->num_region = (size_t)h_out->num_region;
  result->num_selected = (size_t)h_out->num_selected;
  result->num_components = (size_t)h_out->num_components;
  if (selected) memcpy(selected, h_selected, sizeof(int32_t) * result->num_selected);
  if (labels) memcpy(labels, h_labels, sizeof(int32_t) * N);
  return GB_OK;
}
